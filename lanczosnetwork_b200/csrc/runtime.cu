// ABI version, thread-local error text, launch counter.
#include "common.cuh"

namespace lnb {

static thread_local char g_err[512] = {0};
static thread_local int64_t g_launches = 0;

char* err_buf() { return g_err; }

void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches += n; }

static unsigned long long* g_prof_buf = nullptr;
unsigned long long* prof_buffer() { return g_prof_buf; }
void set_prof_buffer(unsigned long long* p) { g_prof_buf = p; }

static int g_max_ctas = 0;
int debug_max_ctas() { return g_max_ctas; }

}  // namespace lnb

extern "C" {

int lnb_abi_version(void) { return 1; }

const char* lnb_last_error(void) { return lnb::err_buf(); }

int64_t lnb_launch_count(void) { return lnb::g_launches; }

// Profiling aid: register (or clear with NULL) a device buffer of SMs x 32 uint64 phase timers.  The
// skeleton kernels read it through their translation unit's copy of the pointer (tcg::g_prof), which
// tcg::launch updates with a synchronous copy at the first launch after a change.  That launch must
// not be inside a stream capture, and until it runs, replays of captured graphs see the old buffer.
int lnb_debug_set_prof(unsigned long long* buf) {
  lnb::set_prof_buffer(buf);
  return LNB_OK;
}

// Testing aid: cap the grid of every persistent wgmma launch (tcg::persistent_grid) at n > 0 CTAs;
// 0 removes the cap.
int lnb_debug_set_max_ctas(int n) {
  LNB_REQUIRE(n >= 0, "debug_set_max_ctas: n=%d must be >= 0", n);
  lnb::g_max_ctas = n;
  return LNB_OK;
}

}  // extern "C"
