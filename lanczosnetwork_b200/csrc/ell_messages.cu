// Operator products over the ELL rows of lnb_graph_prepare / lnb_graph_prepare_sparse and their adjoints:
// the training formulation's L_e X and sum_e L_e^T (w_e . G_e) without the dense [B,N,N,E1] operators.
//
//   forward:  out[b*N+n, col0 + (e-c0)*D + d] = sum_t (val[b,e,t,n] w[b,n,e]) X[b*N + idx[b,e,t,n], d]
//   adjoint:  gX[b*N+m, d] = sum_e sum_t (valT[b,e,t,m] w[b,i,e]) G[b*N + i, (e-c0)*D + d],  i = idxT[b,e,t,m]
//
// One thread per output row and column group (4 columns on the vector path, 1 otherwise).  A molecule has
// 2-3 bonds per atom, so a row's ELL list is a handful of entries: the kernels are gathers bound by memory
// latency, not arithmetic.  Every output element is one thread's sum in ascending column order (the adjoint:
// per channel, then over the channels in order), with no atomics -- repeated launches are bit-identical, and
// the products are those of the dense training path (see ell_row).  Extents (gext, ell_max) are read on the
// device, so the launches are graph-capturable and never synchronise with the host.
#include "common.cuh"

namespace {

constexpr int EM_THREADS = 256;

struct EllParams {
  const float* val;          // [B, E1, N(slot), N(row)]
  const uint8_t* idx;
  const int32_t* ell_max;    // [B, E1]
  const int32_t* gext;       // [B, 2]: rows past gext[b, 0] are zero
  const float* w;            // [B, N, E1] row weights or nullptr (1)
  const float* in;           // forward: X [B*N, ld_in]; adjoint: G [B*N, ld_in]
  float* out;                // forward: out [B*N, ld_out] from column col0; adjoint: gX [B*N, ld_out]
  int64_t ld_in, ld_out;
  int B, N, E1, c0, nc, D, col0;
};

template <int V> struct Vec;
template <> struct Vec<1> {
  using T = float;
  static __device__ __forceinline__ T load(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void store(float* p, T v) { *p = v; }
  static __device__ __forceinline__ T zero() { return 0.f; }
  static __device__ __forceinline__ void fma(float a, T x, T& acc) { acc = fmaf(a, x, acc); }
  static __device__ __forceinline__ void add(T x, T& acc) { acc += x; }
};
template <> struct Vec<4> {
  using T = float4;
  static __device__ __forceinline__ T load(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
  static __device__ __forceinline__ void store(float* p, T v) { *reinterpret_cast<float4*>(p) = v; }
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ void fma(float a, T x, T& acc) {
    acc.x = fmaf(a, x.x, acc.x); acc.y = fmaf(a, x.y, acc.y); acc.z = fmaf(a, x.z, acc.z); acc.w = fmaf(a, x.w, acc.w);
  }
  static __device__ __forceinline__ void add(T x, T& acc) { acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w; }
};

// One ELL row's sum over src rows, in ascending column order: graph_prepare lists a row's diagonal first
// (slot 0, when present) and the other columns ascending, so the diagonal is taken between the columns
// below and above it.  With one accumulator, fmaf and ascending columns this is the order in which the
// strided batched GEMM sums a dense operator row (its zero entries leave the sum unchanged), and each entry's
// coefficient is val * w rounded once, as the dense path's row-normalised operator holds it: on 0/1 operators
// the two paths give the same bits.  wb: the channel's weights w[b, 0, e] (stride E1) or nullptr; wfix >= 0
// reads the weight of row wfix for every entry (forward), else that of the gathered row (adjoint).
template <int V>
__device__ __forceinline__ void ell_row(const EllParams& p, int64_t line, int len, int self, const float* src,
                                        const float* wb, int wfix, typename Vec<V>::T& acc) {
  using Op = Vec<V>;
  auto coef = [&](float v, int m) { return wb ? v * __ldg(wb + (int64_t)(wfix >= 0 ? wfix : m) * p.E1) : v; };
  int t = 0;
  float dv = 0.f;
  if (len > 0 && __ldg(p.idx + line) == self) { dv = __ldg(p.val + line); t = 1; }
  for (; t < len; ++t) {
    const float v = __ldg(p.val + line + (int64_t)t * p.N);
    if (v == 0.f) break;                                 // slots past the row's entries are zero padding
    const int m = __ldg(p.idx + line + (int64_t)t * p.N);
    if (dv != 0.f && m > self) {
      Op::fma(coef(dv, self), Op::load(src + (int64_t)self * p.ld_in), acc);
      dv = 0.f;
    }
    Op::fma(coef(v, m), Op::load(src + (int64_t)m * p.ld_in), acc);
  }
  if (dv != 0.f) Op::fma(coef(dv, self), Op::load(src + (int64_t)self * p.ld_in), acc);
}

// idx = ((row * nc) + (e - c0)) * groups + g: consecutive threads read consecutive columns of one gathered row
template <int V>
__global__ void __launch_bounds__(EM_THREADS) ell_messages_kernel(const EllParams p) {
  using Op = Vec<V>;
  const int groups = (p.D + V - 1) / V;
  const int64_t total = (int64_t)p.B * p.N * p.nc * groups;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= total) return;
  const int d = (int)(tid % groups) * V;
  const int ec = (int)((tid / groups) % p.nc);
  const int64_t row = tid / ((int64_t)groups * p.nc);
  const int b = (int)(row / p.N), n = (int)(row - (int64_t)b * p.N);
  const int e = p.c0 + ec;
  typename Op::T acc = Op::zero();
  if (n < __ldg(p.gext + 2 * b)) {
    const int64_t line = ((int64_t)(b * p.E1 + e) * p.N) * p.N + n;
    ell_row<V>(p, line, __ldg(p.ell_max + b * p.E1 + e), n, p.in + (int64_t)b * p.N * p.ld_in + d,
               p.w ? p.w + (int64_t)b * p.N * p.E1 + e : nullptr, n, acc);
  }
  Op::store(p.out + row * p.ld_out + p.col0 + (int64_t)ec * p.D + d, acc);
}

// idx = row * groups + g; the transposed operator's ELL rows (val, idx, ell_max, gext of prep_t).  Each
// channel's sum is its own partial, added to the total in channel order (the dense path sums its per-channel
// products the same way).
template <int V>
__global__ void __launch_bounds__(EM_THREADS) ell_messages_adjoint_kernel(const EllParams p) {
  using Op = Vec<V>;
  const int groups = (p.D + V - 1) / V;
  const int64_t total = (int64_t)p.B * p.N * groups;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= total) return;
  const int d = (int)(tid % groups) * V;
  const int64_t row = tid / groups;
  const int b = (int)(row / p.N), m = (int)(row - (int64_t)b * p.N);
  typename Op::T acc = Op::zero();
  if (m < __ldg(p.gext + 2 * b)) {
    const float* gb = p.in + (int64_t)b * p.N * p.ld_in + d;
    for (int ec = 0; ec < p.nc; ++ec) {
      const int e = p.c0 + ec;
      typename Op::T part = Op::zero();
      ell_row<V>(p, ((int64_t)(b * p.E1 + e) * p.N) * p.N + m, __ldg(p.ell_max + b * p.E1 + e), m,
                 gb + (int64_t)ec * p.D, p.w ? p.w + (int64_t)b * p.N * p.E1 + e : nullptr, -1, part);
      Op::add(part, acc);
    }
  }
  Op::store(p.out + row * p.ld_out + d, acc);
}

int ell_checks(const char* who, const EllParams& p) {
  LNB_REQUIRE(p.val && p.idx && p.ell_max && p.gext && p.in && p.out, "%s: null pointer", who);
  LNB_REQUIRE(p.B >= 0 && p.N >= 1 && p.E1 >= 1 && p.D >= 1, "%s: bad dims B=%d N=%d E1=%d D=%d", who, p.B, p.N,
              p.E1, p.D);
  if (p.N > LNB_MAX_N || p.E1 > LNB_MAX_E1) {
    lnb::set_err("%s: N=%d E1=%d outside the kernel (N <= %d, E1 <= %d)", who, p.N, p.E1, LNB_MAX_N, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  LNB_REQUIRE(p.c0 >= 0 && p.nc >= 1 && p.c0 + p.nc <= p.E1, "%s: channels [%d, %d) outside [0, %d)", who, p.c0,
              p.c0 + p.nc, p.E1);
  LNB_REQUIRE(p.col0 >= 0, "%s: negative column offset", who);
  return LNB_OK;
}

// the vector path needs every row start and column offset on a 16-byte boundary
bool vec4_ok(const EllParams& p) {
  return p.D % 4 == 0 && p.ld_in % 4 == 0 && p.ld_out % 4 == 0 && p.col0 % 4 == 0 &&
         ((uintptr_t)p.in | (uintptr_t)p.out) % 16 == 0;
}

}  // namespace

extern "C" {

int lnb_ell_messages(lnb_stream_t stream, const float* X, int64_t ldx, const float* ell_val, const uint8_t* ell_idx,
                     const int32_t* ell_max, const int32_t* gext, const float* w, int B, int N, int E1, int c0,
                     int nc, int D, float* out, int64_t ldo, int col0) {
  EllParams p{ell_val, ell_idx, ell_max, gext, w, X, out, ldx, ldo, B, N, E1, c0, nc, D, col0};
  const int rc = ell_checks("ell_messages", p);
  if (rc != LNB_OK) return rc;
  LNB_REQUIRE(ldx >= D && ldo >= (int64_t)col0 + (int64_t)nc * D,
              "ell_messages: row strides ldx=%lld ldo=%lld too short for D=%d, col0=%d, nc=%d", (long long)ldx,
              (long long)ldo, D, col0, nc);
  const bool v4 = vec4_ok(p);
  const int64_t total = (int64_t)B * N * nc * (v4 ? D / 4 : D);
  if (total == 0) return LNB_OK;
  const int grid = lnb::ceil_div(total, EM_THREADS);
  if (v4) ell_messages_kernel<4><<<grid, EM_THREADS, 0, (cudaStream_t)stream>>>(p);
  else ell_messages_kernel<1><<<grid, EM_THREADS, 0, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("ell_messages");
}

int lnb_ell_messages_adjoint(lnb_stream_t stream, const float* G, int64_t ldg, const float* ellT_val,
                             const uint8_t* ellT_idx, const int32_t* ellT_max, const int32_t* gextT, const float* w,
                             int B, int N, int E1, int c0, int nc, int D, float* gX, int64_t ldgx) {
  EllParams p{ellT_val, ellT_idx, ellT_max, gextT, w, G, gX, ldg, ldgx, B, N, E1, c0, nc, D, 0};
  const int rc = ell_checks("ell_messages_adjoint", p);
  if (rc != LNB_OK) return rc;
  LNB_REQUIRE(ldg >= (int64_t)nc * D && ldgx >= D,
              "ell_messages_adjoint: row strides ldg=%lld ldgx=%lld too short for D=%d, nc=%d", (long long)ldg,
              (long long)ldgx, D, nc);
  LNB_REQUIRE(gX != G, "ell_messages_adjoint: gX must not alias G");
  const bool v4 = vec4_ok(p);
  const int64_t total = (int64_t)B * N * (v4 ? D / 4 : D);
  if (total == 0) return LNB_OK;
  const int grid = lnb::ceil_div(total, EM_THREADS);
  if (v4) ell_messages_adjoint_kernel<4><<<grid, EM_THREADS, 0, (cudaStream_t)stream>>>(p);
  else ell_messages_adjoint_kernel<1><<<grid, EM_THREADS, 0, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("ell_messages_adjoint");
}

}  // extern "C"
