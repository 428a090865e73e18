// Persistent wgmma 3xTF32 GEMM skeleton (sm_90a):
//     D[128 x 128 tile] = sum_k A[rows, k] * W[n, k]        fp32-grade accuracy from TF32 MMAs
// The A operand of every 128x32 k-block is PRODUCED BY CUDA-CORE WARPS straight into shared
// memory (row r <-> 128-byte row r of the SWIZZLE_128B operand layout, split into tf32 hi / lo),
// so a policy can either load rows from HBM (dense layer) or compute them on the fly (fused graph
// messages) -- the tensor-core side is identical.  W_hi / W_lo tiles arrive by TMA (SWIZZLE_128B)
// through an mbarrier ring.
//
// Accuracy: tensor-core accumulation truncates, so the 3 split products are kept in two
// accumulators -- D_main += A_hi*W_hi and D_corr += A_lo*W_hi + A_hi*W_lo -- and summed in fp32
// by the epilogue (the small terms no longer add truncation steps to the large accumulator).
//
// CTA = 12 warps, 1 CTA / SM, persistent over tiles (12 warps = 3 per SM sub-partition, which
// leaves 168 registers per thread for the 128 accumulator registers of a consumer):
//   warps 0-3       producers (thread r <-> tile row r), then epilogue (Policy::store)
//   warps 4-11      two consumer warpgroups: warpgroup c owns tile rows [64 c, 64 c + 64) and
//                   keeps D_main and D_corr (64 x 128 fp32 each) in registers; per k-step three
//                   m64n128k8 wgmma: A_hi W_hi -> D_main, A_hi W_lo -> D_corr, A_lo W_hi -> D_corr.
//                   Every consumer warp runs the W cursor and its waits; the elected lane of warp 4
//                   issues the W tile loads (TMA, predicated inside the asm), kStagesB k-blocks ahead.
//                   Policies without acc_init keep one MMA group queued (wgmma.wait_group 1).
// A policy with kProducerGroups = 2 runs 16 warps: two producer warpgroups (warps 0-7) that take
// alternate k-blocks and split the epilogue's columns, and the consumers in warps 8-15.  512 threads
// start at 128 registers; setmaxnreg takes the producers down to 88 and the consumers up to 168.
// The accumulators reach the epilogue through shared memory: once a step's last k-block is
// multiplied the A ring is dead, and the consumers drain [D_main + D_corr] into it in column
// passes that the producer threads read back row by row.  A policy may instead have the consumers
// turn a step's accumulators straight into the next step's A operand (operand_from_acc below).
#pragma once
#include "common.cuh"
#include "sm90.cuh"
#include <stdlib.h>
#include <type_traits>
#include <utility>

namespace tcg {

constexpr int BM = 128, BN = 128, BK = 32;
static_assert(LNB_MAX_WIDTH <= BN, "a row of the widest layer fits one output tile");
constexpr int TILE_B_BYTES = BN * BK * 4;          // 16 KB per hi or lo tile
constexpr int STAGE_B_BYTES = 2 * TILE_B_BYTES;    // [W_hi tile | W_lo tile] = 256 rows x 128 B
constexpr int TILE_A_BYTES = BM * BK * 4;          // 16 KB per hi or lo A block
constexpr int STAGE_A_BYTES = 2 * TILE_A_BYTES;    // [A_hi | A_lo]
constexpr int EW = 16;                             // epilogue unit: 16 accumulator columns
constexpr int CONSUMER_THREADS = 256;
constexpr int CONSUMER_REGS = 168;                 // registers per consumer thread with two producer groups
constexpr int MAX_B_STAGES = 6, MAX_A_STAGES = 4;

// Producer groups of a policy: Policy::kProducerGroups (1 or 2), 1 without it.  Group g is warps
// [4 g, 4 g + 4) and produces the k-blocks whose running count (over all steps) is g modulo the
// group count; thread r of every group owns tile row r.
template <class P, class = void> struct ProducerGroups : std::integral_constant<int, 1> {};
template <class P>
struct ProducerGroups<P, std::void_t<decltype(P::kProducerGroups)>> : std::integral_constant<int, P::kProducerGroups> {};
template <class P> constexpr int producer_threads = 128 * ProducerGroups<P>::value;
template <class P> constexpr int cta_threads = producer_threads<P> + CONSUMER_THREADS;
// With two groups the 512 threads start at 128 registers each: the producers give theirs down to
// this and the consumers take CONSUMER_REGS (2 x 128 x 88 + 2 x 128 x 168 = 65,536)
template <class P> constexpr int producer_regs = (65536 - CONSUMER_THREADS * CONSUMER_REGS) / producer_threads<P> / 8 * 8;
// shared memory of the skeleton: W ring + A ring (Policy::kStagesB / kStagesA stages) + barriers
__host__ __device__ constexpr int core_smem(int stages_b, int stages_a) {
  return stages_b * STAGE_B_BYTES + stages_a * STAGE_A_BYTES + 256;
}
// accumulator columns one drain pass moves through the A ring
__host__ __device__ constexpr int pass_cols(int stages_a) {
  return stages_a * STAGE_A_BYTES / (BM * 4) < BN ? stages_a * STAGE_A_BYTES / (BM * 4) : BN;
}

// The A ring, from the policy's shared memory (which follows the skeleton's)
__device__ __forceinline__ uint8_t* a_ring(uint8_t* policy_smem, int stages_b, int stages_a) {
  return policy_smem - core_smem(stages_b, stages_a) + stages_b * STAGE_B_BYTES;
}

struct Core {
  uint8_t* Bst;        // [kStagesB][hi 16 KB | lo 16 KB]   W tiles
  uint8_t* Ast;        // [kStagesA][hi 16 KB | lo 16 KB]   A k-blocks; drain buffer of the epilogue
  uint64_t* b_full;    // [kStagesB]  TMA arrive.expect_tx
  uint64_t* b_empty;   // [kStagesB]  one arrival per consumer warp
  uint64_t* a_full;    // [kStagesA]  one arrival per producer thread
  uint64_t* a_empty;   // [kStagesA]  one arrival per consumer warp
  uint64_t* stg_full;  // [1]         drain pass written (every consumer thread)
  uint64_t* stg_empty; // [1]         drain pass read (every producer thread)
  uint64_t* kept_read; // [1]         a drain kept in the A ring has been read (one arrival per consumer warp)
};

__device__ __forceinline__ Core carve(uint8_t* base, int stages_b, int stages_a) {
  Core c;
  c.Bst = base;
  c.Ast = base + stages_b * STAGE_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(c.Ast + stages_a * STAGE_A_BYTES);
  c.b_full = bars;
  c.b_empty = c.b_full + MAX_B_STAGES;
  c.a_full = c.b_empty + MAX_B_STAGES;
  c.a_empty = c.a_full + MAX_A_STAGES;
  c.stg_full = c.a_empty + MAX_A_STAGES;
  c.stg_empty = c.stg_full + 1;
  c.kept_read = c.stg_empty + 1;
  return c;
}

// Optional phase timers (profiling aid): when a buffer is registered with lnb_debug_set_prof (launch()
// points g_prof at it), thread 0 of every CTA accumulates clock64() deltas per phase into
// prof[cta*32 + phase] (slots 8 / 9: k-loop / accumulator wait of odd sub-steps, 10: post_epilogue):
//   0 staging issue  1 staging wait (policy)  3 k-loop  4 pre_epilogue
//   5 wait for the accumulator  7 epilogue store
// Slot 14 is the consumers' operand hand-over (operand_from_acc), timed by the first consumer thread.
__device__ unsigned long long* g_prof = nullptr;

struct PhaseTimer {          // thread 0 of the CTA only; no-op unless a buffer is registered
  unsigned long long* buf;
  long long t0;
  __device__ __forceinline__ void start(int cta, int tid) {
    buf = (tid == 0 && g_prof) ? g_prof + cta * 32 : nullptr;
    if (buf) t0 = clock64();
  }
  __device__ __forceinline__ void start_if(int cta, bool owner) {   // timed by another thread than 0
    buf = (owner && g_prof) ? g_prof + cta * 32 : nullptr;
    if (buf) t0 = clock64();
  }
  __device__ __forceinline__ void lap(int slot) {
    if (buf) { long long t = clock64(); atomicAdd(&buf[slot], (unsigned long long)(t - t0)); t0 = t; }
  }
};

template <class Policy>
__device__ __forceinline__ void producers_sync() {   // named barrier 1: all producer threads (every group)
  asm volatile("bar.sync 1, %0;" ::"n"(producer_threads<Policy>) : "memory");
}
__device__ __forceinline__ void consumers_sync() {   // named barrier 2: both consumer warpgroups
  asm volatile("bar.sync 2, %0;" ::"n"(CONSUMER_THREADS) : "memory");
}

// Element (row, col) of a drain pass of `pw` columns: 16-byte chunks XOR-swizzled by row, so the
// row-per-thread reads of the producers are free of bank conflicts.
__device__ __forceinline__ int stg_index(int row, int col, int pw) {
  return row * pw + ((((col >> 2) ^ row) & (pw / 4 - 1)) << 2) + (col & 3);
}

// Policy contract (all __device__).  A "step" is one accumulator lifetime: its k-blocks are
// produced / multiplied, then the epilogue hands the 128 x 128 result to the policy.
//   static constexpr int kStagesB                        depth of the W (shared memory) ring: 1 .. 6
//   static constexpr int kStagesA                        depth of the A (shared memory) ring: 1 .. 4
//   struct Params;                                       kernel parameter block (by value)
//   static int  num_steps(const Params&, int cta, int ncta)       steps this CTA runs
//   static void decode(const Params&, int cta, int ncta, int it, int& m_tile, int& sub)
//   static int  num_kblocks(const Params&, int sub)
//   static void w_coords(const Params&, int sub, int kb, int& col0, int& row0)   TMA coords of W
//   static constexpr int kProducerGroups                  optional, 1 (default) or 2: see ProducerGroups
//   Policy(const Params&, uint8_t* policy_smem, int tid)  constructed by producer threads only (tid <
//                                                         producer_threads<Policy>)
//   void step_begin(int m_tile, int sub, int kb_first, PhaseTimer&)   may call producers_sync(); kb_first =
//                                                         this thread's group's first k-block of the step
//   void produce(int sub, int kb, float (&v)[32])         the 32 A values of this thread's row; called
//                                                         for this thread's group's k-blocks only
//   void pre_epilogue(int sub)                            after the step's last produce()
//   void post_epilogue(int sub)                           after the step's last store(), behind
//                                                         producers_sync()
//   void store(int sub, int col, float (&x)[EW])          accumulator columns [col, col+EW) of
//                                                         this thread's row (main + corr summed); with
//                                                         two groups, group g stores the 16-column
//                                                         units col / EW = g (mod 2)
// Optional pair (a policy whose step starts from the previous step's result; without it every
// accumulator starts at zero):
//   static bool drain_kept(const Params&, int sub)        the step's drain ([D_main + D_corr], one pass)
//                                                         stays in the A ring: the producers read none of
//                                                         it, and write the next step's first k-block only
//                                                         after every consumer warp has run acc_init();
//                                                         that step and the next have k-blocks
//   static bool acc_init(const Params&, const uint8_t* policy_smem, const float* ring, int sub,
//                        int row0, int cl, float (&d)[128])
//                                                         consumers, before the step's first MMA: true
//                                                         when it set the fragment d (rows row0 and
//                                                         row0 + 8, columns 8 j + cl + {0, 1}); the
//                                                         MMAs then add to it
// Optional pair (a policy whose step multiplies the previous step's activated result; needs
// kStagesA * BK >= BN; acc_operand may read policy shared memory that the producers wrote before
// they produced the previous step's k-blocks, or before an earlier one's):
//   static bool operand_from_acc(const Params&, int sub)  the step's A k-blocks are written by the
//                                                         consumers from the previous step's accumulators
//   static float acc_operand(const Params&, const uint8_t* policy_smem, int sub, int col, float x)
//                                                         consumers: A value of column col of the next
//                                                         step, from column col of step sub's result
//                                                         x = D_main + D_corr
//   The previous step then has no drain.  After its last wgmma.wait every consumer thread writes
//   acc_operand() of its fragment, split into tf32 hi / lo, into k-block col / 32 = A stage col / 32
//   (its own warpgroup's rows, which only its own, retired MMAs read), runs fence.proxy.async, and
//   the consumers meet at named barrier 2; the step's MMAs then read stages 0 .. nkb - 1 without
//   a_full waits or a_empty arrivals (the A ring's mbarrier phases count produced k-blocks only).
//   The producers produce nothing for the step and skip the previous step's drain.  Ordering: the
//   producers write no A stage again until they have read a drain that follows the step (every
//   producer thread reads its row, then producers_sync), and the consumers write that drain only
//   after all of the step's MMAs have retired.  (Consecutive operand_from_acc steps are fine: the
//   drain is then that of the last of them; a CTA's last step is always drained.)
// Optional form of produce (a policy that reuses a row across several of its k-blocks):
//   float produce(int sub, int kb, float (&v)[32])        returns a scale: the A values are
//                                                         __fmul_rn(scale, v[j]).  v is kept from the
//                                                         thread's previous produce() call of the step
//                                                         (undefined at its first), so the policy may
//                                                         leave it as it was.
template <class P, class = void> struct HasAccInit : std::false_type {};
template <class P> struct HasAccInit<P, std::void_t<decltype(&P::acc_init)>> : std::true_type {};
template <class P, class = void> struct HasOperandFromAcc : std::false_type {};
template <class P> struct HasOperandFromAcc<P, std::void_t<decltype(&P::operand_from_acc)>> : std::true_type {};
template <class P>
constexpr bool kScaledProduce =
    std::is_same_v<decltype(std::declval<P&>().produce(0, 0, std::declval<float (&)[32]>())), float>;

// Whether step it + 1 takes its operand from step it's accumulators (operand_from_acc policies only)
template <class Policy>
__device__ __forceinline__ bool next_from_acc(const typename Policy::Params& p, int cta, int ncta, int it,
                                              int nsteps, int& nkb_next) {
  if (it + 1 >= nsteps) return false;
  int m_tile, sub;
  Policy::decode(p, cta, ncta, it + 1, m_tile, sub);
  nkb_next = Policy::num_kblocks(p, sub);
  return Policy::operand_from_acc(p, sub);
}

// Pipeline experiments (LNB_DBG, profiling only; results are wrong with any bit set): bits of the
// kernel's kSkip template parameter, so the production kernel has no branch around its MMAs.
constexpr int SKIP_MMA = 2;      // issue no wgmma
constexpr int SKIP_TMA = 4;      // load no W tile (b_full is armed without a transfer)
// Bits 1 (skip the A stores) and 8 (skip produce()) are read from Params::dbg by the producer warps,
// which issue no wgmma.

template <class Policy, int kSkip>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& map_hi, const CUtensorMap& map_lo,
                                             const typename Policy::Params& p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  // 1024-byte alignment (SWIZZLE_128B) by OFFSETTING the __shared__ array -- keeps the
  // shared address space visible to the compiler (LDS/STS instead of generic LD/ST)
  const uint32_t pad = (1024u - (sm90::smem_u32(smem_raw) & 1023u)) & 1023u;
  uint8_t* base = smem_raw + pad;
  constexpr int SB = Policy::kStagesB, SA = Policy::kStagesA;
  static_assert(SB >= 1 && SB <= MAX_B_STAGES && SA >= 1 && SA <= MAX_A_STAGES, "ring depths");
  constexpr int PW = pass_cols(SA);                 // columns per drain pass
  constexpr int NPASS = BN / PW;
  constexpr bool kAccInit = HasAccInit<Policy>::value;
  static_assert(!kAccInit || NPASS == 1, "a drain kept in the A ring must fit it in one pass");
  constexpr bool kOpAcc = HasOperandFromAcc<Policy>::value;
  // One MMA group queued across k-blocks.  Not with acc_init(): ptxas (CUDA 12.9) then serialises
  // every wgmma (C7515) because acc_init's FMAs define the accumulators, even with the operand
  // fences below; those policies wait for every group, as before.
  constexpr bool kQueue = !kAccInit;
  static_assert(!kOpAcc || SA * BK >= BN, "an operand written from the accumulators needs one A stage per k-block");
  constexpr int NG = ProducerGroups<Policy>::value, PT = producer_threads<Policy>;
  constexpr bool kScaled = kScaledProduce<Policy>;
  static_assert(NG == 1 || (NG == 2 && !kOpAcc && PW % (2 * EW) == 0), "two producer groups: no operand_from_acc");
  Core c = carve(base, SB, SA);
  uint8_t* policy_smem = base + core_smem(SB, SA);
  float* stg = reinterpret_cast<float*>(c.Ast);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // 0 .. NG - 1: producer groups, NG / NG + 1: consumer warpgroups; broadcast from lane 0, so ptxas
  // sees a warp-uniform value
  const int role = __shfl_sync(0xffffffffu, tid / 128, 0);
  const int cta = blockIdx.x, ncta = gridDim.x;
  // num_steps may read memory (the stack's schedule): broadcast, so every count the consumers' loops
  // derive from it is warp-uniform to ptxas as well
  const int nsteps = __shfl_sync(0xffffffffu, Policy::num_steps(p, cta, ncta), 0);
  unsigned long long prof_ns0 = 0;                  // whole-CTA wall time / cycles (slots 11, 12)
  long long prof_c0 = 0;
  if (tid == 0 && g_prof) {
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(prof_ns0));
    prof_c0 = clock64();
  }

  if (warp == PT / 32 && lane == 0) {
    sm90::tma_prefetch_desc(&map_hi);
    sm90::tma_prefetch_desc(&map_lo);
    for (int s = 0; s < SB; ++s) {
      sm90::mbar_init(&c.b_full[s], 1);
      sm90::mbar_init(&c.b_empty[s], CONSUMER_THREADS / 32);
    }
    for (int s = 0; s < SA; ++s) {
      sm90::mbar_init(&c.a_full[s], PT / NG);        // one group produces a k-block
      sm90::mbar_init(&c.a_empty[s], CONSUMER_THREADS / 32);
    }
    sm90::mbar_init(c.stg_full, CONSUMER_THREADS);
    sm90::mbar_init(c.stg_empty, PT);
    sm90::mbar_init(c.kept_read, CONSUMER_THREADS / 32);
    sm90::fence_barrier_init();
  }
  __syncthreads();

  if (NG == 1 ? role == 0 : role < NG) {
    // ================================ producers + epilogue ================================
    if constexpr (NG > 1) sm90::setmaxnreg_dec<producer_regs<Policy>>();
    const int r = tid & 127;                         // tile row of this thread
    const int grp = NG == 1 ? 0 : role;              // producer group
    Policy pol(p, policy_smem, tid);
    uint32_t cnt = 0;                                // k-blocks produced so far
    uint32_t npass = 0;                              // drain passes read so far
    uint32_t nkept = 0;                              // drains kept in the A ring so far
    bool after_kept = false;                         // the previous step's drain is in the A ring
    for (int it = 0; it < nsteps; ++it) {
      int m_tile, sub;
      Policy::decode(p, cta, ncta, it, m_tile, sub);
      int nkb = Policy::num_kblocks(p, sub);
      bool kept = false, to_acc = false;
      if constexpr (kAccInit) kept = Policy::drain_kept(p, sub);
      if constexpr (kOpAcc) {
        if (Policy::operand_from_acc(p, sub)) nkb = 0;      // the consumers write this step's k-blocks
        int nkb_next;
        to_acc = next_from_acc<Policy>(p, cta, ncta, it, nsteps, nkb_next);   // no drain
      }
      PhaseTimer tm;
      tm.start(cta, tid);
      pol.step_begin(m_tile, sub, NG == 1 ? 0 : (int)((grp + NG - cnt % NG) % NG), tm);
      [[maybe_unused]] float v_kept[32];             // kScaled: the row kept across this thread's k-blocks
      for (int kb = 0; kb < nkb; ++kb, ++cnt) {
        if constexpr (NG > 1) {
          if (cnt % NG != (uint32_t)grp) continue;   // another group's k-block
        }
        float v[32];
        [[maybe_unused]] float scale = 1.f;
        if (!(p.dbg & 8)) {
          if constexpr (kScaled) scale = pol.produce(sub, kb, v_kept);
          else pol.produce(sub, kb, v);
        }
        const uint32_t sa = cnt % SA;
        // this group's first k-block of the step: the consumers have read the kept drain, which
        // fills the whole A ring
        if (kAccInit && (NG == 1 ? kb == 0 : kb < NG) && after_kept) {
          sm90::mbar_wait(c.kept_read, nkept & 1u);
          if constexpr (NG == 1) ++nkept;
        }
        sm90::mbar_wait(&c.a_empty[sa], ((cnt / SA) & 1u) ^ 1u);
        if (!(p.dbg & 1)) {
          uint8_t* hi = c.Ast + sa * STAGE_A_BYTES + r * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if constexpr (kScaled) {
#pragma unroll
              for (int i = 4 * j; i < 4 * j + 4; ++i) v[i] = __fmul_rn(scale, v_kept[i]);
            }
            uint4 h, l;
            h.x = sm90::tf32_rna_bits(v[4 * j + 0]); h.y = sm90::tf32_rna_bits(v[4 * j + 1]);
            h.z = sm90::tf32_rna_bits(v[4 * j + 2]); h.w = sm90::tf32_rna_bits(v[4 * j + 3]);
            l.x = sm90::tf32_rna_bits(v[4 * j + 0] - __uint_as_float(h.x));
            l.y = sm90::tf32_rna_bits(v[4 * j + 1] - __uint_as_float(h.y));
            l.z = sm90::tf32_rna_bits(v[4 * j + 2] - __uint_as_float(h.z));
            l.w = sm90::tf32_rna_bits(v[4 * j + 3] - __uint_as_float(h.w));
            const int off = (j ^ (r & 7)) * 16;      // SWIZZLE_128B: 16-byte chunk j of row r
            *reinterpret_cast<uint4*>(hi + off) = h;
            *reinterpret_cast<uint4*>(hi + TILE_A_BYTES + off) = l;
          }
        }
        sm90::fence_proxy_async();                   // visible to the tensor core's operand reads
        sm90::mbar_arrive(&c.a_full[sa]);
      }
      if constexpr (NG > 1) {
        if (kAccInit && after_kept) ++nkept;         // also when the group had no k-block to wait for
      }
      tm.lap((sub & 1) ? 8 : 3);
      pol.pre_epilogue(sub);
      tm.lap(4);
      // ---- epilogue: the consumers drain the accumulators in passes of PW columns; group g takes
      // the 16-column units g, g + NG, ... of its row ----
#pragma unroll 1
      for (int q = 0; q < (kept || to_acc ? 0 : NPASS); ++q, ++npass) {
        sm90::mbar_wait(c.stg_full, npass & 1u);
        if (q == 0) tm.lap((sub & 1) ? 9 : 5);
#pragma unroll 1
        for (int col = q * PW + grp * EW; col < (q + 1) * PW; col += NG * EW) {
          float x[EW];
#pragma unroll
          for (int j = 0; j < EW; j += 4) {
            const float4 t = *reinterpret_cast<const float4*>(stg + stg_index(r, col - q * PW + j, PW));
            x[j] = t.x; x[j + 1] = t.y; x[j + 2] = t.z; x[j + 3] = t.w;
          }
          pol.store(sub, col, x);
        }
        sm90::mbar_arrive(c.stg_empty);
      }
      tm.lap(7);
      producers_sync<Policy>();                      // every row is read before the A ring is rewritten
      pol.post_epilogue(sub);
      tm.lap(10);
      after_kept = kept;
    }
  } else {
    // ================================ MMA consumers ========================================
    if constexpr (NG > 1) sm90::setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = role - NG;                        // rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp & 3;
    float d[128];                                    // [D_main (64 x 128) | D_corr (64 x 128)]
    uint32_t cnt = 0, npass = 0;
    uint32_t nacc = 0;                               // k-blocks written by the consumers (not in the A ring's count)
    bool after_kept = false;                         // the previous step's drain is in the A ring
    const int row0 = wg * 64 + wq * 16 + (lane >> 2), cl = 2 * (lane & 3);
    // W loads: the cursor walks the k-blocks of all steps in order; the load of k-block i waits until
    // every consumer warp has released k-block i - kStagesB.  Every consumer warp runs the cursor and
    // the wait, and the elected lane of the first consumer warp issues the load under a predicate inside
    // the asm: between two MMA groups no consumer warp takes a path another one does not.
    const bool w_issuer = warp == PT / 32;
    int l_it = 0, l_kb = 0, l_nkb = -1, l_sub = 0;
    uint32_t l_cnt = 0;
    auto load_next = [&]() {
      while (l_it < nsteps) {
        if (l_nkb < 0) {
          int mt;
          Policy::decode(p, cta, ncta, l_it, mt, l_sub);
          l_nkb = Policy::num_kblocks(p, l_sub);
        }
        if (l_kb < l_nkb) break;
        ++l_it; l_kb = 0; l_nkb = -1;
      }
      if (l_it >= nsteps) return;
      int col0, row0;
      Policy::w_coords(p, l_sub, l_kb, col0, row0);
      const uint32_t st = l_cnt % SB;
      sm90::mbar_wait_uniform(&c.b_empty[st], ((l_cnt / SB) & 1u) ^ 1u);
      uint8_t* dst = c.Bst + st * STAGE_B_BYTES;
      sm90::tma_load_2d_pair_elected<(kSkip & SKIP_TMA) != 0>(w_issuer, &c.b_full[st], STAGE_B_BYTES, dst, &map_hi,
                                                               dst + TILE_B_BYTES, &map_lo, col0, row0);
      ++l_kb; ++l_cnt;
    };
    // releases the W stage sb_rel and, with a_stage, the A stage sa_rel of a k-block whose MMAs have
    // retired, and loads W kStagesB k-blocks ahead
    auto release = [&](uint32_t sb_rel, bool a_stage, uint32_t sa_rel) {
      sm90::mbar_arrive_pred(&c.a_empty[sa_rel], a_stage && lane == 0);
      sm90::mbar_arrive_pred(&c.b_empty[sb_rel], lane == 0);
      load_next();
    };
    for (int i = 0; i < SB; ++i) load_next();
    for (int it = 0; it < nsteps; ++it) {
      int m_tile, sub;
      Policy::decode(p, cta, ncta, it, m_tile, sub);
      const int nkb = Policy::num_kblocks(p, sub);
      bool kept = false, from_acc = false, to_acc = false;
      int nkb_next = 0;
      if constexpr (kOpAcc) {
        from_acc = Policy::operand_from_acc(p, sub);
        to_acc = next_from_acc<Policy>(p, cta, ncta, it, nsteps, nkb_next);
      }
      if constexpr (kAccInit) {
        kept = Policy::drain_kept(p, sub);
        sm90::wgmma_fence_operand(d);              // acc_init() writes d only after the last step's wait
        if (!Policy::acc_init(p, policy_smem, stg, sub, row0, cl, d)) {
#pragma unroll
          for (int i = 0; i < 128; ++i) d[i] = 0.f;
        }
        if (after_kept) {                            // this warp is done reading the kept drain
          __syncwarp();
          if (lane == 0) sm90::mbar_arrive(c.kept_read);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 128; ++i) d[i] = 0.f;
      }
      sm90::wgmma_fence_operand(d);
      // kQueue: one MMA group stays queued: k-block kb is issued before k-block kb - 1 is waited for,
      // and kb - 1's stages are released once it has retired.  Between two groups there are only
      // mbarrier waits whose retry loops are inside their asm, predicated arrivals and the W
      // cursor, whose branches depend on kernel parameters and loop counters alone.
      for (int kb = 0; kb < nkb; ++kb, ++cnt) {
        const uint32_t acnt = cnt - nacc;            // A ring position (cnt without operand_from_acc)
        const uint32_t sb = cnt % SB, sa = from_acc ? (uint32_t)kb : acnt % SA;
        sm90::mbar_wait_uniform(&c.b_full[sb], (cnt / SB) & 1u);
        if (!from_acc) sm90::mbar_wait_uniform(&c.a_full[sa], (acnt / SA) & 1u);
        if constexpr (!(kSkip & SKIP_MMA)) {
          const uint32_t a_hi = sm90::smem_u32(c.Ast + sa * STAGE_A_BYTES) + wg * 64 * 128;
          const uint32_t a_lo = a_hi + TILE_A_BYTES;
          const uint32_t b = sm90::smem_u32(c.Bst + sb * STAGE_B_BYTES);
          sm90::wgmma_fence_operand(d);
          sm90::wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 8; ++k) {
            const uint64_t ah = sm90::wgmma_desc_kmajor_sw128(a_hi + 32 * k);
            const uint64_t wh = sm90::wgmma_desc_kmajor_sw128(b + 32 * k);
            sm90::wgmma_n128(d, ah, wh, 1u);                                                   // D_main += A_hi W_hi^T
            sm90::wgmma_n128_hi(d, ah, sm90::wgmma_desc_kmajor_sw128(b + TILE_B_BYTES + 32 * k), 1u);   // D_corr += A_hi W_lo^T
            sm90::wgmma_n128_hi(d, sm90::wgmma_desc_kmajor_sw128(a_lo + 32 * k), wh, 1u);     // D_corr += A_lo W_hi^T
          }
          sm90::wgmma_commit();
          if constexpr (kQueue) sm90::wgmma_wait_one();   // k-block kb - 1 has retired
          else sm90::wgmma_wait_all();
          sm90::wgmma_fence_operand(d);
        }
        if constexpr (kQueue) {
          if (kb > 0) release((cnt - 1) % SB, !from_acc, from_acc ? (uint32_t)(kb - 1) : (acnt - 1) % SA);
        } else {
          release(sb, !from_acc, sa);
        }
      }
      // unconditional, so that on every path ptxas sees no group in flight past this point
      if constexpr (!(kSkip & SKIP_MMA)) {
        sm90::wgmma_wait_all();
        sm90::wgmma_fence_operand(d);
      }
      if (kQueue && nkb > 0)                         // the step's last k-block
        release((cnt - 1) % SB, !from_acc, from_acc ? (uint32_t)(nkb - 1) : (cnt - nacc - 1) % SA);
      if (from_acc) nacc += nkb;
      PhaseTimer ctm;
      if (to_acc) ctm.start_if(cta, tid == PT);
      consumers_sync();                              // both warpgroups are done reading the A ring
      if (to_acc) {
        // The next step's operand: k-block kb = A stage kb holds columns [32 kb, 32 kb + 32) of
        // acc_operand(D_main + D_corr), split as the producers split theirs, in SWIZZLE_128B layout
        if constexpr (kOpAcc) {
#pragma unroll
          for (int i = 0; i < 64; i += 2) {
            const int col = 8 * (i / 4) + cl, row = row0 + 8 * ((i / 2) % 2), kb = i / 16;
            if (kb < nkb_next) {
              const float y0 = Policy::acc_operand(p, policy_smem, sub, col, d[i] + d[i + 64]);
              const float y1 = Policy::acc_operand(p, policy_smem, sub, col + 1, d[i + 1] + d[i + 65]);
              uint2 h, l;
              h.x = sm90::tf32_rna_bits(y0); h.y = sm90::tf32_rna_bits(y1);
              l.x = sm90::tf32_rna_bits(y0 - __uint_as_float(h.x));
              l.y = sm90::tf32_rna_bits(y1 - __uint_as_float(h.y));
              uint8_t* dst = c.Ast + kb * STAGE_A_BYTES + row * 128 + (((((col & 31) >> 2) ^ row) & 7) << 4) +
                             (col & 3) * 4;
              *reinterpret_cast<uint2*>(dst) = h;
              *reinterpret_cast<uint2*>(dst + TILE_A_BYTES) = l;
            }
          }
          sm90::fence_proxy_async();                 // visible to the tensor core's operand reads
          consumers_sync();
          ctm.lap(14);
        }
      } else {
        // A kept drain needs no hand-over: the producers read the last drain before they wrote this
        // step's k-blocks, and they write no more until kept_read
#pragma unroll
        for (int q = 0; q < NPASS; ++q, npass += kept ? 0 : 1) {
          if (!kept) sm90::mbar_wait(c.stg_empty, (npass & 1u) ^ 1u);
#pragma unroll
          for (int i = 0; i < 64; i += 2) {
            const int col = 8 * (i / 4) + cl, row = row0 + 8 * ((i / 2) % 2);
            if (col >= q * PW && col < (q + 1) * PW)
              *reinterpret_cast<float2*>(stg + stg_index(row, col - q * PW, PW)) =
                  make_float2(d[i] + d[i + 64], d[i + 1] + d[i + 65]);
          }
          if (!kept) sm90::mbar_arrive(c.stg_full);
        }
      }
      if (kept) consumers_sync();                    // the next acc_init() reads rows of both halves
      after_kept = kept;
    }
  }

  __syncthreads();
  if (tid == 0 && g_prof) {
    unsigned long long ns1;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(ns1));
    atomicAdd(&g_prof[cta * 32 + 11], ns1 - prof_ns0);
    atomicAdd(&g_prof[cta * 32 + 12], (unsigned long long)(clock64() - prof_c0));
    g_prof[cta * 32 + 13] = prof_ns0;               // CTA start (ns), for launch skew
  }
}

template <class Policy>
__global__ void __launch_bounds__(cta_threads<Policy>, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_hi,
               const __grid_constant__ CUtensorMap map_lo, const typename Policy::Params p) {
  tc_gemm_body<Policy, 0>(map_hi, map_lo, p);
}

// The skeleton with pipeline parts switched off (kSkip: SKIP_MMA | SKIP_TMA), for LNB_DBG experiments
template <class Policy, int kSkip>
__global__ void __launch_bounds__(cta_threads<Policy>, 1)
tc_gemm_probe_kernel(const __grid_constant__ CUtensorMap map_hi,
                     const __grid_constant__ CUtensorMap map_lo, const typename Policy::Params p) {
  tc_gemm_body<Policy, kSkip>(map_hi, map_lo, p);
}

// Epilogue helper: bias / ReLU / bounds-checked store of EW accumulator columns of one row.
__device__ __forceinline__ void store_row_chunk(float* orow, int ncols, const float* bias, bool relu,
                                                int col, const float (&x)[EW]) {
  if (orow == nullptr || col >= ncols) return;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(orow + col) & 15) == 0;
#pragma unroll
  for (int j = 0; j < EW; j += 4) {
    float o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int n = col + j + u;
      float y = x[j + u];
      if (n < ncols) {
        if (bias) y += __ldg(bias + n);
        if (relu) y = fmaxf(y, 0.f);
      }
      o[u] = y;
    }
    if (vec_ok && col + j + 3 < ncols) {
      *reinterpret_cast<float4*>(orow + col + j) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (col + j + u < ncols) orow[col + j + u] = o[u];
    }
  }
}

// ---- host helpers --------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;   // idempotent lookup; benign if two threads race
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// Row-major [rows, cols] fp32 weight matrix; box = 32 columns (128 B) x 128 rows; 128 B swizzle.
inline int make_weight_map(CUtensorMap* map, const float* W, int rows, int cols, const char* who,
                           int box_rows = BN) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) { lnb::set_err("%s: cuTensorMapEncodeTiled unavailable", who); return LNB_ERR_UNSUPPORTED; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(W), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    lnb::set_err("%s: cuTensorMapEncodeTiled failed (CUresult %d)", who, (int)r);
    return LNB_ERR_ARG;
  }
  return LNB_OK;
}

// LNB_DBG=<bits>: pipeline experiments (1 skip A stores, 2 skip MMA issue, 4 skip TMA loads,
// 8 skip produce()).  Results are wrong with any bit set; for profiling only.  Bits 2 and 4 select a
// tc_gemm_probe_kernel instantiation in launch(); bits 1 and 8 are read by the producer warps.
inline int debug_flags() {
  const char* e = getenv("LNB_DBG");
  return e ? atoi(e) : 0;
}

inline int sm_count() {
  int dev = 0, n = 132;
  if (cudaGetDevice(&dev) == cudaSuccess)
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

// CTAs of a persistent launch over `items` work items: min(items, SMs), and at most each positive
// bound of max_ctas and the testing cap of lnb_debug_set_max_ctas
inline int persistent_grid(int items, int max_ctas = 0) {
  int grid = items < sm_count() ? items : sm_count();
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  const int cap = lnb::debug_max_ctas();
  if (cap > 0 && grid > cap) grid = cap;
  return grid;
}

// g_prof is defined in this header, so every translation unit has its own copy.  Each points its
// copy at the buffer registered with lnb_debug_set_prof when that has changed since its last launch
// (a synchronous copy; with no buffer ever registered nothing is copied).
static unsigned long long* g_prof_mirrored = nullptr;

static int sync_prof_buffer(const char* who) {
  unsigned long long* buf = lnb::prof_buffer();
  if (buf == g_prof_mirrored) return LNB_OK;
  cudaError_t e = cudaMemcpyToSymbol(g_prof, &buf, sizeof(buf));
  if (e != cudaSuccess) { lnb::set_err("%s: %s", who, cudaGetErrorString(e)); return (int)e; }
  g_prof_mirrored = buf;
  return LNB_OK;
}

// Launches tc_gemm_kernel<Pol> on persistent_grid(items, max_ctas) persistent CTAs with `smem` bytes of
// dynamic shared memory; W_hi / W_lo are the split row-major [w_rows, w_cols] weights the TMA streams.
template <class Pol>
static int launch(lnb_stream_t stream, const float* W_hi, const float* W_lo, int w_rows, int w_cols,
                  size_t smem, int items, const typename Pol::Params& p, const char* who,
                  int max_ctas = 0) {
  CUtensorMap map_hi, map_lo;
  int rc = make_weight_map(&map_hi, W_hi, w_rows, w_cols, who);
  if (rc != LNB_OK) return rc;
  rc = make_weight_map(&map_lo, W_lo, w_rows, w_cols, who);
  if (rc != LNB_OK) return rc;
  rc = sync_prof_buffer(who);
  if (rc != LNB_OK) return rc;
  const int skip = p.dbg & (SKIP_MMA | SKIP_TMA);
  auto kern = skip == 0                    ? tc_gemm_kernel<Pol>
              : skip == SKIP_MMA           ? tc_gemm_probe_kernel<Pol, SKIP_MMA>
              : skip == SKIP_TMA           ? tc_gemm_probe_kernel<Pol, SKIP_TMA>
                                           : tc_gemm_probe_kernel<Pol, SKIP_MMA | SKIP_TMA>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kern<<<persistent_grid(items, max_ctas), cta_threads<Pol>, smem, (cudaStream_t)stream>>>(map_hi, map_lo, p);
  lnb::count_launch();
  return lnb::finish_launch(who);
}

}  // namespace tcg
