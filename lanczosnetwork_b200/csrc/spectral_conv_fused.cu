// Fused spectral graph-convolution layer (reference: model/lanczos_net.py:157-182):
//     msg = [ V diag(f_s) V^T X  (s < S) ] ++ [ L_e X  (e <= E) ];   X' = ReLU(cat(msg) W^T + b)
// as ONE persistent wgmma kernel (skeleton: tc_gemm.cuh).  Nothing of the reference's
// intermediate tensors exists in HBM: not the N x N filters, not the [B*N, C*D] message matrix.
//
// Tiles are PACKED: lnb_graph_prepare measures every graph's real extent (n_eff rows/columns
// of the operators that are not identically zero, k_eff non-zero Ritz vectors) and assigns
// graphs to 128-row tiles by first-fit decreasing (sum n_eff <= 128, sum k_eff <= 128, <= 32
// graphs; the tile schedule, below the next-fit table of the C ABI).  A QM8-shaped batch of 1024
// molecules (16 real atoms on average, padded to 26) becomes 128-129 tiles -- one wave of the 132
// SMs -- instead of 256 fixed-slot tiles (next-fit over consecutive graphs: 142-143, two waves).
// Rows that are pure padding are never multiplied; their (constant) output act(b) is written directly.
// Dropping exact zeros is exact, so the result equals the dense reference for arbitrary inputs.
//
// Two accumulator lifetimes ("steps") per tile:
//   step 0  Z = sum_s (f_s . U) W_s^T      rows = (graph, Ritz index), k-blocks by pairs of d-blocks
//           (s0_kblock: each producer group takes all k-blocks of one d-block of a pair): at the
//           group's first k-block of a d-block the producer thread of row (g, k) computes its 32
//           columns of U_g = V_g^T X_g into registers, then scales them by f_s for every s; Z is
//           drained into the A ring and stays there;
//   step 1  E = sum_e (L_e X) W_e^T        rows = (graph, node): sparse ELL rows of the operators
//           times X, accumulated on top of V Z, which the consumers compute from the Z in the A
//           ring before the first MMA; epilogue: out = act(acc + b).
// Algebra: sum_s V diag(f_s) V^T X W_s^T = V [ sum_s diag(f_s) (V^T X) W_s^T ].
#include "tc_gemm.cuh"

namespace {

constexpr int GMAX = 32;        // max graphs per tile
constexpr int RMAX = 128;       // rows per tile
static_assert(LNB_MAX_N <= RMAX, "every graph of the envelope fits one tile");

// --------------------------------------------------------------------------------------------
// Per-forward operator compression and extents.
//   ell_val/ell_idx [B, E1, N(t), N(n)]: the t-th non-zero of row n of channel e (t-major so a
//   warp of consecutive rows reads consecutive addresses; the diagonal entry first, then by
//   column); ell_max[b,e] = max non-zeros per row.
//   gext[b] = {n_eff, k_eff}: the operators are zero outside their leading n_eff rows/columns,
//   Q[b] is zero outside its leading n_eff rows / k_eff columns.
// --------------------------------------------------------------------------------------------
template <bool STAGE>   // STAGE: this graph's operators fit in shared memory
__global__ void __launch_bounds__(256)
graph_prepare_kernel(const float* __restrict__ L, const float* __restrict__ Q, int N, int E1, int K,
                     float* __restrict__ ell_val, uint8_t* __restrict__ ell_idx,
                     int32_t* __restrict__ ell_max, int32_t* __restrict__ gext, int binarize) {
  extern __shared__ __align__(16) float gp_smem[];     // [N*N*E1] this graph's operators (optional)
  __shared__ int s_max[LNB_MAX_E1];
  __shared__ int s_ext[2];
  __shared__ uint8_t cnt_s[(LNB_MAX_N_ELL + 1) * LNB_MAX_E1];  // non-zeros per (row, channel)
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid < LNB_MAX_E1) s_max[tid] = 0;
  if (tid < 2) s_ext[tid] = 0;
  const int64_t per = (int64_t)N * N * E1;
  const float* Lg = L + b * per;
  if (STAGE) {                                         // coalesced async copy; strided reads then hit smem
    if ((per & 3) == 0) {
      for (int i = tid; i < (int)(per >> 2); i += 256) sm90::cp_async_16(gp_smem + 4 * i, Lg + 4 * i);
    } else {
      for (int i = tid; i < (int)per; i += 256) sm90::cp_async_4(gp_smem + i, Lg + i);
    }
  }
  const float* Lb = STAGE ? gp_smem : Lg;
  // extents of Q while the operator copy is in flight
  const float* Qb = Q + (int64_t)b * N * K;
  int ne = 0, ke = 0;
  for (int i = tid; i < N * K; i += 256) {
    if (__ldg(Qb + i) != 0.f) {
      ne = max(ne, i / K + 1);
      ke = max(ke, i % K + 1);
    }
  }
  if (STAGE) sm90::cp_async_wait_all();
  __syncthreads();
  const int pairs = N * E1;
  // thread <-> (row n, channel e), p = n*E1 + e: one pass over the row, compacting as it goes
  for (int p = tid; p < pairs; p += 256) {
    const int n = p / E1, e = p - n * E1;
    const float* row = Lb + (n * N) * E1 + e;
    float* val = ell_val + ((int64_t)(b * E1 + e) * N) * N + n;
    uint8_t* idx = ell_idx + ((int64_t)(b * E1 + e) * N) * N + n;
    int cnt = 0, far = 0;
    // the diagonal entry goes first: consecutive rows then gather consecutive rows of X for
    // entry 0 (conflict-free in the fused kernel), the other entries follow in column order
    const float dg = row[n * E1];
    if (dg != 0.f) {
      val[0] = binarize ? 1.f : dg;
      idx[0] = (uint8_t)n;
      cnt = 1;
      far = n + 1;
    }
#pragma unroll 2
    for (int i = 0; i < N; ++i) {
      const float v = row[i * E1];
      if (v != 0.f && i != n) {
        val[cnt * N] = binarize ? 1.f : v;
        idx[cnt * N] = (uint8_t)i;
        ++cnt;
        far = max(far, i + 1);
      }
    }
    cnt_s[p] = (uint8_t)cnt;
    if (cnt) {
      atomicMax(&s_max[e], cnt);
      ne = max(ne, max(n + 1, far));
    }
  }
  if (ne) atomicMax(&s_ext[0], ne);
  if (ke) atomicMax(&s_ext[1], ke);
  __syncthreads();
  // zero-fill the tail of every row up to the channel maximum of this graph, so consumers can
  // run all rows of a (graph, channel) to the same length without per-row guards
  for (int pr = tid; pr < pairs; pr += 256) {
    const int n = pr / E1, e = pr - n * E1;
    float* val = ell_val + ((int64_t)(b * E1 + e) * N) * N + n;
    uint8_t* idx = ell_idx + ((int64_t)(b * E1 + e) * N) * N + n;
    for (int t = cnt_s[pr]; t < s_max[e]; ++t) {
      val[(int64_t)t * N] = 0.f;
      idx[(int64_t)t * N] = 0;
    }
  }
  if (tid < E1) ell_max[b * E1 + tid] = s_max[tid];
  if (tid < 2) gext[b * 2 + tid] = s_ext[tid];
}

// (n_eff, k_eff) classes of the schedule's counting sort: n_eff <= RMAX, k_eff <= LNB_CONV_MAX_K
constexpr int SCH_KC = LNB_CONV_MAX_K + 1;
constexpr int SCH_NCLS = (RMAX + 1) * SCH_KC;

// Exclusive prefix sum over the 1024 threads of a block; `total` = sum of all values.
__device__ __forceinline__ int block_scan_excl(int v, int* ws /* [33] shared */, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) ws[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const int w = ws[lane];
    int s = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    ws[lane] = s - w;
    if (lane == 31) ws[32] = s;
  }
  __syncthreads();
  const int r = ws[warp] + inc - v;
  total = ws[32];
  __syncthreads();
  return r;
}

// Schedule = the next-fit tiles in graph order (always valid: next-fit keeps sum ceil4(k_eff) <= 128,
// so also sum k_eff <= 128).  Reads the finished table; every thread of the block calls it.
__device__ void identity_schedule(int32_t* __restrict__ tiles, int B, int T) {
  int32_t* S = tiles + B + 2;
  for (int i = threadIdx.x; i <= T; i += blockDim.x) S[1 + i] = tiles[1 + i];
  for (int i = threadIdx.x; i < B; i += blockDim.x) S[T + 2 + i] = i;
  if (threadIdx.x == 0) S[0] = T;
}

// Next-fit assignment of consecutive graphs to tiles.  tiles[0] = T, tiles[1 + t] = first graph
// of tile t, tiles[1 + T] = B.  One CTA, all of it parallel: inclusive prefix sums of the row /
// Ritz-row counts; for every graph i the end NX[i] of the tile that would start at i (a window of
// <= 32 graphs); the tile starts are the graphs reachable from 0 along NX, found by pointer
// jumping (round k marks the starts 2^k .. 2^(k+1)-1 hops away and squares the jump table); a
// prefix sum over the marks numbers the tiles.  The arrays live in shared memory (6 (B+1) ints);
// batches too large for that use the global scratch and a serial walk.
//
// Then, for B >= 2, the schedule the stack kernel runs, at S = tiles + B + 2:
//   S[0] = T', S[1 + t] = first slot of tile t (t <= T', S[1 + T'] = B), S[T' + 2 + slot] = graph id.
// Rule (data.host_tile_schedule): first-fit decreasing -- graphs by n_eff descending, k_eff
// descending, index ascending; each goes into the lowest tile with sum n_eff <= 128, sum k_eff <= 128
// (unpadded) and <= 32 graphs, or opens a new one.  Identical graphs are placed in bulk, which gives
// exactly what first-fit gives one at a time: a stable counting sort by class (warps 1..31) runs
// beside warp 0, which walks the classes in order and gives every tile, lowest first, as many graphs
// of the class as still fit.  Batches outside the shared-memory path, with K > LNB_CONV_MAX_K or with an
// n_eff > 128 (shapes the stack kernel does not run) get the next-fit tiles in graph order instead.
template <bool in_smem>
__global__ void __launch_bounds__(1024)
tile_assign_kernel(const int32_t* __restrict__ gext, int B, int K, int32_t* __restrict__ tiles,
                   int32_t* __restrict__ scratch /* [3 * B] */, int32_t* __restrict__ rowmap,
                   int32_t* __restrict__ nrows) {
  extern __shared__ int32_t ta_smem[];
  __shared__ int warp_n[32], warp_k[32], warp_r[32];
  __shared__ int run_n, run_k, run_r;
  __shared__ int scan_ws[33];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int32_t* PN = in_smem ? ta_smem : scratch;                     // inclusive prefix of n_eff
  int32_t* PK = PN + B;                                          // inclusive prefix of ceil4(k_eff)
  int32_t* NX = PK + B;                                          // [B + 1] end of the tile starting at i
  int32_t* PR = NX + 3 * (B + 1);                                // (shared memory only) inclusive prefix of k_eff
  if (tid == 0) { run_n = 0; run_k = 0; run_r = 0; }
  __syncthreads();
  for (int b0 = 0; b0 < B; b0 += 1024) {
    const int b = b0 + tid;
    const int n = (b < B) ? gext[b * 2] : 0;
    const int kr = (b < B) ? min(gext[b * 2 + 1], K) : 0;      // rows of the compact Ritz row list
    const int k = (b < B) ? ((gext[b * 2 + 1] + 3) & ~3) : 0;
    int in = n, ik = k, ir = kr;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int tn = __shfl_up_sync(0xffffffffu, in, o), tk = __shfl_up_sync(0xffffffffu, ik, o);
      const int tr = __shfl_up_sync(0xffffffffu, ir, o);
      if (lane >= o) { in += tn; ik += tk; ir += tr; }
    }
    if (lane == 31) { warp_n[warp] = in; warp_k[warp] = ik; warp_r[warp] = ir; }
    __syncthreads();
    if (warp == 0) {
      int wn = warp_n[lane], wk = warp_k[lane], wr = warp_r[lane], sn = wn, sk = wk, sr = wr;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int tn = __shfl_up_sync(0xffffffffu, sn, o), tk = __shfl_up_sync(0xffffffffu, sk, o);
        const int tr = __shfl_up_sync(0xffffffffu, sr, o);
        if (lane >= o) { sn += tn; sk += tk; sr += tr; }
      }
      warp_n[lane] = sn - wn;
      warp_k[lane] = sk - wk;
      warp_r[lane] = sr - wr;
    }
    __syncthreads();
    if (b < B) {
      PN[b] = run_n + warp_n[warp] + in;
      PK[b] = run_k + warp_k[warp] + ik;
      if (in_smem) {
        PR[b] = run_r + warp_r[warp] + ir;
      } else if (rowmap) {                // {b*K + k : k < k_eff(b)}, see lnb_ritz_rowmap
        const int base = run_r + warp_r[warp] + ir - kr;
        for (int i = 0; i < kr; ++i) rowmap[base + i] = b * K + i;
      }
    }
    __syncthreads();
    if (tid == 1023) { run_n += warp_n[31] + in; run_k += warp_k[31] + ik; run_r += warp_r[31] + ir; }
    __syncthreads();
  }
  if (tid == 0 && nrows) nrows[0] = run_r;
  __threadfence_block();
  if (in_smem && rowmap) {
    // coalesced expansion of the row list: a warp writes the k_eff consecutive entries of a graph
    for (int b = warp; b < B; b += 32) {
      const int base = b ? PR[b - 1] : 0, kr = PR[b] - base;
      for (int i = lane; i < kr; i += 32) rowmap[base + i] = b * K + i;
    }
  }
  for (int i = tid; i < B; i += 1024) {
    const int pn0 = i ? PN[i - 1] : 0, pk0 = i ? PK[i - 1] : 0;
    int j = i + 1;                                   // the first graph always fits (n_eff <= 128)
    const int jmax = min(B, i + GMAX);
    while (j < jmax && PN[j] - pn0 <= RMAX && PK[j] - pk0 <= RMAX) ++j;
    NX[i] = j;
  }
  __syncthreads();
  if (!in_smem) {                                    // huge batch: serial walk over the jump table
    if (tid == 0) {
      int T = 0, i = 0;
      while (i < B) { tiles[1 + T] = i; ++T; i = NX[i]; }
      tiles[0] = T;
      tiles[1 + T] = B;
      run_n = T;
    }
    __syncthreads();                                 // the scratch (under the schedule) is dead
    if (B >= 2) identity_schedule(tiles, B, run_n);
    return;
  }
  int32_t* Ja = NX;
  int32_t* Jb = NX + (B + 1);
  int32_t* MK = Jb + (B + 1);
  for (int i = tid; i <= B; i += 1024) MK[i] = (i == 0) ? 1 : 0;
  if (tid == 0) { Ja[B] = B; Jb[B] = B; }
  __syncthreads();
  for (int span = 1; span < B; span <<= 1) {
    // starts fewer than `span` hops from graph 0 are marked; Ja = NX applied `span` times
    for (int i = tid; i < B; i += 1024)
      if (MK[i]) MK[Ja[i]] = 1;                      // late marks only add true starts (idempotent)
    for (int i = tid; i < B; i += 1024) Jb[i] = Ja[Ja[i]];
    __syncthreads();
    int32_t* t = Ja; Ja = Jb; Jb = t;
  }
  // number the starts: exclusive prefix sum of the marks
  if (tid == 0) run_n = 0;
  __syncthreads();
  for (int b0 = 0; b0 < B; b0 += 1024) {
    const int b = b0 + tid;
    const int m = (b < B) ? MK[b] : 0;
    int in = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int tn = __shfl_up_sync(0xffffffffu, in, o);
      if (lane >= o) in += tn;
    }
    if (lane == 31) warp_n[warp] = in;
    __syncthreads();
    if (warp == 0) {
      int wn = warp_n[lane], sn = wn;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int tn = __shfl_up_sync(0xffffffffu, sn, o);
        if (lane >= o) sn += tn;
      }
      warp_n[lane] = sn - wn;
    }
    __syncthreads();
    if (m) tiles[1 + run_n + warp_n[warp] + in - 1] = b;
    __syncthreads();
    if (tid == 1023) run_n += warp_n[31] + in;
    __syncthreads();
  }
  if (tid == 0) {
    tiles[0] = run_n;
    tiles[1 + run_n] = B;
  }
  __syncthreads();                                   // table done; the shared arrays above are dead
  if (B < 2) return;                                 // no room for a schedule: the kernel runs the table
  if (K > LNB_CONV_MAX_K) {
    identity_schedule(tiles, B, run_n);
    return;
  }
  int32_t* S = tiles + B + 2;
  int32_t* key = ta_smem;                            // [B] class of graph b
  int32_t* order = key + B;                          // [B] graph ids sorted by class, stable
  int32_t* tst = order + B;                          // [B] tile state: sum n | sum k << 8 | graphs << 16
  int32_t* rec_t = tst + B;                          // [B] placement records: tile,
  int32_t* rec_src = rec_t + B;                      //     first position in `order`,
  int32_t* rec_sm = rec_src + B;                     //     first slot in the tile | count << 8
  int32_t* hist = ta_smem + 6 * (B + 1);             // [SCH_NCLS] first position of each class in `order`
  int32_t* cls = hist + SCH_NCLS;                    // [SCH_NCLS] the non-empty classes, in order
  for (int i = tid; i < SCH_NCLS; i += 1024) hist[i] = 0;
  __syncthreads();
  // class = (128 - n_eff) * 33 + (32 - k_eff): ascending class = n_eff descending, then k_eff descending
  // A batch has few classes, so the lanes of a warp that share one add to it once.
  bool big = false;
  for (int b0 = 0; b0 < B; b0 += 1024) {
    const int b = b0 + tid;
    int c = -1;
    if (b < B) {
      const int n = gext[b * 2];
      big |= n > RMAX;
      c = (RMAX - min(n, RMAX)) * SCH_KC + (LNB_CONV_MAX_K - min(gext[b * 2 + 1], K));
      key[b] = c;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    if (c >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[c], __popc(peers));
  }
  if (__syncthreads_or(big)) {
    identity_schedule(tiles, B, run_n);
    return;
  }
  {
    constexpr int PER = (SCH_NCLS + 1023) / 1024;
    int cnt[PER], s = 0, ne = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int i = tid * PER + j;
      cnt[j] = i < SCH_NCLS ? hist[i] : 0;
      s += cnt[j];
      ne += cnt[j] > 0;
    }
    int tot;                                         // graphs (low 16 bits) and classes (high bits) at once
    const int ex = block_scan_excl(s | (ne << 16), scan_ws, tot);
    int pos = ex & 0xffff, ci = ex >> 16;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int i = tid * PER + j;
      if (i < SCH_NCLS) {
        hist[i] = pos;
        if (cnt[j]) cls[ci++] = i;
        pos += cnt[j];
      }
    }
    if (tid == 0) run_k = tot >> 16;
  }
  __syncthreads();
  const int ncls = run_k;
  if (warp == 0) {
    // first-fit of whole classes, 32 tiles at a time: lane l looks at tile t0 + l.  A ballot skips
    // the chunks where no tile has room for the class; in the others one warp scan of the room
    // gives every tile, in tile order, the graphs it takes, and a second ballot numbers the
    // placement records.  A class stops at the chunk that uses it up, so a class that fits in
    // the first tiles costs one or two chunks however many tiles are open.
    int T2 = 0, nrec = 0;
    for (int i0 = 0; i0 < ncls; i0 += 32) {
      // lane j describes class i0 + j: first position in `order`, count, n_eff, k_eff, and
      // ceil(2^16 / n), ceil(2^16 / k) for floor(free / n) = free * ceil(2^16 / n) >> 16 (exact for
      // free, n <= 128), the most graphs an empty tile takes
      int c_first = 0, c_count = 0, c_n = 1, c_k = 1;
      if (i0 + lane < ncls) {
        const int c = cls[i0 + lane];
        c_first = hist[c];
        c_count = (i0 + lane + 1 < ncls ? hist[cls[i0 + lane + 1]] : B) - c_first;
        c_n = RMAX - c / SCH_KC;
        c_k = LNB_CONV_MAX_K - c % SCH_KC;
      }
      const int c_rn = c_n ? (65536 + c_n - 1) / c_n : 0, c_rk = c_k ? (65536 + c_k - 1) / c_k : 0;
      const int c_ce = max(1, min(GMAX, min(c_n ? RMAX / c_n : GMAX, c_k ? RMAX / c_k : GMAX)));
      const int nc = min(32, ncls - i0);
      for (int j = 0; j < nc; ++j) {
        const int first = __shfl_sync(0xffffffffu, c_first, j), count = __shfl_sync(0xffffffffu, c_count, j);
        const int n = __shfl_sync(0xffffffffu, c_n, j), k = __shfl_sync(0xffffffffu, c_k, j);
        const int rn = __shfl_sync(0xffffffffu, c_rn, j), rk = __shfl_sync(0xffffffffu, c_rk, j);
        const int ce = __shfl_sync(0xffffffffu, c_ce, j);
        int done = 0;                                  // graphs of the class placed so far
        for (int t0 = 0; t0 < T2 && done < count; t0 += 32) {
          const int t = t0 + lane;
          const int st = t < T2 ? tst[t] : GMAX << 16; // past the last open tile: no room
          int cap = GMAX - (st >> 16);
          if (n) cap = min(cap, ((RMAX - (st & 255)) * rn) >> 16);
          if (k) cap = min(cap, ((RMAX - ((st >> 8) & 255)) * rk) >> 16);
          if (!__ballot_sync(0xffffffffu, cap > 0)) continue;
          int inc = cap;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
          }
          const int m = min(cap, count - done - (inc - cap));   // <= 0: the class is used up before tile t
          const unsigned took = __ballot_sync(0xffffffffu, m > 0);
          if (m > 0) {
            const int r = nrec + __popc(took & ((1u << lane) - 1));
            rec_t[r] = t;
            rec_src[r] = first + done + inc - cap;
            rec_sm[r] = (st >> 16) | (m << 8);
            tst[t] = st + m * n + ((m * k) << 8) + (m << 16);
          }
          nrec += __popc(took);
          done = min(count, done + __shfl_sync(0xffffffffu, inc, 31));
        }
        if (done < count) {                            // the rest opens new tiles, each as full as the limits allow
          const int rem = count - done, nt = (rem + ce - 1) / ce;
          const int rb = nrec;
          nrec += nt;
          for (int q = lane; q < nt; q += 32) {
            const int m = min(ce, rem - q * ce);
            rec_t[rb + q] = T2 + q;
            rec_src[rb + q] = first + done + q * ce;
            rec_sm[rb + q] = m << 8;
            tst[T2 + q] = m * n + ((m * k) << 8) + (m << 16);
          }
          T2 += nt;
        }
        __syncwarp();
      }
    }
    if (lane == 0) { run_n = T2; run_r = nrec; }
  } else {
    // stable counting sort: warp w gathers the graphs of classes w - 1, w + 30, ... in index order
    for (int i = warp - 1; i < ncls; i += 31) {
      const int c = cls[i];
      int dst = hist[c];
      const int end = i + 1 < ncls ? hist[cls[i + 1]] : B;
      for (int b0 = 0; b0 < B && dst < end; b0 += 32) {
        const int b = b0 + lane;
        const bool hit = b < B && key[b] == c;
        const unsigned mk = __ballot_sync(0xffffffffu, hit);
        if (hit) order[dst + __popc(mk & ((1u << lane) - 1))] = b;
        dst += __popc(mk);
      }
    }
  }
  __syncthreads();
  const int T2 = run_n, nrec = run_r;
  // first slot of every tile: exclusive prefix of the graph counts
  int run = 0;
  for (int t0 = 0; t0 < T2; t0 += 1024) {
    const int t = t0 + tid;
    const int c = t < T2 ? tst[t] >> 16 : 0;
    int tot;
    const int ex = block_scan_excl(c, scan_ws, tot);
    if (t < T2) { S[1 + t] = run + ex; tst[t] = run + ex; }
    run += tot;
  }
  if (tid == 0) { S[0] = T2; S[1 + T2] = B; }
  __syncthreads();
  for (int r = warp; r < nrec; r += 32) {
    const int sm = rec_sm[r];
    if (lane < (sm >> 8)) S[T2 + 2 + tst[rec_t[r]] + (sm & 255) + lane] = order[rec_src[r] + lane];
  }
}

// --------------------------------------------------------------------------------------------
// Layer variants of the stack kernel, fixed at compile time (lnb_sage_stack_forward):
//   STACK_PLAIN      out = act(E + V Z + b)                          (LanczosNet, GCN, ...)
//   STACK_SAGE_MEAN  then every finished row divided by (||row||_2 + eps) (model/graph_sage.py:150-153)
//   STACK_SAGE_MAX   the same, and the edge producer takes the elementwise max over the ELL row
//                    instead of the weighted sum (the Max aggregator, model/graph_sage.py:141-142)
constexpr int STACK_PLAIN = 0;
constexpr int STACK_SAGE_MEAN = 1;
constexpr int STACK_SAGE_MAX = 2;
constexpr float SAGE_EPS = 1.1920928955078125e-07f;   // np.finfo(np.float32).eps (graph_sage.py:6)

template <int kVariant>
struct SpectralPolicyT {
  static constexpr bool kNormRows = kVariant != STACK_PLAIN;
  static constexpr bool kMaxAgg = kVariant == STACK_SAGE_MAX;
  static constexpr bool kLongScales = kVariant == STACK_PLAIN;    // GraphSAGE runs S = 0: no step 0
  static constexpr int kStagesB = 2;      // k-block i + 1 is produced and its W tile loaded during MMA i
  static constexpr int kStagesA = 2;      // 64 KB: also holds Z (Ztot <= 128 rows x H <= 128) in one pass
  // Two producer warpgroups take alternate k-blocks: producing a k-block (an ELL gather or U, then
  // the hi / lo split) takes one group about as long as the MMAs that consume it
  static constexpr int kProducerGroups = 2;
  struct Params {
    const float* X;         // [B, N, Din0] input state, or nullptr with node_ids/emb (embedding)
    const int64_t* node_ids;// [B, N]
    const float* emb;       // [emb_rows, Din0]
    const float* Q;         // [B, N, K]
    const float* coeff;     // layer l: coeff + l * coeff_stride -> [B, K, S]
    int64_t coeff_stride;
    const float* ell_val;   // [B, E1, N, N]
    const uint8_t* ell_idx; // [B, E1, N, N]
    const int32_t* ell_max; // [B, E1]
    const int32_t* gext;    // [B, 2]
    const int32_t* tiles;   // next-fit table [B + 2], then (B >= 2) the schedule the kernel runs
    const float* bias;     // layer l: bias + l * H (may be null)
    float* out;             // [B, N, H] final state (may be null when the readout is fused)
    // fused readout (model/lanczos_net.py:185-194); score == nullptr disables it
    const float* W_out;     // [P, H]
    const float* b_out;     // [P]
    const float* w_att;     // [H]
    const float* b_att;     // [1]
    const uint8_t* mask;    // [B, N] or null (mean over all N nodes)
    float* score;           // [B, P]
    int P, emb_rows;
    int L;                  // number of layers in this launch
    int Din[LNB_CONV_MAX_LAYERS];          // input width of each layer (Din[l>0] == H)
    int B, N, E1, K, S, H, relu;
    int LB;                 // ELL lines (channel, t) that fit in shared memory
    int write_pad;          // also write the constant rows of padded nodes of `out`
    int dbg;                // debug experiment flags (LNB_DBG), 0 in production
  };
  // tile schedule (tile_assign_kernel): [T', first slot of tile 0 .. T', graph ids]; with B <= 1 there is
  // no room for it and the next-fit table [T, first graph of tile 0 .. T] is run in graph order
  static __device__ __forceinline__ const int32_t* schedule(const Params& p) {
    return p.B >= 2 ? p.tiles + p.B + 2 : p.tiles;
  }
  // sub = layer * 2 + step  (step 0: Z accumulation, step 1: edge accumulation + epilogue)
  static __device__ __forceinline__ int num_steps(const Params& p, int cta, int ncta) {
    const int T = __ldg(schedule(p));
    const int mine = T > cta ? (T - cta + ncta - 1) / ncta : 0;
    return (p.S > 0 ? 2 : 1) * p.L * mine;
  }
  static __device__ __forceinline__ void decode(const Params& p, int cta, int ncta, int it,
                                                int& m_tile, int& sub) {
    const int per = (p.S > 0 ? 2 : 1) * p.L;
    const int rem = it % per;
    m_tile = cta + (it / per) * ncta;
    sub = p.S > 0 ? rem : rem * 2 + 1;
  }
  static __device__ __forceinline__ int num_kblocks(const Params& p, int sub) {
    return ((sub & 1) == 0 ? p.S : p.E1) * p.Din[sub >> 1] / tcg::BK;
  }
  // Step 0's k-block kb is (d-block dblk, scale s), W columns s * Din + 32 dblk.  The d-blocks run in
  // pairs, the k-blocks of a pair alternating between its two d-blocks (kb = 2 (pair S + s) + dblk % 2).
  // The producer groups take alternate k-blocks, so each group takes every k-block of one d-block of
  // the pair and computes that d-block's U once, at s = 0 (d-block-major order, kb = dblk S + s, has both
  // groups compute every U).  An odd last d-block runs on its own (kb = pairs 2 S + s), alternating
  // between the groups, each computing U at its first k-block of it (s < 2).  first: this k-block is
  // where the group that takes it computes U.
  static __device__ __forceinline__ void s0_kblock(int Din, int S, int kb, int& dblk, int& s, bool& first) {
    const int paired = (Din / tcg::BK) & ~1;       // d-blocks that run in pairs
    if (kb < paired * S) {
      const int pr = kb / (2 * S), r = kb - pr * 2 * S;
      s = r >> 1;
      dblk = 2 * pr + (r & 1);
      first = s == 0;
    } else {
      s = kb - paired * S;
      dblk = paired;
      first = s < kProducerGroups;
    }
  }
  static __device__ __forceinline__ void w_coords(const Params& p, int sub, int kb, int& col0, int& row0) {
    const int Din = p.Din[sub >> 1];
    if (kLongScales && (sub & 1) == 0) {          // (the GraphSAGE variants run S = 0: no step 0)
      int dblk, s;
      bool first;
      s0_kblock(Din, p.S, kb, dblk, s, first);
      col0 = s * Din + dblk * tcg::BK;
    } else {
      col0 = p.S * Din + kb * tcg::BK;
    }
    row0 = (sub >> 1) * p.H;
  }
  // Z of step 0 stays in the A ring for the edge step's acc_init()
  static __device__ __forceinline__ bool drain_kept(const Params&, int sub) { return kLongScales && (sub & 1) == 0; }
  // row pitch (floats) of the X rows in shared memory
  static __host__ __device__ __forceinline__ int x_pitch(int Din0, int H) { return (Din0 > H ? Din0 : H) + 4; }

  // Row tables of the tile being run.  Node rows: graph after graph, n_eff rows each; Ritz rows
  // (Z): graph after graph, k_eff rows each (unpadded); quads: groups of 4 rows of one graph.
  struct Tables {
    int ng, Rtot, Ztot, nquads, nzquads, nlines;
    int gid[GMAX];                                  // graph ids of the tile's graphs
    int nbase[GMAX + 1], kbase[GMAX + 1], gn[GMAX], gk[GMAX];
    int cnt_e[LNB_MAX_E1], base_e[LNB_MAX_E1], tmax_e[LNB_MAX_E1];
    uint8_t emax[GMAX][LNB_MAX_E1];
    uint8_t row_g[RMAX], row_n[RMAX], z_g[RMAX], z_k[RMAX];
    uint8_t q_g[RMAX / 4 + GMAX], q_n0[RMAX / 4 + GMAX];     // node-row quads
    uint8_t zq_g[RMAX / 4 + GMAX], zq_k0[RMAX / 4 + GMAX];   // Ritz-row quads
    uint8_t line_e[256], line_t[256];
  };

  const Params& p;
  const int tid, r;
  const int N, K, S, E1, H, XP;           // hot parameters in registers
  int Din;                                // input width of the current layer
  // Shared memory, in this order (acc_init() finds Tables and Qs the same way)
  Tables* tb;
  float* Xs;                // X rows [RMAX][XP]; the finished output rows are the next layer's X
  float* Qs;                // [RMAX][K]
  float* Ev;                // [LB][RMAX] staged ELL values
  uint8_t* Ei;              // [LB][RMAX] staged ELL columns as tile-local row indices
  const float* frow;        // this (graph, k) row's filter coefficients f[k, 0..S) of the layer
  float* ring;              // the skeleton's A ring: the fused readout's scratch
  tcg::PhaseTimer* ptm = nullptr;   // profiling aid: the current step's timer

  static __host__ __device__ constexpr size_t tables_bytes() { return (sizeof(Tables) + 15) & ~size_t(15); }

  __device__ SpectralPolicyT(const Params& p_, uint8_t* smem, int tid_)
      : p(p_), tid(tid_), r(tid_ & 127), N(p_.N), K(p_.K), S(p_.S), E1(p_.E1),
        H(p_.H), XP(x_pitch(p_.Din[0], p_.H)), Din(p_.Din[0]) {
    tb = reinterpret_cast<Tables*>(smem);
    Xs = reinterpret_cast<float*>(smem + tables_bytes());
    Qs = Xs + (size_t)RMAX * XP;
    Ev = Qs + (size_t)RMAX * K;
    Ei = reinterpret_cast<uint8_t*>(Ev + (size_t)p.LB * RMAX);
    ring = reinterpret_cast<float*>(tcg::a_ring(smem, kStagesB, kStagesA));
  }
  static size_t smem_fixed(int Din, int K, int H) {
    return (size_t)RMAX * x_pitch(Din, H) * 4 + (size_t)RMAX * K * 4 + tables_bytes() + 16;
  }
  static size_t ell_line_bytes() { return (size_t)RMAX * 5; }
  // scratch of readout(), laid out from the start of the A ring: Wr, Yr, cx and the node masks of
  // up to GMAX graphs
  static size_t readout_bytes(int H, int P, int N) {
    const size_t P1 = (size_t)P + 1, PQ = (P1 + 3) / 4, yr = (RMAX + 1) * P1;
    return (4 * PQ * (H + 4) + yr + ((4 - (yr & 3)) & 3) + H) * 4 + (size_t)GMAX * N;
  }

  // ------------------------------------------------------------------------------------------
  __device__ void build_tables(int m_tile) {
    // executed by warp 0: lane j <-> j-th graph of the tile
    const int lane = tid & 31;
    const int32_t* sc = schedule(p);
    const int s0 = __ldg(sc + 1 + m_tile), s1 = __ldg(sc + 2 + m_tile);
    const int ng = s1 - s0;
    int g = s0 + lane, n = 0, k = 0;
    if (lane < ng) {
      if (p.B >= 2) g = __ldg(sc + __ldg(sc) + 2 + s0 + lane);
      n = __ldg(p.gext + g * 2);
      k = __ldg(p.gext + g * 2 + 1);
    }
    const int nq = (n + 3) >> 2, kq = (k + 3) >> 2;
    int pn = n, pk = k, pq = nq, pz = kq;              // inclusive prefix sums
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, pn, o), bq = __shfl_up_sync(0xffffffffu, pk, o);
      const int c = __shfl_up_sync(0xffffffffu, pq, o), d = __shfl_up_sync(0xffffffffu, pz, o);
      if (lane >= o) { pn += a; pk += bq; pq += c; pz += d; }
    }
    const int nb = pn - n, kb = pk - k, qb = pq - nq, zb = pz - kq;
    if (lane < ng) {
      tb->gid[lane] = g;
      tb->nbase[lane] = nb; tb->kbase[lane] = kb; tb->gn[lane] = n; tb->gk[lane] = k;
      for (int i = 0; i < n; ++i) { tb->row_g[nb + i] = (uint8_t)lane; tb->row_n[nb + i] = (uint8_t)i; }
      for (int i = 0; i < k; ++i) { tb->z_g[kb + i] = (uint8_t)lane; tb->z_k[kb + i] = (uint8_t)i; }
      for (int i = 0; i < nq; ++i) { tb->q_g[qb + i] = (uint8_t)lane; tb->q_n0[qb + i] = (uint8_t)(4 * i); }
      for (int i = 0; i < kq; ++i) { tb->zq_g[zb + i] = (uint8_t)lane; tb->zq_k0[zb + i] = (uint8_t)(4 * i); }
    }
    const int Rtot = __shfl_sync(0xffffffffu, pn, 31), Ztot = __shfl_sync(0xffffffffu, pk, 31);
    const int nquads = __shfl_sync(0xffffffffu, pq, 31), nzquads = __shfl_sync(0xffffffffu, pz, 31);
    // per-channel maximum row length over the tile's graphs, per-graph row lengths
    // (all loads issued before the first reduction: one global round trip instead of E1)
    int em[LNB_MAX_E1];
#pragma unroll
    for (int e = 0; e < LNB_MAX_E1; ++e)
      em[e] = (e < E1 && lane < ng) ? __ldg(p.ell_max + g * E1 + e) : 0;
#pragma unroll
    for (int e = 0; e < LNB_MAX_E1; ++e) {
      if (e < E1) {
        int m = em[e];
        if (lane < ng) tb->emax[lane][e] = (uint8_t)m;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) tb->tmax_e[e] = m;
      }
    }
    __syncwarp();
    if (lane == 0) {
      tb->ng = ng; tb->Rtot = Rtot; tb->Ztot = Ztot; tb->nquads = nquads; tb->nzquads = nzquads;
      tb->nbase[ng] = Rtot; tb->kbase[ng] = Ztot;
      int left = p.LB, base = 0;
      for (int e = 0; e < E1; ++e) {            // staged lines per channel, in channel order
        const int c = min(tb->tmax_e[e], left);
        tb->cnt_e[e] = c; tb->base_e[e] = base;
        for (int t = 0; t < c; ++t) { tb->line_e[base + t] = (uint8_t)e; tb->line_t[base + t] = (uint8_t)t; }
        base += c; left -= c;
      }
      tb->nlines = base;
    }
  }

  __device__ void step_begin(int m_tile, int sub, int /*kb_first*/, tcg::PhaseTimer& tm) {
    tcg::producers_sync<SpectralPolicyT>();              // previous step's smem readers / writers are done
    const int layer = sub >> 1, step = sub & 1;
    if (step == 1 && S > 0) return;     // tile state was staged by step 0 of this layer
    Din = p.Din[layer];
    const int warp = tid >> 5, lane = tid & 31;
    constexpr int NW = tcg::producer_threads<SpectralPolicyT> / 32;
    const int dv = Din / 4;
    ptm = &tm;
    if (layer == 0) {
    if (warp == 0) build_tables(m_tile);
    tcg::producers_sync<SpectralPolicyT>();
    tm.lap(16);
    const int Rtot = tb->Rtot;
    // ---- phase A: asynchronous copies of the real rows of X and Q (one warp per row) --------
    int64_t my_id = 0;                           // lane j: embedding id of this warp's j-th row
    if (!p.X && warp + lane * NW < Rtot) {
      const int row = warp + lane * NW;
      my_id = __ldg(p.node_ids + (int64_t)tb->gid[tb->row_g[row]] * N + tb->row_n[row]);
    }
    for (int row = warp, j = 0; row < Rtot; row += NW, ++j) {
      const int64_t src_row = (int64_t)tb->gid[tb->row_g[row]] * N + tb->row_n[row];
      const float* xsrc;
      if (p.X) {
        xsrc = p.X + src_row * Din;
      } else {                                  // embedding rows (model/lanczos_net.py:154)
        int64_t id = __shfl_sync(0xffffffffu, my_id, j);
        id = id < 0 ? 0 : (id >= p.emb_rows ? p.emb_rows - 1 : id);
        xsrc = p.emb + id * Din;
      }
      float* xd = Xs + (size_t)row * XP;
      for (int q4 = lane; q4 < dv; q4 += 32) sm90::cp_async_16(xd + 4 * q4, xsrc + 4 * q4);
      const float* qsrc = p.Q + src_row * K;            // K % 4 == 0: 16-byte pieces
      float* qd = Qs + (size_t)row * K;
      for (int k4 = lane; k4 < (K >> 2); k4 += 32) sm90::cp_async_16(qd + 4 * k4, qsrc + 4 * k4);
    }
    tm.lap(17);
    // ---- staged ELL lines: line l <-> (channel e, entry t); a warp per line, batched loads ---
    {
      constexpr int ELL_BATCH = 4;
      const int nlines = tb->nlines;
      for (int base = warp; base < nlines; base += NW * ELL_BATCH) {
        for (int r0 = 0; r0 < Rtot; r0 += 32) {
          const int rr = r0 + lane;
          float vv[ELL_BATCH];
          int ii[ELL_BATCH];
#pragma unroll
          for (int u = 0; u < ELL_BATCH; ++u) {
            const int line = base + u * NW;
            vv[u] = 0.f; ii[u] = 0;
            if (line < nlines && rr < Rtot) {
              const int e = tb->line_e[line], t = tb->line_t[line];
              const int g = tb->row_g[rr], n = tb->row_n[rr];
              if (t < tb->emax[g][e]) {
                const int64_t off = (((int64_t)tb->gid[g] * E1 + e) * N + t) * N + n;
                vv[u] = __ldg(p.ell_val + off);
                ii[u] = tb->nbase[g] + __ldg(p.ell_idx + off);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < ELL_BATCH; ++u) {
            const int line = base + u * NW;
            if (line < nlines && rr < Rtot) {
              Ev[(size_t)line * RMAX + rr] = vv[u];
              Ei[(size_t)line * RMAX + rr] = (uint8_t)ii[u];
            }
          }
        }
      }
    }
    tm.lap(18);
    }  // layer == 0: tile state staged once, reused by every layer
    const int Ztot = tb->Ztot;
    // this thread's (graph, k) row of this layer's filter coefficients (read once per k-block, from L1)
    frow = p.coeff;                     // a valid address for the rows past Ztot as well
    if (S > 0 && r < Ztot)
      frow = p.coeff + layer * p.coeff_stride + ((int64_t)tb->gid[tb->z_g[r]] * K + tb->z_k[r]) * S;
    tm.lap(0);
    sm90::cp_async_wait_all();
    tcg::producers_sync<SpectralPolicyT>();
    tm.lap(1);
  }

  // The A row of k-block kb is scale * v (the skeleton multiplies while it splits), so that step 0
  // keeps only U in registers across the k-blocks of a d-block
  __device__ __forceinline__ float produce(int sub, int kb, float (&v)[32]) {
    if (kLongScales && (sub & 1) == 0) {
      // row = (graph, Ritz index): f[k, s] * U[row, d0:d0+32], (dblk, s) from s0_kblock; v holds U
      // (zero for the rows past Ztot, whose scale is 0)
      int dblk, s;
      bool first;
      s0_kblock(Din, S, kb, dblk, s, first);
      const float f = __ldg(frow + s);             // issued before U is summed
      if (first) {
        // U[(g, k), d0:d0+32] = sum_n Q_g[n, k] X_g[n, d0:d0+32]: every thread of graph g reads the
        // same X row (a broadcast), consecutive Q entries.  Computed once per d-block of a pair (by
        // the group that takes it), twice for an odd last d-block (each group for itself).
#pragma unroll
        for (int j = 0; j < tcg::BK; ++j) v[j] = 0.f;
        if (r < tb->Ztot) {
          const int g = tb->z_g[r], n_g = tb->gn[g], nb = tb->nbase[g];
          const float* xs = Xs + (size_t)nb * XP + dblk * tcg::BK;
          const float* qs = Qs + (size_t)nb * K + tb->z_k[r];
#pragma unroll 2
          for (int n = 0; n < n_g; ++n) {
            const float q = qs[(size_t)n * K];
            const float4* x4 = reinterpret_cast<const float4*>(xs + (size_t)n * XP);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 t = x4[j];
              v[4 * j + 0] = fmaf(q, t.x, v[4 * j + 0]); v[4 * j + 1] = fmaf(q, t.y, v[4 * j + 1]);
              v[4 * j + 2] = fmaf(q, t.z, v[4 * j + 2]); v[4 * j + 3] = fmaf(q, t.w, v[4 * j + 3]);
            }
          }
        }
      }
      return r < tb->Ztot ? f : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    const int j0 = kb * tcg::BK;
    const int c = j0 / Din, d0 = j0 - c * Din;
    // edge type e = c: sparse row of L_e (ELL) times X[:, d0:d0+32]; row = (graph, node)
    if (r >= tb->Rtot) return 1.f;
    const int e = c;
    if constexpr (kMaxAgg) {
      produce_max(e, d0, v);
      return 1.f;
    }
    const float* xs = Xs + d0;
    const int ts = tb->cnt_e[e], tmax = tb->tmax_e[e];
    const float* ev = Ev + (size_t)tb->base_e[e] * RMAX + r;
    const uint8_t* ei = Ei + (size_t)tb->base_e[e] * RMAX + r;
#pragma unroll 2
    for (int t = 0; t < ts; ++t) {
      const float a = ev[t * RMAX];
      if (a == 0.f) continue;                        // zero fill up to the tile's longest row
      const int i = ei[t * RMAX];
      const float4* x4 = reinterpret_cast<const float4*>(xs + (size_t)i * XP);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 tt = x4[q];
        v[4 * q + 0] = fmaf(a, tt.x, v[4 * q + 0]);
        v[4 * q + 1] = fmaf(a, tt.y, v[4 * q + 1]);
        v[4 * q + 2] = fmaf(a, tt.z, v[4 * q + 2]);
        v[4 * q + 3] = fmaf(a, tt.w, v[4 * q + 3]);
      }
    }
    if (ts < tmax) {                               // lines that did not fit the staging budget
      const int g = tb->row_g[r], n = tb->row_n[r];
      const int my = tb->emax[g][e], nb = tb->nbase[g];
      const int64_t off0 = (((int64_t)tb->gid[g] * E1 + e) * N) * N + n;
      for (int t = ts; t < tmax; ++t) {
        float a = 0.f;
        int i = 0;
        if (t < my) {
          a = __ldg(p.ell_val + off0 + (int64_t)t * N);
          i = nb + __ldg(p.ell_idx + off0 + (int64_t)t * N);
        }
        if (a == 0.f) continue;
        const float4* x4 = reinterpret_cast<const float4*>(xs + (size_t)i * XP);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 tt = x4[q];
          v[4 * q + 0] = fmaf(a, tt.x, v[4 * q + 0]);
          v[4 * q + 1] = fmaf(a, tt.y, v[4 * q + 1]);
          v[4 * q + 2] = fmaf(a, tt.z, v[4 * q + 2]);
          v[4 * q + 3] = fmaf(a, tt.w, v[4 * q + 3]);
        }
      }
    }
    return 1.f;
  }

  // Max aggregator (STACK_SAGE_MAX): v = elementwise max over X[i, d0:d0+32] for the entries i of
  // row r of channel e.  The entry values (sample counts / K) are ignored: a non-zero only says the
  // neighbour was drawn; zero entries are the fill up to the tile's longest row.  A row without
  // entries (nonempty = 0) gives 0, like the reference's `agg * nonempty_mask`.
  __device__ __forceinline__ void produce_max(int e, int d0, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = -INFINITY;
    bool any = false;
    const float* xs = Xs + d0;
    const int ts = tb->cnt_e[e], tmax = tb->tmax_e[e];
    const float* ev = Ev + (size_t)tb->base_e[e] * RMAX + r;
    const uint8_t* ei = Ei + (size_t)tb->base_e[e] * RMAX + r;
    for (int t = 0; t < ts; ++t) {
      if (ev[t * RMAX] == 0.f) continue;
      const float4* x4 = reinterpret_cast<const float4*>(xs + (size_t)ei[t * RMAX] * XP);
      any = true;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 tt = x4[q];
        v[4 * q + 0] = fmaxf(v[4 * q + 0], tt.x);
        v[4 * q + 1] = fmaxf(v[4 * q + 1], tt.y);
        v[4 * q + 2] = fmaxf(v[4 * q + 2], tt.z);
        v[4 * q + 3] = fmaxf(v[4 * q + 3], tt.w);
      }
    }
    if (ts < tmax) {                               // lines that did not fit the staging budget
      const int g = tb->row_g[r], n = tb->row_n[r];
      const int my = tb->emax[g][e], nb = tb->nbase[g];
      const int64_t off0 = (((int64_t)tb->gid[g] * E1 + e) * N) * N + n;
      for (int t = ts; t < tmax && t < my; ++t) {
        if (__ldg(p.ell_val + off0 + (int64_t)t * N) == 0.f) continue;
        const int i = nb + __ldg(p.ell_idx + off0 + (int64_t)t * N);
        const float4* x4 = reinterpret_cast<const float4*>(xs + (size_t)i * XP);
        any = true;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 tt = x4[q];
          v[4 * q + 0] = fmaxf(v[4 * q + 0], tt.x);
          v[4 * q + 1] = fmaxf(v[4 * q + 1], tt.y);
          v[4 * q + 2] = fmaxf(v[4 * q + 2], tt.z);
          v[4 * q + 3] = fmaxf(v[4 * q + 3], tt.w);
        }
      }
    }
    if (!any) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.f;
    }
  }

  // GraphSAGE row normalisation (model/graph_sage.py:152): y / (||y||_2 + eps), a division like the
  // reference.  The squares are summed in feature order, so a row equal to act(b) gets exactly the
  // denominator of pad_den() below.
  __device__ __forceinline__ void normalize_row(float* row) const {
    float4* r4 = reinterpret_cast<float4*>(row);
    float ss = 0.f;
    for (int h4 = 0; h4 < H / 4; ++h4) {
      const float4 t = r4[h4];
      ss = fmaf(t.x, t.x, ss); ss = fmaf(t.y, t.y, ss); ss = fmaf(t.z, t.z, ss); ss = fmaf(t.w, t.w, ss);
    }
    const float den = sqrtf(ss) + SAGE_EPS;
    for (int h4 = 0; h4 < H / 4; ++h4) {
      const float4 t = r4[h4];
      r4[h4] = make_float4(t.x / den, t.y / den, t.z / den, t.w / den);
    }
  }
  // denominator of the constant row act(b) of padded nodes (every calling thread computes it alone)
  __device__ __forceinline__ float pad_den(const float* bias) const {
    float ss = 0.f;
    for (int h = 0; h < H; ++h) {
      float t = bias ? __ldg(bias + h) : 0.f;
      t = (p.relu != 0) ? fmaxf(t, 0.f) : t;
      ss = fmaf(t, t, ss);
    }
    return sqrtf(ss) + SAGE_EPS;
  }

  // The edge step's store() overwrites rows of X that other producers may still be reading.
  __device__ void pre_epilogue(int sub) {
    if ((sub & 1) == 0) return;
    tcg::producers_sync<SpectralPolicyT>();              // every producer is done reading X
    if (ptm) ptm->lap(22);              // (profiling) wait for the slowest producer group
  }

  // Consumers, before the first MMA of an edge step: D_main = (V Z) for the rows of this thread's
  // fragment (Z of the layer, left in the A ring by step 0's drain: row (graph, k), swizzled like
  // any drain pass), D_corr = 0.  Reads the tile's Tables and Qs, which the producers staged
  // before they produced step 0.
  static __device__ __forceinline__ bool acc_init(const Params& p, const uint8_t* smem, const float* zr,
                                                  int sub, int row0, int cl, float (&d)[128]) {
    if (!kLongScales || (sub & 1) == 0 || p.S == 0) return false;
    const Tables* tb = reinterpret_cast<const Tables*>(smem);
    const int K = p.K;
    const float* Qs = reinterpret_cast<const float*>(smem + tables_bytes()) + (size_t)RMAX * x_pitch(p.Din[0], p.H);
    const int Rtot = tb->Rtot;
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (row >= Rtot) continue;
      const int g = tb->row_g[row], k_g = tb->gk[g], zb = tb->kbase[g];
      const float* q = Qs + (size_t)row * K;
      // Ritz index order, like the reference's V (Z): rows past k_eff belong to the next graph
      for (int k = 0; k < k_g; ++k) {
        const float a = q[k];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 t = *reinterpret_cast<const float2*>(zr + tcg::stg_index(zb + k, 8 * j + cl, tcg::BN));
          d[4 * j + 2 * h] = fmaf(a, t.x, d[4 * j + 2 * h]);
          d[4 * j + 2 * h + 1] = fmaf(a, t.y, d[4 * j + 2 * h + 1]);
        }
      }
    }
    return true;
  }

  // Edge steps only (step 0's drain is kept).  Rows of Xs are XP = max(Din0, H) + 4 floats long,
  // which a 16-column chunk can overrun when H % 16 != 0: only the float4 pieces below column H are
  // written (H % 4 == 0, so a piece is either wholly inside the row or wholly outside it).
  __device__ __forceinline__ void store(int sub, int col, float (&x)[tcg::EW]) {
    if (col >= H || r >= tb->Rtot) return;
    float4* o4 = reinterpret_cast<float4*>(Xs + (size_t)r * XP + col);
    const bool relu = p.relu != 0;
    const float* bias = p.bias ? p.bias + (sub >> 1) * H : nullptr;
#pragma unroll
    for (int q = 0; q < tcg::EW / 4; ++q) {
      if (col + 4 * q >= H) break;
      float y[4] = {x[4 * q + 0], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]};
      if (bias) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + col) + q);
        y[0] += b4.x; y[1] += b4.y; y[2] += b4.z; y[3] += b4.w;
      }
      if (relu) { y[0] = fmaxf(y[0], 0.f); y[1] = fmaxf(y[1], 0.f); y[2] = fmaxf(y[2], 0.f); y[3] = fmaxf(y[3], 0.f); }
      o4[q] = make_float4(y[0], y[1], y[2], y[3]);   // finished row chunk = next layer's X row
    }
  }

  // After the last layer: coalesced write-back of the final state (real rows from shared
  // memory, one warp per 512-byte row, plus the constant rows act(b) of padded nodes when
  // requested) and / or the fused readout.  Between layers the state never leaves the SM.
  __device__ void post_epilogue(int sub) {
    if constexpr (kNormRows) {
      // every chunk of every row is stored (the skeleton's producers_sync); thread r of the first
      // group normalises row r, and the next reader of other rows (next layer's producers, the
      // write-back and readout below) is behind another producers_sync()
      if ((sub & 1) != 0 && tid < tcg::BM && r < tb->Rtot) normalize_row(Xs + (size_t)r * XP);
    }
    if ((sub & 1) == 0 || (sub >> 1) != p.L - 1) return;
    tcg::producers_sync<SpectralPolicyT>();              // every chunk of every row is in shared memory
    if (ptm) ptm->lap(19);
    const int warp = tid >> 5, lane = tid & 31;
    constexpr int NW = tcg::producer_threads<SpectralPolicyT> / 32;
    const int hv = H / 4, Rtot = tb->Rtot;
    const float* bias = p.bias ? p.bias + (p.L - 1) * H : nullptr;
    if (p.out) {
      for (int row = warp; row < Rtot; row += NW) {
        const float4* src = reinterpret_cast<const float4*>(Xs + (size_t)row * XP);
        float4* dst = reinterpret_cast<float4*>(
            p.out + ((int64_t)tb->gid[tb->row_g[row]] * N + tb->row_n[row]) * H);
        for (int q4 = lane; q4 < hv; q4 += 32) dst[q4] = src[q4];
      }
      if (p.write_pad) {
        [[maybe_unused]] float den = 1.f;
        if constexpr (kNormRows) den = pad_den(bias);
        const int npad = tb->ng * N - Rtot;
        for (int i = warp; i < npad; i += NW) {
          // i-th padded (graph, node) pair of the tile, found by walking the per-graph pad counts
          int g = 0, rem = i;
          while (rem >= N - tb->gn[g]) { rem -= N - tb->gn[g]; ++g; }
          float4* dst = reinterpret_cast<float4*>(p.out + ((int64_t)tb->gid[g] * N + tb->gn[g] + rem) * H);
          for (int q4 = lane; q4 < hv; q4 += 32) {
            float y[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float t = bias ? __ldg(bias + 4 * q4 + u) : 0.f;
              y[u] = (p.relu != 0) ? fmaxf(t, 0.f) : t;
              if constexpr (kNormRows) y[u] = y[u] / den;
            }
            dst[q4] = make_float4(y[0], y[1], y[2], y[3]);
          }
        }
      }
    }
    if (p.score) readout(bias);
  }

  // Fused readout (model/lanczos_net.py:185-194): y = (W_out x + b_out) * sigmoid(w_att.x + b_att)
  // per node, masked mean over the nodes of each graph.  Rows of padded nodes are the constant
  // act(b_last); they count only where the mask says so (or when there is no mask).
  __device__ void readout(const float* bias_last) {
    const int P = p.P, P1 = p.P + 1, PQ = (P1 + 3) >> 2, HP = H + 4;
    float* Wr = ring;                                // [4 PQ][HP]  W_out rows, w_att, zero rows (the ring is idle)
    float* Yr = Wr + (size_t)4 * PQ * HP;            // [RMAX + 1][P1]  per-row outputs; last = pad row
    float* cx = Yr + (size_t)(RMAX + 1) * P1 + ((4 - ((RMAX + 1) * P1 & 3)) & 3);   // [H], 16 B aligned
    for (int e = tid; e < 4 * PQ * H; e += tcg::producer_threads<SpectralPolicyT>) {
      const int o = e / H, h = e - o * H;
      Wr[o * HP + h] = (o < P) ? __ldg(p.W_out + o * H + h) : (o == P ? __ldg(p.w_att + h) : 0.f);
    }
    [[maybe_unused]] float den = 1.f;
    if constexpr (kNormRows) den = pad_den(bias_last);
    for (int h = tid; h < H; h += tcg::producer_threads<SpectralPolicyT>) {
      float t = bias_last ? __ldg(bias_last + h) : 0.f;
      cx[h] = (p.relu != 0) ? fmaxf(t, 0.f) : t;
      if constexpr (kNormRows) cx[h] = cx[h] / den;
    }
    uint8_t* mk = reinterpret_cast<uint8_t*>(cx + H);   // [ng][N] node masks of the tile's graphs
    for (int e = tid; e < tb->ng * N; e += tcg::producer_threads<SpectralPolicyT>) {
      const int g = e / N;
      mk[e] = p.mask ? __ldg(p.mask + (int64_t)tb->gid[g] * N + (e - g * N)) : (uint8_t)1;
    }
    tcg::producers_sync<SpectralPolicyT>();
    if (ptm) ptm->lap(20);
    const int Rtot = tb->Rtot;
    // warp <-> (block of 32 rows, half of the outputs): lane = row, so the row loads are
    // conflict-free and every weight load is one broadcast wavefront
    {
      const int warp = tid >> 5, lane = tid & 31;
      const int rb = warp & 3, og = warp >> 2;
      const int per = (P1 + kProducerGroups - 1) / kProducerGroups;
      const int o_end = min(P1, (og + 1) * per);
      const int row = rb * 32 + lane;
      const float4* x4 = reinterpret_cast<const float4*>(Xs + (size_t)(row < Rtot ? row : 0) * XP);
      for (int o0 = og * per; o0 < o_end; o0 += 6) {
        const int cnt = min(6, o_end - o0);
        const float4* w4 = reinterpret_cast<const float4*>(Wr + (size_t)o0 * HP);
        float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int h4 = 0; h4 < H / 4; ++h4) {
          const float4 x = x4[h4];
#pragma unroll
          for (int j = 0; j < 6; ++j) {
            if (j < cnt) {
              const float4 wv = w4[j * (HP / 4) + h4];
              acc[j] = fmaf(x.x, wv.x, acc[j]); acc[j] = fmaf(x.y, wv.y, acc[j]);
              acc[j] = fmaf(x.z, wv.z, acc[j]); acc[j] = fmaf(x.w, wv.w, acc[j]);
            }
          }
        }
        if (row < Rtot) {
#pragma unroll
          for (int j = 0; j < 6; ++j)
            if (j < cnt) {
              const int o = o0 + j;
              const float v = acc[j] + ((o < P) ? __ldg(p.b_out + o) : __ldg(p.b_att));
              Yr[row * P1 + o] = (o < P) ? v : 1.f / (1.f + expf(-v));     // column P: the gate
            }
        }
      }
      // the constant padded-node row: one warp per output, lanes stride the H features
      for (int o = warp; o < P1; o += tcg::producer_threads<SpectralPolicyT> / 32) {
        float acc = 0.f;
        for (int h = lane; h < H; h += 32) acc = fmaf(cx[h], Wr[o * HP + h], acc);
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
        if (lane == 0) {
          const float v = acc + ((o < P) ? __ldg(p.b_out + o) : __ldg(p.b_att));
          Yr[RMAX * P1 + o] = (o < P) ? v : 1.f / (1.f + expf(-v));
        }
      }
    }
    tcg::producers_sync<SpectralPolicyT>();
    if (ptm) ptm->lap(21);
    for (int e = tid; e < tb->ng * P; e += tcg::producer_threads<SpectralPolicyT>) {
      const int g = e / P, o = e - g * P;
      const int nb = tb->nbase[g], n_g = tb->gn[g];
      const uint8_t* m = mk + g * N;
      float acc = 0.f;
      int cnt = 0;
      for (int n = 0; n < N; ++n) {
        if (m[n] == 0) continue;
        const float* y = Yr + (n < n_g ? nb + n : RMAX) * P1;
        acc += y[P] * y[o];
        ++cnt;
      }
      p.score[(int64_t)tb->gid[g] * P + o] = acc / (float)cnt;
    }
  }
};
using SpectralPolicy = SpectralPolicyT<STACK_PLAIN>;

}  // namespace

namespace lnb {
// tile table, tile schedule and compact Ritz row list from the extents (shared by lnb_graph_prepare
// and lnb_graph_prepare_sparse); tiles = [4*B + 2] ints: B + 2 table entries followed by 3*B ints
// that hold the schedule (2*B + 2 at most; B >= 2) and serve as scratch before it
void launch_tile_assign(cudaStream_t s, const int32_t* gext, int B, int K, int32_t* tiles,
                        int32_t* rowmap, int32_t* nrows) {
  const size_t tbytes = ((size_t)6 * (B + 1) + 2 * SCH_NCLS) * sizeof(int32_t);
  const int tsm = tbytes <= 200 * 1024;
  if (tsm && tbytes > 40 * 1024)
    cudaFuncSetAttribute(tile_assign_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tbytes);
  if (tsm)
    tile_assign_kernel<true><<<1, 1024, tbytes, s>>>(gext, B, K, tiles, tiles + B + 2, rowmap, nrows);
  else
    tile_assign_kernel<false><<<1, 1024, 0, s>>>(gext, B, K, tiles, tiles + B + 2, rowmap, nrows);
}

int launch_tiles_or_rowmap(cudaStream_t s, int flags, const int32_t* gext, int B, int K,
                           int32_t* tiles, int32_t* rowmap, int32_t* nrows, const char* who) {
  if (flags & LNB_PREP_DEFER_TILES) {            // the caller runs lnb_tile_assign
    int rc = lnb::finish_launch(who);
    if (rc == LNB_OK && rowmap) rc = lnb_ritz_rowmap((lnb_stream_t)s, gext, B, K, rowmap, nrows);
    return rc;
  }
  launch_tile_assign(s, gext, B, K, tiles, rowmap, nrows);
  count_launch();
  return finish_launch(who);
}
}  // namespace lnb

extern "C" {

int lnb_graph_prepare(lnb_stream_t stream, const float* L, const float* Q, int B, int N, int E1,
                      int K, float* ell_val, uint8_t* ell_idx, int32_t* ell_max, int32_t* gext,
                      int32_t* tiles /* [4*B + 2]: B + 2 tile table followed by 3*B scratch */,
                      int32_t* rowmap, int32_t* nrows, int flags) {
  LNB_REQUIRE(L && Q && ell_val && ell_idx && ell_max && gext && tiles, "graph_prepare: null pointer");
  LNB_REQUIRE((rowmap == nullptr) == (nrows == nullptr), "graph_prepare: rowmap and nrows go together");
  LNB_REQUIRE(B >= 0 && N >= 1 && N <= LNB_MAX_N_ELL && E1 >= 1 && E1 <= LNB_MAX_E1 && K >= 1,
              "graph_prepare: bad dims B=%d N=%d E1=%d K=%d", B, N, E1, K);
  if (B == 0) return LNB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t lbytes = (size_t)N * N * E1 * sizeof(float);
  const int stage = lbytes <= 64 * 1024;
  if (stage) {
    if (lbytes > 40 * 1024)
      cudaFuncSetAttribute(graph_prepare_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbytes);
    graph_prepare_kernel<true><<<B, 256, lbytes, s>>>(L, Q, N, E1, K, ell_val, ell_idx, ell_max, gext,
                                                      flags & 1);
  } else {
    graph_prepare_kernel<false><<<B, 256, 0, s>>>(L, Q, N, E1, K, ell_val, ell_idx, ell_max, gext,
                                                  flags & 1);
  }
  lnb::count_launch(1);
  return lnb::launch_tiles_or_rowmap(s, flags, gext, B, K, tiles, rowmap, nrows, "graph_prepare");
}

int lnb_tile_assign(lnb_stream_t stream, const int32_t* gext, int B, int K, int32_t* tiles) {
  LNB_REQUIRE(gext && tiles, "tile_assign: null pointer");
  LNB_REQUIRE(B >= 0 && K >= 1, "tile_assign: bad dims B=%d K=%d", B, K);
  if (B == 0) return LNB_OK;
  lnb::launch_tile_assign((cudaStream_t)stream, gext, B, K, tiles, nullptr, nullptr);
  lnb::count_launch();
  return lnb::finish_launch("tile_assign");
}

// one launcher for every variant of the stack kernel
extern "C++" {
template <class Pol>
static int launch_stack(lnb_stream_t stream, const lnb_spectral_stack& d, const char* who) {
  LNB_REQUIRE((d.X || (d.node_ids && d.emb_table)) && d.Q && d.ell_val && d.ell_idx && d.ell_max &&
                  d.gext && d.tiles && d.W_hi && d.W_lo && (d.out_state || d.score) &&
                  (d.coeff || d.S == 0),
              "%s: null pointer", who);
  LNB_REQUIRE(d.B >= 0 && d.N >= 1 && d.E1 >= 1 && d.K >= 1 && d.S >= 0 && d.H >= 1 &&
                  d.num_layers >= 1 && d.num_layers <= LNB_CONV_MAX_LAYERS,
              "%s: bad dims", who);
  LNB_REQUIRE(!d.score || (d.W_out && d.b_out && d.w_att && d.b_att && d.P >= 1 && d.P <= 48),
              "%s: readout needs W_out, b_out, w_att, b_att and 1 <= P <= 48", who);
  int dmax = 0;
  bool ok = d.N <= LNB_MAX_N && d.K <= LNB_CONV_MAX_K && d.K % 4 == 0 && d.H % 4 == 0 && d.H <= LNB_MAX_WIDTH &&
            d.E1 <= LNB_MAX_E1;
  for (int l = 0; l < d.num_layers; ++l) {
    ok = ok && d.Din[l] % 32 == 0 && d.Din[l] >= 32 && (l == 0 || d.Din[l] == d.H);
    dmax = d.Din[l] > dmax ? d.Din[l] : dmax;
  }
  ok = ok && (d.S + d.E1) * dmax <= d.Kw;
  if (!ok) {
    lnb::set_err("%s: unsupported shape N=%d K=%d H=%d E1=%d (needs N<=128, Din%%32==0, inner "
                 "layers Din==H, K%%4==0, K<=%d, H%%4==0, H<=128, E1<=%d)", who, d.N, d.K, d.H, d.E1,
                 LNB_CONV_MAX_K, LNB_MAX_E1);
    return LNB_ERR_UNSUPPORTED;
  }
  if ((d.bias && (reinterpret_cast<uintptr_t>(d.bias) & 15)) || (reinterpret_cast<uintptr_t>(d.Q) & 15) ||
      (d.X && (reinterpret_cast<uintptr_t>(d.X) & 15)) || (d.emb_table && (reinterpret_cast<uintptr_t>(d.emb_table) & 15))) {
    lnb::set_err("%s: X / emb_table / Q / bias must be 16-byte aligned", who);
    return LNB_ERR_ARG;
  }
  if (d.B == 0) return LNB_OK;
  size_t smem = tcg::core_smem(Pol::kStagesB, Pol::kStagesA) + 1024 +
                Pol::smem_fixed(dmax, d.K, d.H);
  if (smem > lnb::SMEM_MAX) {
    lnb::set_err("%s: tile state (Din=%d, K=%d, H=%d) needs %zu B of shared memory", who, dmax, d.K,
                 d.H, smem);
    return LNB_ERR_UNSUPPORTED;
  }
  int lb = (int)((lnb::SMEM_MAX - smem) / Pol::ell_line_bytes());
  if (lb > 255) lb = 255;
  // The readout scratch (at most 56 KiB: P = 48, H = 128, N = 128) fits the A ring (64 KiB), which
  // is idle after the last drain, at every shape accepted above; the check keeps it that way.
  if (d.score && Pol::readout_bytes(d.H, d.P, d.N) > (size_t)Pol::kStagesA * tcg::STAGE_A_BYTES) {
    lnb::set_err("%s: fused readout (P=%d, H=%d, N=%d) does not fit the free shared memory", who, d.P,
                 d.H, d.N);
    return LNB_ERR_UNSUPPORTED;
  }
  smem += (size_t)lb * Pol::ell_line_bytes();
  typename Pol::Params p{};
  p.X = d.X; p.node_ids = d.node_ids; p.emb = d.emb_table; p.Q = d.Q;
  p.coeff = d.coeff; p.coeff_stride = d.coeff_layer_stride;
  p.ell_val = d.ell_val; p.ell_idx = d.ell_idx; p.ell_max = d.ell_max; p.gext = d.gext; p.tiles = d.tiles;
  p.bias = d.bias; p.out = d.out_state;
  p.W_out = d.W_out; p.b_out = d.b_out; p.w_att = d.w_att; p.b_att = d.b_att; p.mask = d.mask;
  p.score = d.score; p.P = d.P; p.emb_rows = d.emb_rows; p.L = d.num_layers;
  for (int l = 0; l < d.num_layers; ++l) p.Din[l] = d.Din[l];
  p.B = d.B; p.N = d.N; p.E1 = d.E1; p.K = d.K; p.S = d.S; p.H = d.H; p.relu = d.relu;
  p.LB = lb; p.write_pad = d.write_pad; p.dbg = tcg::debug_flags();
  // the tile count lives in device memory (no host sync): one persistent CTA per SM, bounded by
  // the worst case of one graph per tile
  return tcg::launch<Pol>(stream, d.W_hi, d.W_lo, d.num_layers * d.H, d.Kw, smem, d.B, p, who);
}

}  // extern "C++"

int lnb_spectral_stack_forward(lnb_stream_t stream, const lnb_spectral_stack* desc) {
  LNB_REQUIRE(desc, "spectral_stack_forward: null descriptor");
  return launch_stack<SpectralPolicy>(stream, *desc, "spectral_stack_forward");
}

int lnb_sage_stack_forward(lnb_stream_t stream, const lnb_spectral_stack* desc, int flags) {
  LNB_REQUIRE(desc, "sage_stack_forward: null descriptor");
  LNB_REQUIRE((flags & ~LNB_SAGE_MAX) == 0, "sage_stack_forward: unknown flags %d", flags);
  if (desc->S != 0) {
    lnb::set_err("sage_stack_forward: S=%d, the GraphSAGE stack has no long scales (S must be 0)", desc->S);
    return LNB_ERR_UNSUPPORTED;
  }
  if (flags & LNB_SAGE_MAX)
    return launch_stack<SpectralPolicyT<STACK_SAGE_MAX>>(stream, *desc, "sage_stack_forward");
  return launch_stack<SpectralPolicyT<STACK_SAGE_MEAN>>(stream, *desc, "sage_stack_forward");
}

int lnb_spectral_conv_fused(lnb_stream_t stream, const float* X, const float* Q, const float* coeff,
                            const float* ell_val, const uint8_t* ell_idx, const int32_t* ell_max,
                            const int32_t* gext, const int32_t* tiles, const float* W_hi,
                            const float* W_lo, const float* bias, int B, int N, int Din, int E1,
                            int K, int S, int H, int relu, int write_pad, float* out) {
  lnb_spectral_stack d{};
  d.X = X; d.Q = Q; d.coeff = coeff; d.coeff_layer_stride = 0;
  d.ell_val = ell_val; d.ell_idx = ell_idx; d.ell_max = ell_max; d.gext = gext; d.tiles = tiles;
  d.W_hi = W_hi; d.W_lo = W_lo; d.Kw = (S + E1) * Din; d.bias = bias;
  d.Din[0] = Din; d.num_layers = 1; d.out_state = out; d.write_pad = write_pad;
  d.B = B; d.N = N; d.E1 = E1; d.K = K; d.S = S; d.H = H; d.relu = relu;
  return launch_stack<SpectralPolicy>(stream, d, "spectral_conv_fused");
}

}  // extern "C"
