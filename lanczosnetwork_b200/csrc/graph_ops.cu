// Small fused graph ops around the spectral convolution: embedding rows, Ritz power table,
// gated masked-mean readout, Gaussian-kernel Laplacian, tf32 hi/lo split.
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------
__global__ void embedding_rows_kernel(const int64_t* __restrict__ idx,
                                      const float* __restrict__ table, int64_t rows, int nemb,
                                      int dim, float* __restrict__ out) {
  const int64_t total = rows * dim;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / dim;
    int c = (int)(i % dim);
    int64_t id = idx[r];
    out[i] = (id >= 0 && id < nemb) ? table[id * dim + c] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------
struct PowerList { int v[32]; };

__global__ void ritz_power_table_kernel(const float* __restrict__ D, int64_t rows, PowerList pw,
                                        int S, float* __restrict__ table) {
  const int64_t total = rows * S;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / S;
    int s = (int)(i % S);
    // double pow then one rounding: correctly rounded fp32 power for integer exponents
    table[i] = (float)pow((double)D[r], (double)pw.v[s]);
  }
}

// ------------------------------------------------------------------------------------------
// Readout: one CTA per graph, nodes processed in chunks of RO_NODES.
constexpr int RO_NODES = 32;
constexpr int RO_THREADS = 256;

__global__ void __launch_bounds__(RO_THREADS)
readout_kernel(const float* __restrict__ state, const float* __restrict__ W_out,
               const float* __restrict__ b_out, const float* __restrict__ w_att,
               const float* __restrict__ b_att, const uint8_t* __restrict__ mask, int N, int H,
               int P, float* __restrict__ score) {
  extern __shared__ float smem[];
  const int HP = H | 1;                 // odd stride
  float* Ws = smem;                     // (P+1) x HP   rows 0..P-1 = W_out, row P = w_att
  float* Xs = Ws + (P + 1) * HP;        // RO_NODES x HP
  float* Ys = Xs + RO_NODES * HP;       // RO_NODES x (P+1)
  const int g = blockIdx.x, tid = threadIdx.x;
  for (int e = tid; e < (P + 1) * H; e += RO_THREADS) {
    int p = e / H, h = e % H;
    Ws[p * HP + h] = (p < P) ? W_out[p * H + h] : w_att[h];
  }
  float acc = 0.f;                      // thread p < P owns score[g][p]
  int count = 0;
  for (int n0 = 0; n0 < N; n0 += RO_NODES) {
    const int nn = min(RO_NODES, N - n0);
    __syncthreads();
    for (int e = tid; e < nn * H; e += RO_THREADS) {
      int n = e / H, h = e % H;
      Xs[n * HP + h] = state[((int64_t)g * N + n0 + n) * H + h];
    }
    __syncthreads();
    for (int e = tid; e < nn * (P + 1); e += RO_THREADS) {
      int n = e / (P + 1), p = e % (P + 1);
      const float* x = Xs + n * HP;
      const float* w = Ws + p * HP;
      float s = 0.f;
      for (int h = 0; h < H; ++h) s = fmaf(x[h], w[h], s);
      s += (p < P) ? b_out[p] : b_att[0];
      Ys[n * (P + 1) + p] = s;
    }
    __syncthreads();
    if (tid < P) {
      for (int n = 0; n < nn; ++n) {
        bool on = mask ? (mask[(int64_t)g * N + n0 + n] != 0) : true;
        if (on) {
          float gate = 1.f / (1.f + expf(-Ys[n * (P + 1) + P]));
          acc += gate * Ys[n * (P + 1) + tid];
          ++count;
        }
      }
    }
  }
  if (tid < P) score[(int64_t)g * P + tid] = acc / (float)count;   // 0/0 -> NaN like torch.mean([])
}

// ------------------------------------------------------------------------------------------
// Gaussian-kernel Laplacian: one CTA per graph; node features staged in shared memory.
constexpr int GL_THREADS = 256;

__device__ __forceinline__ float gl_block_sum(float v, float* red) {
  v = lnb::warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < GL_THREADS / 32) ? red[lane] : 0.f;
  t = lnb::warp_sum(t);
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(GL_THREADS)
gaussian_laplacian_kernel(const float* __restrict__ x, const float* __restrict__ L, int N, int Dx,
                          int E1, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int DP = Dx | 1;
  float* Xs = smem;                // N x DP
  float* dv = Xs + (int64_t)N * DP;  // N
  float* red = dv + N;             // 32
  const int g = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nwarps = GL_THREADS / 32;
  for (int e = tid; e < N * Dx; e += GL_THREADS) {
    int n = e / Dx, d = e % Dx;
    Xs[n * DP + d] = x[((int64_t)g * N + n) * Dx + d];
  }
  __syncthreads();
  // pass 1: sigma2 = mean_{i,j} |x_i - x_j|^2 over ALL N^2 pairs (padded nodes included)
  float part = 0.f;
  for (int e = tid; e < N * N; e += GL_THREADS) {
    int i = e / N, j = e % N;
    const float* xi = Xs + i * DP;
    const float* xj = Xs + j * DP;
    float s = 0.f;
    for (int d = 0; d < Dx; ++d) { float t = xj[d] - xi[d]; s = fmaf(t, t, s); }
    part += s;
  }
  const float sigma2 = gl_block_sum(part, red) / (float)(N * N);
  // pass 2: A_ij = exp(-dist2/sigma2) * adj_ij, row sums  (one warp per row)
  const float* Lg = L + (int64_t)g * N * N * E1;
  float* og = out + (int64_t)g * N * N;
  for (int i = warp; i < N; i += nwarps) {
    const float* xi = Xs + i * DP;
    float rs = 0.f;
    for (int j = lane; j < N; j += 32) {
      const float* xj = Xs + j * DP;
      float s = 0.f;
      for (int d = 0; d < Dx; ++d) { float t = xj[d] - xi[d]; s = fmaf(t, t, s); }
      float adj = (Lg[((int64_t)i * N + j) * E1] != 0.f) ? 1.f : 0.f;
      float a = expf(-s / sigma2) * adj;
      og[(int64_t)i * N + j] = a;
      rs += a;
    }
    rs = lnb::warp_sum(rs);
    if (lane == 0) {
      float padv = (rs == 0.f) ? 1.f : 0.f;
      dv[i] = 1.f / sqrtf(rs + padv);
    }
  }
  __syncthreads();
  // pass 3: out_ij = (d_i * A_ij) * d_j  (same thread re-reads what it wrote)
  for (int i = warp; i < N; i += nwarps) {
    const float di = dv[i];
    for (int j = lane; j < N; j += 32) {
      float a = og[(int64_t)i * N + j];
      og[(int64_t)i * N + j] = (di * a) * dv[j];
    }
  }
}

// ------------------------------------------------------------------------------------------
// Operator chain on channel 0 of the operators, one CTA per graph, thread <-> feature column:
//   power mode     w_s = L_0 w_{s-1}, w_0 = X               (model/dcnn.py:88-92, lanczos_net.py:164-169)
//   Chebyshev mode s_0 = L_0 X, s_k = 2 L_0 s_{k-1} - s_{k-2}, s_{-1} = X   (model/cheby_net.py:88-93)
// The N x N operator (transposed, so 4 rows of one column are one LDS.128) and the current walk
// live in shared memory; a thread keeps its column of the new walk in N <= 32 registers, so one
// step costs N^2 FMA + N^2/4 broadcast loads per thread.  Selected steps are written straight into
// their column block of the message matrix (block index = sel[step], < 0: not stored).
struct ChainSel { int8_t blk[LNB_CHAIN_MAX_STEPS]; };

__global__ void __launch_bounds__(128)
operator_chain_kernel(const float* __restrict__ L, const float* __restrict__ X, int N, int E1, int D,
                      int steps, int cheby, ChainSel sel, float* __restrict__ out, int64_t out_sb,
                      int64_t out_sn, int out_col0) {
  __shared__ __align__(16) float Lt[LNB_CHAIN_MAX_N][LNB_CHAIN_MAX_N];   // Lt[i][n] = L_0[n][i]
  extern __shared__ __align__(16) float walk[];                // [2][N][Dc] ping-pong, Dc = blockDim.x
  const int g = blockIdx.x, d0 = blockIdx.y * blockDim.x, t = threadIdx.x;
  const int Dc = blockDim.x;
  const bool live = d0 + t < D;
  const float* Lg = L + (int64_t)g * N * N * E1;
  for (int e = t; e < LNB_CHAIN_MAX_N * LNB_CHAIN_MAX_N; e += Dc) {
    const int i = e / LNB_CHAIN_MAX_N, n = e % LNB_CHAIN_MAX_N;
    Lt[i][n] = (i < N && n < N) ? __ldg(Lg + ((int64_t)n * N + i) * E1) : 0.f;
  }
  float* w0 = walk;
  float* w1 = walk + (size_t)N * Dc;
  const float* Xg = X + (int64_t)g * N * D + d0;
  for (int n = 0; n < N; ++n) w0[n * Dc + t] = live ? __ldg(Xg + (int64_t)n * D + t) : 0.f;
  __syncthreads();
  float* og = out + (int64_t)g * out_sb + d0 + t;
  float prev2[LNB_CHAIN_MAX_N];                                     // Chebyshev: s_{k-2} of this column
#pragma unroll
  for (int n = 0; n < LNB_CHAIN_MAX_N; ++n) prev2[n] = (cheby && n < N) ? w0[n * Dc + t] : 0.f;
  for (int s = 0; s < steps; ++s) {
    float acc[LNB_CHAIN_MAX_N];
#pragma unroll
    for (int n = 0; n < LNB_CHAIN_MAX_N; ++n) acc[n] = 0.f;
    for (int i = 0; i < N; ++i) {
      const float o = w0[i * Dc + t];
      const float4* l4 = reinterpret_cast<const float4*>(&Lt[i][0]);
#pragma unroll
      for (int q = 0; q < LNB_CHAIN_MAX_N / 4; ++q) {
        const float4 l = l4[q];
        acc[4 * q + 0] = fmaf(l.x, o, acc[4 * q + 0]); acc[4 * q + 1] = fmaf(l.y, o, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(l.z, o, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(l.w, o, acc[4 * q + 3]);
      }
    }
    const int blk = sel.blk[s];
#pragma unroll
    for (int n = 0; n < LNB_CHAIN_MAX_N; ++n) {
      if (n < N) {
        float v = acc[n];
        if (cheby && s > 0) {                                  // s_k = 2 L s_{k-1} - s_{k-2}
          v = 2.0f * v - prev2[n];
          prev2[n] = w0[n * Dc + t];
        }
        w1[n * Dc + t] = v;
        if (blk >= 0 && live) og[(int64_t)n * out_sn + (int64_t)(out_col0 + blk) * D] = v;
      }
    }
    __syncthreads();
    float* tmp = w0; w0 = w1; w1 = tmp;
  }
}

// ------------------------------------------------------------------------------------------
// Whole message matrix of a general-shape spectral convolution layer in ONE launch
// (model/lanczos_net.py:157-180, model/ada_lanczos_net.py:321-345):
//   msg = [ L_0^k X  (k in short) ] ++ [ Q G_s Q^T X  (s < S) ] ++ [ L_e X  (e < E1) ]
// with G_s either dense symmetric K x K blocks (AdaLanczosNet's learned filter) or diag(f[:, s])
// (LanczosNet).  One CTA per graph, thread <-> feature column d: the column X[:, d] and every
// intermediate (walk, U = Q^T x, G u, Q w) live in registers with fully unrolled static indexing;
// the operators (transposed), Q, Q^T and the filters are staged once in shared memory and read as
// 16-byte broadcasts.  Replaces five launches of the FFMA batched GEMM per layer (36 us each at
// B = 256, tiles of 64 x 64 for 26-row operands) by one.

struct MsgParams {
  const float* L; const float* X; const float* Q; const float* G; const float* coeff;
  int N, E1, D, K, S, dense_filter, short_steps, n_short;
  ChainSel sel;
  float* out; int64_t out_sb, out_sn;
};

__device__ __forceinline__ void msg_matvec(const float* __restrict__ Mt /* [32][32]: Mt[i][n] */,
                                           const float (&in)[LNB_MESSAGES_MAX_N], float (&acc)[LNB_MESSAGES_MAX_N]) {
#pragma unroll
  for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n) acc[n] = 0.f;
#pragma unroll
  for (int i = 0; i < LNB_MESSAGES_MAX_N; ++i) {
    const float o = in[i];
    const float4* l4 = reinterpret_cast<const float4*>(Mt + i * LNB_MESSAGES_MAX_N);
#pragma unroll
    for (int q = 0; q < LNB_MESSAGES_MAX_N / 4; ++q) {
      const float4 l = l4[q];
      acc[4 * q + 0] = fmaf(l.x, o, acc[4 * q + 0]); acc[4 * q + 1] = fmaf(l.y, o, acc[4 * q + 1]);
      acc[4 * q + 2] = fmaf(l.z, o, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(l.w, o, acc[4 * q + 3]);
    }
  }
}

__global__ void __launch_bounds__(128)
graph_messages_kernel(const MsgParams P) {
  extern __shared__ __align__(16) float msg_smem[];
  const int N = P.N, E1 = P.E1, D = P.D, K = P.K, S = P.S;
  float* Lt = msg_smem;                                   // [E1][32][32]  Lt[e][i][n] = L[n][i][e]
  float* Qs = Lt + (size_t)E1 * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_N;   // [32 n][32 k]
  float* Qt = Qs + LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_K;                // [32 k][32 n]
  float* Gs = Qt + LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_K;                // [S][32][32] dense blocks, or [S][32] diagonals
  const int g = blockIdx.x, d = blockIdx.y * blockDim.x + threadIdx.x, t = threadIdx.x, nt = blockDim.x;
  // blockIdx.z: 0 = edge types + short walk, 1 = long scales (two CTAs per graph halve the serial
  // work of a column; each stages only what it reads)
  const bool do_edges = blockIdx.z == 0, do_long = (gridDim.z == 1 || blockIdx.z == 1) && S > 0;
  const bool live = d < D;
  const float* Lg = P.L + (int64_t)g * N * N * E1;
  if (do_edges) for (int e = t; e < E1 * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_N; e += nt) Lt[e] = 0.f;
  if (do_long) for (int e = t; e < 2 * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_K; e += nt) Qs[e] = 0.f;
  __syncthreads();
  if (do_edges) for (int e = t; e < N * N * E1; e += nt) {              // coalesced read, transposed scatter
    const int ch = e % E1, ij = e / E1, r = ij / N, c = ij - r * N;
    Lt[((size_t)ch * LNB_MESSAGES_MAX_N + c) * LNB_MESSAGES_MAX_N + r] = __ldg(Lg + e);
  }
  if (do_long) {
    const float* Qg = P.Q + (int64_t)g * N * K;
    for (int e = t; e < N * K; e += nt) {
      const int n = e / K, k = e - n * K;
      const float v = __ldg(Qg + e);
      Qs[n * LNB_MESSAGES_MAX_K + k] = v;
      Qt[k * LNB_MESSAGES_MAX_N + n] = v;
    }
    if (P.dense_filter) {
      const float* Gg = P.G + (int64_t)g * S * K * K;
      for (int e = t; e < S * LNB_MESSAGES_MAX_K * LNB_MESSAGES_MAX_K; e += nt) {
        const int s = e / (LNB_MESSAGES_MAX_K * LNB_MESSAGES_MAX_K);
        const int rc = e - s * LNB_MESSAGES_MAX_K * LNB_MESSAGES_MAX_K;
        const int r = rc / LNB_MESSAGES_MAX_K, c = rc - r * LNB_MESSAGES_MAX_K;
        // row r of Gs = column r of G_s (what the unrolled product over the input index reads)
        Gs[e] = (r < K && c < K) ? __ldg(Gg + ((int64_t)s * K + c) * K + r) : 0.f;
      }
    } else {
      const float* fg = P.coeff + (int64_t)g * K * S;       // [K][S]
      for (int e = t; e < S * LNB_MESSAGES_MAX_K; e += nt) {
        const int s = e / LNB_MESSAGES_MAX_K, k = e - s * LNB_MESSAGES_MAX_K;
        Gs[e] = (k < K) ? __ldg(fg + (int64_t)k * S + s) : 0.f;
      }
    }
  }
  float x[LNB_MESSAGES_MAX_N];
  const float* Xg = P.X + (int64_t)g * N * D + d;
#pragma unroll
  for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n) x[n] = (live && n < N) ? __ldg(Xg + (int64_t)n * D) : 0.f;
  __syncthreads();
  float* og = P.out + (int64_t)g * P.out_sb + d;
  float y[LNB_MESSAGES_MAX_N];
  // ---- edge types (and the first step of the short walk: both are L_0 X) ------------------------
  if (do_edges)
  for (int e = E1 - 1; e >= 0; --e) {                      // channel 0 last: its result seeds the walk
    msg_matvec(Lt + (size_t)e * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_N, x, y);
    if (live) {
#pragma unroll
      for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n)
        if (n < N) og[(int64_t)n * P.out_sn + (int64_t)(P.n_short + S + e) * D] = y[n];
    }
  }
  // ---- short diffusion walk: w_k = L_0 w_{k-1} (lanczos_net.py:164-169) ---------------------------
  for (int step = 1; do_edges && step <= P.short_steps; ++step) {
    if (step > 1) {
      float w[LNB_MESSAGES_MAX_N];
#pragma unroll
      for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n) w[n] = y[n];
      msg_matvec(Lt, w, y);
    }
    const int blk = P.sel.blk[step - 1];
    if (blk >= 0 && live) {
#pragma unroll
      for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n)
        if (n < N) og[(int64_t)n * P.out_sn + (int64_t)blk * D] = y[n];
    }
  }
  // ---- long scales: Q G_s (Q^T x) -------------------------------------------------------------------
  if (do_long) {
    float u[LNB_MESSAGES_MAX_K];
#pragma unroll
    for (int k = 0; k < LNB_MESSAGES_MAX_K; ++k) u[k] = 0.f;
#pragma unroll
    for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n) {                   // u = Q^T x
      const float o = x[n];
      const float4* q4 = reinterpret_cast<const float4*>(Qs + n * LNB_MESSAGES_MAX_K);
#pragma unroll
      for (int q = 0; q < LNB_MESSAGES_MAX_K / 4; ++q) {
        const float4 l = q4[q];
        u[4 * q + 0] = fmaf(l.x, o, u[4 * q + 0]); u[4 * q + 1] = fmaf(l.y, o, u[4 * q + 1]);
        u[4 * q + 2] = fmaf(l.z, o, u[4 * q + 2]); u[4 * q + 3] = fmaf(l.w, o, u[4 * q + 3]);
      }
    }
    for (int s = 0; s < S; ++s) {
      float w[LNB_MESSAGES_MAX_K];
      if (P.dense_filter) {
        msg_matvec(Gs + (size_t)s * LNB_MESSAGES_MAX_K * LNB_MESSAGES_MAX_K, u, w);        // w = G_s u
      } else {
        const float4* f4 = reinterpret_cast<const float4*>(Gs + s * LNB_MESSAGES_MAX_K);
#pragma unroll
        for (int q = 0; q < LNB_MESSAGES_MAX_K / 4; ++q) {
          const float4 f = f4[q];
          w[4 * q + 0] = f.x * u[4 * q + 0]; w[4 * q + 1] = f.y * u[4 * q + 1];
          w[4 * q + 2] = f.z * u[4 * q + 2]; w[4 * q + 3] = f.w * u[4 * q + 3];
        }
      }
      msg_matvec(Qt, w, y);                                             // y = Q w
      if (live) {
#pragma unroll
        for (int n = 0; n < LNB_MESSAGES_MAX_N; ++n)
          if (n < N) og[(int64_t)n * P.out_sn + (int64_t)(P.n_short + s) * D] = y[n];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_rna(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

__global__ void split_tf32_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ hi,
                                  float* __restrict__ lo) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v = x[i];
    float h = tf32_rna(v);
    hi[i] = h;
    lo[i] = tf32_rna(v - h);
  }
}

int flat_grid(int64_t total) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = 132 * 16;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

extern "C" {

int lnb_embedding_rows(lnb_stream_t stream, const int64_t* idx, const float* table, int64_t rows,
                       int num_embeddings, int dim, float* out) {
  LNB_REQUIRE(idx && table && out, "embedding_rows: null pointer");
  LNB_REQUIRE(rows >= 0 && num_embeddings > 0 && dim > 0, "embedding_rows: bad dims");
  if (rows == 0) return LNB_OK;
  embedding_rows_kernel<<<flat_grid(rows * dim), 256, 0, (cudaStream_t)stream>>>(
      idx, table, rows, num_embeddings, dim, out);
  lnb::count_launch();
  return lnb::finish_launch("embedding_rows");
}

int lnb_ritz_power_table(lnb_stream_t stream, const float* D, int64_t rows, const int* powers,
                         int S, float* table) {
  LNB_REQUIRE(D && powers && table, "ritz_power_table: null pointer");
  LNB_REQUIRE(rows >= 0 && S >= 1 && S <= LNB_FILTER_MLP_MAX_S, "ritz_power_table: bad dims rows=%lld S=%d",
              (long long)rows, S);
  if (rows == 0) return LNB_OK;
  PowerList pw;
  for (int i = 0; i < S; ++i) pw.v[i] = powers[i];
  ritz_power_table_kernel<<<flat_grid(rows * S), 256, 0, (cudaStream_t)stream>>>(D, rows, pw, S,
                                                                                 table);
  lnb::count_launch();
  return lnb::finish_launch("ritz_power_table");
}

int lnb_readout(lnb_stream_t stream, const float* state, const float* W_out, const float* b_out,
                const float* w_att, const float* b_att, const uint8_t* mask, int B, int N, int H,
                int P, float* score) {
  LNB_REQUIRE(state && W_out && b_out && w_att && b_att && score, "readout: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && H >= 1 && P >= 1 && P < RO_THREADS, "readout: bad dims");
  if (B == 0) return LNB_OK;
  const int HP = H | 1;
  size_t shm = ((size_t)(P + 1) * HP + (size_t)RO_NODES * HP + (size_t)RO_NODES * (P + 1)) *
               sizeof(float);
  LNB_REQUIRE(shm <= lnb::SMEM_MAX, "readout: H=%d P=%d exceed shared memory", H, P);
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(readout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  readout_kernel<<<B, RO_THREADS, shm, (cudaStream_t)stream>>>(state, W_out, b_out, w_att, b_att,
                                                                mask, N, H, P, score);
  lnb::count_launch();
  return lnb::finish_launch("readout");
}

int lnb_gaussian_laplacian(lnb_stream_t stream, const float* x, const float* L, int B, int N,
                           int Dx, int E1, float* out) {
  LNB_REQUIRE(x && L && out, "gaussian_laplacian: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && Dx >= 1 && E1 >= 1, "gaussian_laplacian: bad dims");
  if (B == 0) return LNB_OK;
  size_t shm = ((size_t)N * (Dx | 1) + N + 32) * sizeof(float);
  if (shm > lnb::SMEM_MAX) {
    lnb::set_err("gaussian_laplacian: N=%d x Dx=%d node features exceed shared memory", N, Dx);
    return LNB_ERR_UNSUPPORTED;
  }
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(gaussian_laplacian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)shm);
  gaussian_laplacian_kernel<<<B, GL_THREADS, shm, (cudaStream_t)stream>>>(x, L, N, Dx, E1, out);
  lnb::count_launch();
  return lnb::finish_launch("gaussian_laplacian");
}

int lnb_operator_chain(lnb_stream_t stream, const float* L, const float* X, int B, int N, int E1,
                       int D, int steps, int chebyshev, const int* block_of_step, float* out,
                       int64_t out_batch_stride, int64_t out_row_stride, int out_col0) {
  LNB_REQUIRE(L && X && out && block_of_step, "operator_chain: null pointer");
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1 && D >= 1 && steps >= 1, "operator_chain: bad dims");
  if (N > LNB_CHAIN_MAX_N || steps > LNB_CHAIN_MAX_STEPS) {
    lnb::set_err("operator_chain: N=%d steps=%d exceed the register-resident kernel (N <= %d, steps <= %d)",
                 N, steps, LNB_CHAIN_MAX_N, LNB_CHAIN_MAX_STEPS);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  ChainSel sel;
  for (int s = 0; s < LNB_CHAIN_MAX_STEPS; ++s) sel.blk[s] = s < steps ? (int8_t)block_of_step[s] : (int8_t)-1;
  const int threads = 128;
  dim3 grid((unsigned)B, (unsigned)lnb::ceil_div(D, threads));
  const size_t shm = (size_t)2 * N * threads * sizeof(float);
  operator_chain_kernel<<<grid, threads, shm, (cudaStream_t)stream>>>(
      L, X, N, E1, D, steps, chebyshev ? 1 : 0, sel, out, out_batch_stride, out_row_stride, out_col0);
  lnb::count_launch();
  return lnb::finish_launch("operator_chain");
}

int lnb_graph_messages(lnb_stream_t stream, const float* L, const float* X, const float* Q,
                       const float* filt, int B, int N, int E1, int D, int K, int S, int dense_filter,
                       int short_steps, const int* block_of_step, int n_short, float* out,
                       int64_t out_batch_stride, int64_t out_row_stride) {
  LNB_REQUIRE(L && X && out, "graph_messages: null pointer");
  LNB_REQUIRE(S == 0 || (Q && filt), "graph_messages: long scales need Q and the filters");
  LNB_REQUIRE(short_steps == 0 || block_of_step, "graph_messages: block_of_step missing");
  LNB_REQUIRE(B >= 0 && N >= 1 && E1 >= 1 && D >= 1 && S >= 0 && short_steps >= 0 && n_short >= 0,
              "graph_messages: bad dims");
  if (N > LNB_MESSAGES_MAX_N || (S > 0 && K > LNB_MESSAGES_MAX_K) || E1 > LNB_MAX_E1 || S > LNB_MESSAGES_MAX_S ||
      short_steps > LNB_CHAIN_MAX_STEPS) {
    lnb::set_err("graph_messages: N=%d K=%d E1=%d S=%d outside the one-launch kernel (N,K <= 32, E1 <= 16, S <= 8)",
                 N, K, E1, S);
    return LNB_ERR_UNSUPPORTED;
  }
  if (B == 0) return LNB_OK;
  MsgParams p;
  p.L = L; p.X = X; p.Q = Q; p.G = dense_filter ? filt : nullptr; p.coeff = dense_filter ? nullptr : filt;
  p.N = N; p.E1 = E1; p.D = D; p.K = K; p.S = S; p.dense_filter = dense_filter;
  p.short_steps = short_steps; p.n_short = n_short;
  for (int s = 0; s < LNB_CHAIN_MAX_STEPS; ++s) p.sel.blk[s] = s < short_steps ? (int8_t)block_of_step[s] : (int8_t)-1;
  p.out = out; p.out_sb = out_batch_stride; p.out_sn = out_row_stride;
  const int threads = 128;
  const size_t shm = ((size_t)E1 * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_N + 2 * LNB_MESSAGES_MAX_N * LNB_MESSAGES_MAX_K +
                      (S > 0 ? (dense_filter ? (size_t)S * LNB_MESSAGES_MAX_K * LNB_MESSAGES_MAX_K
                                             : (size_t)S * LNB_MESSAGES_MAX_K) : 0)) * sizeof(float);
  if (shm > 48 * 1024)
    cudaFuncSetAttribute(graph_messages_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
  dim3 grid((unsigned)B, (unsigned)lnb::ceil_div(D, threads), S > 0 ? 2u : 1u);
  graph_messages_kernel<<<grid, threads, shm, (cudaStream_t)stream>>>(p);
  lnb::count_launch();
  return lnb::finish_launch("graph_messages");
}

int lnb_split_tf32(lnb_stream_t stream, const float* x, int64_t n, float* hi, float* lo) {
  LNB_REQUIRE(x && hi && lo, "split_tf32: null pointer");
  LNB_REQUIRE(n >= 0, "split_tf32: negative length");
  if (n == 0) return LNB_OK;
  split_tf32_kernel<<<flat_grid(n), 256, 0, (cudaStream_t)stream>>>(x, n, hi, lo);
  lnb::count_launch();
  return lnb::finish_launch("split_tf32");
}

}  // extern "C"
