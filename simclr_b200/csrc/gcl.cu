// Generalized contrastive loss (Chen, Luo, Li, "Intriguing Properties of Contrastive Losses", NeurIPS 2021):
// L = loss_scaling * (L_align + lambda * L_dist) on z = l2_normalize(hidden) (or hidden), h1 = z[:B], h2 = z[B:].
//
//   L_align = sum (h1 - h2)^2 / (2 B D)                                    over this replica's rows
//   L_dist  = mean_i [logsumexp_j (z_i . z_j / tau) - ln D]               'logsumexp': local rows i, all 2G rows j
//           = mean over the 2G x D entries of (sort(P W) - sort(z W))^2    sliced Wasserstein ('normal', 'uniform')
//
// All fp32 on CUDA cores (the QR in fp64), every reduction in a fixed order: the same bits on every run and replica.
// The logsumexp term is tiled like ntxent.cu (online LSE forward, recomputed tiles backward with the gathered lse);
// the sliced Wasserstein term sorts each projected column in shared memory with one CTA per column.
#include "common.cuh"

namespace simclr {
namespace {

constexpr int MAXD = 256;
constexpr int MAX_SORT = 16384;     // rows per sorted column: 16384 64-bit keys = 128 KiB of shared memory
constexpr int RB = 32;              // logsumexp tiles: local rows per block
constexpr int CT = 64;              //                  gathered columns per tile
constexpr int NT = 256;             //                  threads: 8 warps x 4 rows
constexpr int QR_THREADS = 256;     // one thread per column of the D x D matrix

__device__ __forceinline__ int64_t zall_row(int v, int64_t g, int64_t B) {
  // z_all is [R][2][B][D]; global sample g = r*B + i
  const int64_t r = g / B, i = g - r * B;
  return (r * 2 + v) * B + i;
}

// global row c in [0, 2G) (view-major over the whole job: c = v*G + r*B + i) -> row of z_all
__device__ __forceinline__ int64_t global_row(int64_t c, int64_t G, int64_t B) {
  const int v = (int)(c / G);
  return zall_row(v, c - (int64_t)v * G, B);
}

template <typename T>
__device__ T block_sum(T v, T* sh) {
  // fixed-order block reduction; every thread gets the total
  v = warp_sum(v);
  const int warps = (blockDim.x + 31) >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  for (int w = 0; w < warps; ++w) s += sh[w];
  return s;
}

// ---- draws: Philox-4x32-10 keyed by (seed, step), counter (column, row, step, stream) -------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

enum { TAG_PRIOR = 1, TAG_ORTHO = 2 };

__device__ __forceinline__ float draw_one(uint64_t seed, uint64_t step, int tag, int64_t row, int col, int uniform) {
  const uint4 ctr = make_uint4((uint32_t)col, (uint32_t)row, (uint32_t)step,
                               (uint32_t)(step >> 32) ^ ((uint32_t)tag << 28));
  const uint4 x = philox4x32_10(ctr, make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  if (uniform) return ((float)(x.x >> 9) + 0.5f) * 0x1p-22f - 1.f;     // U(-1, 1), symmetric, never +-1
  // Box-Muller in fp64: u1 in (0, 1], u2 in [0, 1)
  const double u1 = ((double)x.x + 1.0) * 0x1p-32, u2 = (double)x.y * 0x1p-32;
  return (float)(sqrt(-2.0 * log(u1)) * cospi(2.0 * u2));
}

// one warp per row: rows [0, prior_rows) of the prior (l2-normalised if `normalize`), then the D rows of the normal
// matrix; out[row][0..D)
__global__ void draw_kernel(uint64_t seed, const int64_t* __restrict__ step_dev, int64_t prior_rows, int64_t w_rows,
                            int D, int uniform, int normalize, float* __restrict__ prior, float* __restrict__ wnormal) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  int64_t row = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= prior_rows + w_rows) return;
  int tag = TAG_PRIOR;
  float* out = prior;
  if (row >= prior_rows) {
    row -= prior_rows;
    tag = TAG_ORTHO; out = wnormal; uniform = 0; normalize = 0;
  }
  const uint64_t step = (uint64_t)step_dev[0];
  float v[MAXD / 32];
  float ss = 0.f;
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    v[e] = d < D ? draw_one(seed, step, tag, row, d, uniform) : 0.f;
    ss = fmaf(v[e], v[e], ss);
  }
  ss = warp_sum(ss);
  const float inv = normalize ? rsqrtf(fmaxf(ss, 1e-12f)) : 1.f;     // tf.math.l2_normalize
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    if (d < D) out[row * D + d] = v[e] * inv;
  }
}

// ---- orthogonal matrix: one-CTA Householder QR in fp64, Q with its columns times sign(diag R) ----------------------
// A [D][D] and V [D][D] (the reflectors) are fp64 scratch in global memory (L2-resident); thread j owns column j.
__global__ void __launch_bounds__(QR_THREADS)
householder_kernel(const float* __restrict__ a_in, int D, double* __restrict__ A, double* __restrict__ V,
                   float* __restrict__ Q) {
  __shared__ double sh[QR_THREADS / 32];
  __shared__ double beta[MAXD];
  __shared__ double sgn[MAXD];
  __shared__ double v[MAXD];
  const int t = threadIdx.x;
  for (int i = t; i < D * D; i += blockDim.x) A[i] = (double)a_in[i];
  __syncthreads();
  for (int k = 0; k < D; ++k) {
    const int i = k + t;
    const double x = i < D ? A[(int64_t)i * D + k] : 0.0;
    const double ss = block_sum(x * x, sh);
    const double x0 = A[(int64_t)k * D + k];
    const double sigma = sqrt(ss);
    const double alpha = x0 >= 0.0 ? -sigma : sigma;            // R[k][k]
    const double vv = 2.0 * sigma * (sigma + fabs(x0));           // |x - alpha e_k|^2
    if (i < D) {
      const double vi = (i == k) ? x0 - alpha : x;
      v[i] = vi;
      V[(int64_t)k * D + i] = vi;
    }
    if (t == 0) {
      beta[k] = vv > 0.0 ? 2.0 / vv : 0.0;
      sgn[k] = alpha < 0.0 ? -1.0 : 1.0;
    }
    __syncthreads();
    if (t > k && t < D) {
      double dot = 0.0;
      for (int r = k; r < D; ++r) dot = fma(v[r], A[(int64_t)r * D + t], dot);
      const double f = beta[k] * dot;
      for (int r = k; r < D; ++r) A[(int64_t)r * D + t] = fma(-f, v[r], A[(int64_t)r * D + t]);
    }
    __syncthreads();
  }
  // Q = H_0 H_1 ... H_{D-1} I, applied from the last reflector on
  for (int i = 0; i < D; ++i)
    if (t < D) A[(int64_t)i * D + t] = (i == t) ? 1.0 : 0.0;
  __syncthreads();
  for (int k = D - 1; k >= 0; --k) {
    for (int i = k + t; i < D; i += blockDim.x) v[i] = V[(int64_t)k * D + i];
    __syncthreads();
    if (t >= k && t < D) {
      double dot = 0.0;
      for (int r = k; r < D; ++r) dot = fma(v[r], A[(int64_t)r * D + t], dot);
      const double f = beta[k] * dot;
      for (int r = k; r < D; ++r) A[(int64_t)r * D + t] = fma(-f, v[r], A[(int64_t)r * D + t]);
    }
    __syncthreads();
  }
  if (t < D)
    for (int i = 0; i < D; ++i) Q[(int64_t)i * D + t] = (float)(A[(int64_t)i * D + t] * sgn[t]);
}

// ---- alignment: loss[1] = sum (h1 - h2)^2 / (2 B D), dz = +-(h1 - h2) / (B D); loss[0] = ls (loss[1] + lambda loss[2])
__global__ void __launch_bounds__(1024)
align_kernel(const float* __restrict__ z, int64_t B, int D, float lambda_weight, float loss_scaling,
             float* __restrict__ loss, float* __restrict__ dz) {
  __shared__ double sh[32];
  const int64_t n = B * D;
  const float inv = (float)(1.0 / (double)n);
  double acc = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    const float d = z[e] - z[n + e];
    acc += (double)d * (double)d;
    if (dz) {
      const float g = d * inv;
      dz[e] = g;
      dz[n + e] = -g;
    }
  }
  const double s = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    const float a = (float)(s / (2.0 * (double)n));
    loss[1] = a;
    loss[0] = loss_scaling * fmaf(lambda_weight, loss[2], a);
  }
}

// ---- logsumexp (decoupled NT-Xent): no mask, self and positive included ---------------------------------------------
__device__ __forceinline__ void load_rows(float* dst, const float* __restrict__ z_all, int64_t first, int count,
                                          int64_t total, int64_t G, int64_t B, int D, int ld) {
  for (int idx = threadIdx.x; idx < count * D; idx += NT) {
    const int r = idx / D, d = idx - r * D;
    const int64_t c = first + r;
    dst[r * ld + d] = c < total ? z_all[global_row(c, G, B) * D + d] : 0.f;
  }
}

__device__ __forceinline__ void load_local(float* dst, const float* __restrict__ z_all, int64_t row0, int64_t B,
                                           int64_t replica_id, int D, int ld) {
  for (int idx = threadIdx.x; idx < RB * D; idx += NT) {
    const int r = idx / D, d = idx - r * D;
    const int64_t lr = row0 + r;
    float v = 0.f;
    if (lr < 2 * B) {
      const int vv = (int)(lr / B);
      v = z_all[zall_row(vv, replica_id * B + (lr - (int64_t)vv * B), B) * D + d];
    }
    dst[r * ld + d] = v;
  }
}

__device__ __forceinline__ void tile_dots(const float* q, const float* k, int D, int ld, float acc[4][2]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = 0.f;
  const float* k0 = k + lane * ld;
  const float* k1 = k + (lane + 32) * ld;
  const float* qb = q + (warp * 4) * ld;
  for (int d = 0; d < D; ++d) {
    const float b0 = k0[d], b1 = k1[d];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = qb[j * ld + d];
      acc[j][0] = fmaf(a, b0, acc[j][0]);
      acc[j][1] = fmaf(a, b1, acc[j][1]);
    }
  }
}

__global__ void __launch_bounds__(NT)
lse_fwd_partial_kernel(const float* __restrict__ z_all, int64_t B, int64_t R, int D, int64_t replica_id,
                       float inv_temp, float* __restrict__ part /*[S][2B][2]*/, int tiles_per_split) {
  extern __shared__ float sm[];
  const int ld = D + 1;
  float* q = sm;
  float* k = sm + RB * ld;
  const int64_t G = R * B, rows = 2 * B, cols = 2 * G;
  const int64_t row0 = (int64_t)blockIdx.x * RB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_local(q, z_all, row0, B, replica_id, D, ld);
  float m[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { m[j] = -INFINITY; l[j] = 0.f; }
  const int64_t n_tiles = (cols + CT - 1) / CT;
  const int64_t t0 = (int64_t)blockIdx.y * tiles_per_split;
  const int64_t t1 = min(n_tiles, t0 + tiles_per_split);
  for (int64_t t = t0; t < t1; ++t) {
    __syncthreads();
    load_rows(k, z_all, t * CT, CT, cols, G, B, D, ld);
    __syncthreads();
    float acc[4][2];
    tile_dots(q, k, D, ld, acc);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (t * CT + lane + 32 * h >= cols) continue;
        const float s = acc[j][h] * inv_temp;
        if (s > m[j]) { l[j] = l[j] * __expf(m[j] - s) + 1.f; m[j] = s; }
        else          { l[j] += __expf(s - m[j]); }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float mm = warp_max(m[j]);
    float ll = (m[j] == -INFINITY) ? 0.f : l[j] * __expf(m[j] - mm);
    ll = warp_sum(ll);
    const int64_t lr = row0 + warp * 4 + j;
    if (lane == 0 && lr < rows) {
      float* p = part + ((int64_t)blockIdx.y * rows + lr) * 2;
      p[0] = mm; p[1] = ll;
    }
  }
}

__global__ void lse_fwd_finalize_kernel(const float* __restrict__ part, int splits, int64_t rows,
                                        float* __restrict__ lse) {
  const int64_t lr = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (lr >= rows) return;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, part[((int64_t)s * rows + lr) * 2]);
  float l = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float* p = part + ((int64_t)s * rows + lr) * 2;
    if (p[0] != -INFINITY) l += p[1] * expf(p[0] - m);
  }
  lse[lr] = m + logf(l);
}

// loss[2] = mean(lse) - ln D
__global__ void __launch_bounds__(1024) lse_mean_kernel(const float* __restrict__ lse, int64_t rows, int D,
                                                        float* __restrict__ loss) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < rows; i += blockDim.x) s += (double)lse[i];
  s = block_sum(s, sh);
  if (threadIdx.x == 0) loss[2] = (float)(s / (double)rows - log((double)D));
}

// dz_a = (1/tau) sum_j (P_aj + P_ja) z_j over this split's columns, P_ij = exp(s_ij - lse_i)
__global__ void __launch_bounds__(NT)
lse_bwd_partial_kernel(const float* __restrict__ z_all, const float* __restrict__ lse_all, int64_t B, int64_t R,
                       int D, int64_t replica_id, float inv_temp, float* __restrict__ part /*[S][2B][D]*/,
                       int tiles_per_split) {
  extern __shared__ float sm[];
  const int ld = D + 1;
  float* q = sm;
  float* k = q + RB * ld;
  float* cs = k + CT * ld;          // [RB][CT]
  float* lse_c = cs + RB * CT;      // [CT]
  const int64_t G = R * B, rows = 2 * B, cols = 2 * G;
  const int64_t row0 = (int64_t)blockIdx.x * RB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_local(q, z_all, row0, B, replica_id, D, ld);
  float rl[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t lr = row0 + warp * 4 + j;
    const int v = (int)(lr / B);
    rl[j] = (lr < rows) ? lse_all[zall_row(v, replica_id * B + (lr - (int64_t)v * B), B)] : 0.f;
  }
  constexpr int DJ = MAXD / 32;
  float dz[4][DJ];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < DJ; ++e) dz[j][e] = 0.f;
  const int64_t n_tiles = (cols + CT - 1) / CT;
  const int64_t t0 = (int64_t)blockIdx.y * tiles_per_split;
  const int64_t t1 = min(n_tiles, t0 + tiles_per_split);
  for (int64_t t = t0; t < t1; ++t) {
    __syncthreads();
    load_rows(k, z_all, t * CT, CT, cols, G, B, D, ld);
    if (threadIdx.x < CT) {
      const int64_t c = t * CT + threadIdx.x;
      lse_c[threadIdx.x] = c < cols ? lse_all[global_row(c, G, B)] : 0.f;
    }
    __syncthreads();
    float acc[4][2];
    tile_dots(q, k, D, ld, acc);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t lr = row0 + warp * 4 + j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cl = lane + 32 * h;
        float coef = 0.f;
        if (lr < rows && t * CT + cl < cols) {
          const float s = acc[j][h] * inv_temp;
          coef = __expf(s - rl[j]) + __expf(s - lse_c[cl]);
        }
        cs[(warp * 4 + j) * CT + cl] = coef;
      }
    }
    __syncwarp();   // each warp only reads back its own 4 rows of cs
    const float* cw = cs + (warp * 4) * CT;
    for (int b = 0; b < CT; ++b) {
      const float* kb = k + b * ld;
      const float c0 = cw[b], c1 = cw[CT + b], c2 = cw[2 * CT + b], c3 = cw[3 * CT + b];
#pragma unroll
      for (int e = 0; e < DJ; ++e) {
        const int d = lane + 32 * e;
        if (d < D) {
          const float kv = kb[d];
          dz[0][e] = fmaf(c0, kv, dz[0][e]);
          dz[1][e] = fmaf(c1, kv, dz[1][e]);
          dz[2][e] = fmaf(c2, kv, dz[2][e]);
          dz[3][e] = fmaf(c3, kv, dz[3][e]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t lr = row0 + warp * 4 + j;
    if (lr >= rows) continue;
    float* p = part + ((int64_t)blockIdx.y * rows + lr) * D;
#pragma unroll
    for (int e = 0; e < DJ; ++e) {
      const int d = lane + 32 * e;
      if (d < D) p[d] = dz[j][e];
    }
  }
}

__global__ void sum_splits_kernel(const float* __restrict__ part, int splits, int64_t n, float scale,
                                  float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = 0.f;
  for (int s = 0; s < splits; ++s) a += part[(int64_t)s * n + i];
  out[i] = a * scale;
}

int pick_splits(int64_t B, int64_t R, int* tiles_per_split) {
  const int64_t rows = 2 * B, cols = 2 * R * B;
  const int64_t row_blocks = (rows + RB - 1) / RB;
  const int64_t n_tiles = (cols + CT - 1) / CT;
  int64_t want = (2 * num_sms() + row_blocks - 1) / row_blocks;
  if (want < 1) want = 1;
  if (want > 16) want = 16;
  if (want > n_tiles) want = n_tiles;
  const int64_t tps = (n_tiles + want - 1) / want;
  *tiles_per_split = (int)tps;
  return (int)((n_tiles + tps - 1) / tps);
}

// ---- sliced Wasserstein --------------------------------------------------------------------------------------------
// C = A op(W) with A [M][K] (AMAP: row m of A is global row m of z_all), W [K][N] (TRANS_W: W is [N][K]);
// C [M][N], or [N][M] with TRANS_C.  64 x 64 tiles, 16-deep K steps, 4 x 4 outputs per thread, k ascending.
constexpr int GM = 64, GN = 64, GK = 16;
template <bool AMAP, bool TRANS_W, bool TRANS_C>
__global__ void __launch_bounds__(256)
gemm_kernel(const float* __restrict__ A, const float* __restrict__ W, float* __restrict__ C, int64_t M, int N, int K,
            int64_t B, int64_t G) {
  __shared__ float As[GK][GM + 4];
  __shared__ float Ws[GK][GN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * GM;
  const int n0 = blockIdx.y * GN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += GK) {
    for (int idx = threadIdx.x; idx < GM * GK; idx += 256) {
      const int r = idx / GK, kk = idx - r * GK;
      const int64_t m = m0 + r;
      float v = 0.f;
      if (m < M && k0 + kk < K) v = A[(AMAP ? global_row(m, G, B) : m) * K + k0 + kk];
      As[kk][r] = v;
    }
    for (int idx = threadIdx.x; idx < GN * GK; idx += 256) {
      int kk, c;
      if (TRANS_W) { c = idx / GK; kk = idx - c * GK; } else { kk = idx / GN; c = idx - kk * GN; }
      const int n = n0 + c;
      float v = 0.f;
      if (n < N && k0 + kk < K) v = TRANS_W ? W[(int64_t)n * K + k0 + kk] : W[(int64_t)(k0 + kk) * N + n];
      Ws[kk][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty + 16 * i]; b[i] = Ws[kk][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty + 16 * i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n >= N) continue;
      if (TRANS_C) C[(int64_t)n * M + m] = acc[i][j];
      else         C[m * N + n] = acc[i][j];
    }
  }
}

// order-preserving key: float bits (-0 keyed as +0) in the high word, row index in the low word
__device__ __forceinline__ unsigned long long sort_key(float x, uint32_t row) {
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | row;
}
__device__ __forceinline__ float key_value(unsigned long long key) {
  const uint32_t u = (uint32_t)(key >> 32);
  return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}

// One CTA sorts column blockIdx.x of x_t [cols][n] ascending (stable: ties by row index) with a bitonic network over
// npad (a power of two) keys in shared memory.  Outputs (each nullable): the sorted values, the permutation
// (perm[k] = source row of sorted position k), and against `ref` (another sorted column): diff = sorted - ref and the
// column's sum of diff^2 in fp64.  `sorted` may alias x_t.
__global__ void __launch_bounds__(1024)
sort_kernel(const float* x_t, int64_t n, int npad, float* sorted, int32_t* __restrict__ perm,
            const float* __restrict__ ref, float* __restrict__ diff, double* __restrict__ col_sq) {
  extern __shared__ unsigned long long keys[];
  __shared__ double sh[32];
  const int64_t col = blockIdx.x;
  const float* x = x_t + col * n;
  for (int i = threadIdx.x; i < npad; i += blockDim.x) keys[i] = i < n ? sort_key(x[i], (uint32_t)i) : ~0ull;
  __syncthreads();
  for (int k = 2; k <= npad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < npad; i += blockDim.x) {
        const int p = i ^ j;
        if (p > i) {
          const unsigned long long a = keys[i], b = keys[p];
          if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[p] = a; }
        }
      }
      __syncthreads();
    }
  }
  double acc = 0.0;
  for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
    const unsigned long long key = keys[k];
    const float v = key_value(key);
    if (sorted) sorted[col * n + k] = v;
    if (perm) perm[col * n + k] = (int32_t)(uint32_t)key;
    if (ref) {
      const float d = v - ref[col * n + k];
      diff[col * n + k] = d;
      acc += (double)d * (double)d;
    }
  }
  if (col_sq) {
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) col_sq[col] = acc;
  }
}

// loss[2] = sum_j col_sq[j] / (n D)
__global__ void swd_loss_kernel(const double* __restrict__ col_sq, int D, int64_t n, float* __restrict__ loss) {
  __shared__ double sh[32];
  double s = threadIdx.x < D ? col_sq[threadIdx.x] : 0.0;
  s = block_sum(s, sh);
  if (threadIdx.x == 0) loss[2] = (float)(s / ((double)n * (double)D));
}

// dS[local row][j] = 2 diff / (2G D) for every sorted position whose source row belongs to this replica: each local
// (row, column) is written exactly once
__global__ void swd_scatter_kernel(const int32_t* __restrict__ perm, const float* __restrict__ diff, int64_t B,
                                   int64_t G, int D, int64_t replica_id, float scale, float* __restrict__ dS) {
  const int64_t n = 2 * G;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * D) return;
  const int j = (int)(idx / n);
  const int64_t c = perm[idx];
  const int v = (int)(c / G);
  const int64_t g = c - (int64_t)v * G;
  if (g / B != replica_id) return;
  dS[(v * B + (g - replica_id * B)) * D + j] = diff[idx] * scale;
}

// ---- the l2-normalise backward of the summed term gradients ---------------------------------------------------------
__global__ void normalize_backward_kernel(const float* __restrict__ z, const float* __restrict__ inv_norm,
                                          int hidden_norm, int64_t rows, int D, const float* __restrict__ t0, float s0,
                                          const float* __restrict__ t1, float s1, const float* __restrict__ t2,
                                          float s2, float* __restrict__ dhidden) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* zr = z + row * D;
  float g[MAXD / 32];
  float dot = 0.f;
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    float a = 0.f;
    if (d < D) {
      const int64_t o = row * D + d;
      if (t0) a = s0 * t0[o];
      if (t1) a = fmaf(s1, t1[o], a);
      if (t2) a = fmaf(s2, t2[o], a);
      dot = fmaf(a, zr[d], dot);
    }
    g[e] = a;
  }
  dot = warp_sum(dot);
  const float inv = hidden_norm ? inv_norm[row] : 1.f;
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    // l2-normalise backward: dx = (dz - z (z . dz)) / ||x||
    if (d < D) dhidden[row * D + d] = hidden_norm ? (g[e] - zr[d] * dot) * inv : g[e];
  }
}

int sort_pad(int64_t n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

int launch_sort(const float* x_t, int64_t n, int64_t cols, float* sorted, int32_t* perm, const float* ref, float* diff,
                double* col_sq, cudaStream_t st) {
  const int npad = sort_pad(n);
  SIMCLR_CHECK_CUDA(cudaFuncSetAttribute(sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SORT * 8));
  sort_kernel<<<(unsigned)cols, 1024, (size_t)npad * 8, st>>>(x_t, n, npad, sorted, perm, ref, diff, col_sq);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

size_t lse_ws(int64_t B, int64_t R, int64_t D) {
  int tps;
  const int splits = pick_splits(B, R, &tps);
  return (size_t)splits * 2 * B * (D > 2 ? D : 2) * sizeof(float);
}

size_t swd_ws(int64_t B, int64_t R, int64_t D) {
  const size_t n = 2 * (size_t)R * B;
  const size_t fwd = align_up(2 * n * D * sizeof(float)) + align_up(D * sizeof(double));
  const size_t bwd = 2 * (size_t)B * D * sizeof(float);
  return fwd > bwd ? fwd : bwd;
}

}  // namespace
}  // namespace simclr

using namespace simclr;

#define GCL_CHECK_SHAPE(name, B, R, D, rid)                                                                        \
  do {                                                                                                             \
    SIMCLR_CHECK_ARG(B > 0 && R > 0 && D > 0 && rid >= 0 && rid < R, name ": need B,R,D > 0 and 0 <= replica_id < R " \
                     "(got B=%lld R=%lld D=%lld replica_id=%lld)", (long long)B, (long long)R, (long long)D,       \
                     (long long)rid);                                                                              \
    if (D > MAXD) {                                                                                                \
      set_error(name ": D=%lld is above the supported %d", (long long)D, MAXD);                                   \
      return SIMCLR_ERR_UNSUPPORTED;                                                                               \
    }                                                                                                              \
  } while (0)

#define GCL_CHECK_WS(name, have, need)                                                                             \
  do {                                                                                                             \
    if ((have) < (need)) {                                                                                         \
      set_error(name ": workspace too small (%zu < %zu)", (size_t)(have), (size_t)(need));                        \
      return SIMCLR_ERR_WORKSPACE;                                                                                 \
    }                                                                                                              \
  } while (0)

extern "C" {

size_t simclr_gcl_workspace_bytes(int64_t B, int64_t R, int64_t D) {
  if (B <= 0 || R <= 0 || D <= 0) return 0;
  const size_t a = lse_ws(B, R, D), b = swd_ws(B, R, D), c = 2 * (size_t)D * D * sizeof(double);
  return a > b ? (a > c ? a : c) : (b > c ? b : c);
}

int simclr_gcl_draw(int64_t seed, const int64_t* step, int64_t rows, int64_t D, int dist, int hidden_norm,
                    float* prior, float* wnormal, void* stream) {
  SIMCLR_CHECK_ARG(step && (prior || wnormal), "gcl_draw: null step, or neither prior nor wnormal");
  SIMCLR_CHECK_ARG((!prior || rows > 0) && D > 0, "gcl_draw: bad shape rows=%lld D=%lld", (long long)rows, (long long)D);
  SIMCLR_CHECK_ARG(dist == 0 || dist == 1, "gcl_draw: dist must be 0 (normal) or 1 (uniform), got %d", dist);
  if (D > MAXD) {
    set_error("gcl_draw: D=%lld is above the supported %d", (long long)D, MAXD);
    return SIMCLR_ERR_UNSUPPORTED;
  }
  // one launch whichever outputs are asked for
  const int64_t prior_rows = prior ? rows : 0, w_rows = wnormal ? D : 0;
  draw_kernel<<<(unsigned)((prior_rows + w_rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      (uint64_t)seed, step, prior_rows, w_rows, (int)D, dist, hidden_norm, prior, wnormal);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_orthogonal(const float* normal, int64_t D, float* W, void* workspace, size_t workspace_bytes,
                          void* stream) {
  SIMCLR_CHECK_ARG(normal && W && workspace, "gcl_orthogonal: null pointer");
  SIMCLR_CHECK_ARG(D > 0, "gcl_orthogonal: D must be > 0");
  if (D > MAXD) {
    set_error("gcl_orthogonal: D=%lld is above the supported %d", (long long)D, MAXD);
    return SIMCLR_ERR_UNSUPPORTED;
  }
  GCL_CHECK_WS("gcl_orthogonal", workspace_bytes, 2 * (size_t)D * D * sizeof(double));
  double* A = (double*)workspace;
  householder_kernel<<<1, QR_THREADS, 0, (cudaStream_t)stream>>>(normal, (int)D, A, A + D * D, W);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_align(const float* z, int64_t B, int64_t D, float lambda_weight, float loss_scaling, float* loss,
                     float* dz, void* stream) {
  SIMCLR_CHECK_ARG(z && loss, "gcl_align: null pointer");
  SIMCLR_CHECK_ARG(B > 0 && D > 0, "gcl_align: need B, D > 0");
  align_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(z, B, (int)D, lambda_weight, loss_scaling, loss, dz);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_lse_forward(const float* z_all, int64_t B, int64_t R, int64_t D, int64_t replica_id, float temperature,
                           float* lse, float* loss, void* workspace, size_t workspace_bytes, void* stream) {
  SIMCLR_CHECK_ARG(z_all && lse && loss && workspace, "gcl_lse_forward: null pointer");
  GCL_CHECK_SHAPE("gcl_lse_forward", B, R, D, replica_id);
  SIMCLR_CHECK_ARG(temperature > 0.f, "gcl_lse_forward: temperature must be > 0");
  GCL_CHECK_WS("gcl_lse_forward", workspace_bytes, lse_ws(B, R, D));
  cudaStream_t st = (cudaStream_t)stream;
  int tps;
  const int splits = pick_splits(B, R, &tps);
  SIMCLR_CHECK_CUDA(cudaFuncSetAttribute(lse_fwd_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (RB + CT) * (MAXD + 1) * 4));
  float* part = (float*)workspace;
  dim3 grid((unsigned)((2 * B + RB - 1) / RB), splits);
  lse_fwd_partial_kernel<<<grid, NT, (size_t)(RB + CT) * (D + 1) * sizeof(float), st>>>(
      z_all, B, R, (int)D, replica_id, 1.f / temperature, part, tps);
  SIMCLR_CHECK_LAUNCH();
  lse_fwd_finalize_kernel<<<(unsigned)((2 * B + 255) / 256), 256, 0, st>>>(part, splits, 2 * B, lse);
  SIMCLR_CHECK_LAUNCH();
  lse_mean_kernel<<<1, 1024, 0, st>>>(lse, 2 * B, (int)D, loss);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_lse_backward(const float* z_all, const float* lse_all, int64_t B, int64_t R, int64_t D,
                            int64_t replica_id, float temperature, float* dz, void* workspace, size_t workspace_bytes,
                            void* stream) {
  SIMCLR_CHECK_ARG(z_all && lse_all && dz && workspace, "gcl_lse_backward: null pointer");
  GCL_CHECK_SHAPE("gcl_lse_backward", B, R, D, replica_id);
  SIMCLR_CHECK_ARG(temperature > 0.f, "gcl_lse_backward: temperature must be > 0");
  GCL_CHECK_WS("gcl_lse_backward", workspace_bytes, lse_ws(B, R, D));
  cudaStream_t st = (cudaStream_t)stream;
  int tps;
  const int splits = pick_splits(B, R, &tps);
  SIMCLR_CHECK_CUDA(cudaFuncSetAttribute(lse_bwd_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         ((RB + CT) * (MAXD + 1) + RB * CT + CT) * 4));
  float* part = (float*)workspace;
  dim3 grid((unsigned)((2 * B + RB - 1) / RB), splits);
  lse_bwd_partial_kernel<<<grid, NT, ((size_t)(RB + CT) * (D + 1) + RB * CT + CT) * sizeof(float), st>>>(
      z_all, lse_all, B, R, (int)D, replica_id, 1.f / temperature, part, tps);
  SIMCLR_CHECK_LAUNCH();
  const int64_t n = 2 * B * D;
  sum_splits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, splits, n, 1.f / temperature, dz);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_sort(const float* x_t, int64_t n, int64_t cols, float* sorted, int32_t* perm, void* stream) {
  SIMCLR_CHECK_ARG(x_t && (sorted || perm), "gcl_sort: null pointer");
  SIMCLR_CHECK_ARG(n > 0 && cols > 0, "gcl_sort: need n, cols > 0");
  if (n > MAX_SORT) {
    set_error("gcl_sort: %lld rows per column is above the supported %d", (long long)n, MAX_SORT);
    return SIMCLR_ERR_UNSUPPORTED;
  }
  return launch_sort(x_t, n, cols, sorted, perm, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int simclr_gcl_swd_forward(const float* z_all, const float* prior, const float* W, int64_t B, int64_t R, int64_t D,
                           float* loss, int32_t* perm, float* diff, void* workspace, size_t workspace_bytes,
                           void* stream) {
  SIMCLR_CHECK_ARG(z_all && prior && W && loss && perm && diff && workspace, "gcl_swd_forward: null pointer");
  GCL_CHECK_SHAPE("gcl_swd_forward", B, R, D, (int64_t)0);
  const int64_t G = R * B, n = 2 * G;
  if (n > MAX_SORT) {
    set_error("gcl_swd_forward: the sliced Wasserstein distance sorts 2*R*B = %lld rows per column, above the "
              "supported %d", (long long)n, MAX_SORT);
    return SIMCLR_ERR_UNSUPPORTED;
  }
  GCL_CHECK_WS("gcl_swd_forward", workspace_bytes, swd_ws(B, R, D));
  cudaStream_t st = (cudaStream_t)stream;
  float* St = (float*)workspace;
  float* Qt = St + n * D;
  double* col_sq = (double*)((char*)workspace + align_up(2 * n * D * sizeof(float)));
  dim3 grid((unsigned)((n + GM - 1) / GM), (unsigned)((D + GN - 1) / GN));
  gemm_kernel<true, false, true><<<grid, 256, 0, st>>>(z_all, W, St, n, (int)D, (int)D, B, G);
  SIMCLR_CHECK_LAUNCH();
  gemm_kernel<false, false, true><<<grid, 256, 0, st>>>(prior, W, Qt, n, (int)D, (int)D, B, G);
  SIMCLR_CHECK_LAUNCH();
  int r = launch_sort(Qt, n, D, Qt, nullptr, nullptr, nullptr, nullptr, st);
  if (r != SIMCLR_OK) return r;
  r = launch_sort(St, n, D, nullptr, perm, Qt, diff, col_sq, st);
  if (r != SIMCLR_OK) return r;
  swd_loss_kernel<<<1, MAXD, 0, st>>>(col_sq, (int)D, n, loss);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_swd_backward(const int32_t* perm, const float* diff, const float* W, int64_t B, int64_t R, int64_t D,
                            int64_t replica_id, float* dz, void* workspace, size_t workspace_bytes, void* stream) {
  SIMCLR_CHECK_ARG(perm && diff && W && dz && workspace, "gcl_swd_backward: null pointer");
  GCL_CHECK_SHAPE("gcl_swd_backward", B, R, D, replica_id);
  const int64_t G = R * B, n = 2 * G;
  SIMCLR_CHECK_ARG(n <= MAX_SORT, "gcl_swd_backward: 2*R*B = %lld above %d", (long long)n, MAX_SORT);
  GCL_CHECK_WS("gcl_swd_backward", workspace_bytes, swd_ws(B, R, D));
  cudaStream_t st = (cudaStream_t)stream;
  float* dS = (float*)workspace;
  const int64_t total = n * D;
  swd_scatter_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(perm, diff, B, G, (int)D, replica_id,
                                                                      (float)(2.0 / ((double)n * (double)D)), dS);
  SIMCLR_CHECK_LAUNCH();
  dim3 grid((unsigned)((2 * B + GM - 1) / GM), (unsigned)((D + GN - 1) / GN));
  gemm_kernel<false, true, false><<<grid, 256, 0, st>>>(dS, W, dz, 2 * B, (int)D, (int)D, B, G);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_gcl_normalize_backward(const float* z, const float* inv_norm, int hidden_norm, int64_t rows, int64_t D,
                                  const float* dz_align, float align_scale, const float* dz_lse, float lse_scale,
                                  const float* dz_swd, float swd_scale, float* dhidden, void* stream) {
  SIMCLR_CHECK_ARG(z && dhidden, "gcl_normalize_backward: null pointer");
  SIMCLR_CHECK_ARG(!hidden_norm || inv_norm, "gcl_normalize_backward: inv_norm required when hidden_norm");
  SIMCLR_CHECK_ARG(rows > 0 && D > 0, "gcl_normalize_backward: need rows, D > 0");
  if (D > MAXD) {
    set_error("gcl_normalize_backward: D=%lld is above the supported %d", (long long)D, MAXD);
    return SIMCLR_ERR_UNSUPPORTED;
  }
  normalize_backward_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      z, inv_norm, hidden_norm, rows, (int)D, dz_align, align_scale, dz_lse, lse_scale, dz_swd, swd_scale, dhidden);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
