// NT-Xent objective kernels (tf2/objective.py:35-89), shared-memory tiled with
// warp-shuffle reductions.  The 2B x 2G similarity matrix is never materialised:
// forward keeps an online log-sum-exp per row, backward recomputes the tiles
// (flash-style) so the only collectives the step needs are the all-gathers of
// z [2B,D] and lse [2B] (SURVEY.md 8e).
#include "common.cuh"

namespace simclr {
namespace {

constexpr int RB = 32;        // local rows per block
constexpr int CT = 64;        // gathered columns per tile
constexpr int NT = 256;       // threads: 8 warps x 4 rows
constexpr int MAXD = 256;

__device__ __forceinline__ int64_t zall_row(int v, int64_t g, int64_t B) {
  // z_all is [R][2][B][D]; global sample g = r*B + i
  const int64_t r = g / B, i = g - r * B;
  return (r * 2 + v) * B + i;
}

__global__ void normalize_kernel(const float* __restrict__ x, int64_t rows, int64_t dim, int hidden_norm,
                                 float* __restrict__ z, float* __restrict__ inv_norm) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * dim;
  float ss = 0.f;
  for (int64_t d = lane; d < dim; d += 32) ss += xr[d] * xr[d];
  ss = warp_sum(ss);
  // tf.math.l2_normalize: x * rsqrt(max(sum(x^2), 1e-12))
  const float inv = hidden_norm ? rsqrtf(fmaxf(ss, 1e-12f)) : 1.f;
  for (int64_t d = lane; d < dim; d += 32) z[row * dim + d] = xr[d] * inv;
  if (lane == 0) inv_norm[row] = inv;
}

__device__ __forceinline__ void load_tile(float* dst, const float* __restrict__ z_all, int64_t first, int count,
                                          int64_t total, int64_t G, int64_t B, int D, int ld, bool columns) {
  // rows [first, first+count) of either the local rows (columns=false: `first`
  // indexes z_all rows directly through `total`-relative mapping done by caller)
  for (int idx = threadIdx.x; idx < count * D; idx += NT) {
    const int r = idx / D, d = idx - r * D;
    const int64_t c = first + r;
    float v = 0.f;
    if (c < total) {
      const int vv = (int)(c / G);
      const int64_t g = c - (int64_t)vv * G;
      v = z_all[zall_row(vv, g, B) * D + d];
    }
    dst[r * ld + d] = v;
  }
  (void)columns;
}

// Forward: per (row block, column split) partial online LSE.
__global__ void __launch_bounds__(NT)
fwd_partial_kernel(const float* __restrict__ z_all, int64_t B, int64_t R, int D, int64_t replica_id,
                   float inv_temp, float* __restrict__ logits_ab, float* __restrict__ part /*[S][2B][2]*/,
                   int tiles_per_split) {
  extern __shared__ float sm[];
  const int ld = D + 1;
  float* q = sm;                 // [RB][ld]
  float* k = sm + RB * ld;       // [CT][ld]
  const int64_t G = R * B, rows = 2 * B, cols = 2 * G;
  const int64_t row0 = (int64_t)blockIdx.x * RB;
  const int split = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // local rows live at global sample replica_id*B + i of each view
  for (int idx = threadIdx.x; idx < RB * D; idx += NT) {
    const int r = idx / D, d = idx - r * D;
    const int64_t lr = row0 + r;
    float v = 0.f;
    if (lr < rows) {
      const int vv = (int)(lr / B);
      const int64_t i = lr - (int64_t)vv * B;
      v = z_all[zall_row(vv, replica_id * B + i, B) * D + d];
    }
    q[r * ld + d] = v;
  }

  float m[4], l[4];
  int rv[4];
  int64_t rg[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    m[j] = -INFINITY; l[j] = 0.f;
    const int64_t lr = row0 + warp * 4 + j;
    rv[j] = (int)(lr / B);
    rg[j] = replica_id * B + (lr - (int64_t)rv[j] * B);
  }

  const int64_t n_tiles = (cols + CT - 1) / CT;
  const int64_t t0 = (int64_t)split * tiles_per_split;
  const int64_t t1 = min(n_tiles, t0 + tiles_per_split);
  for (int64_t t = t0; t < t1; ++t) {
    __syncthreads();
    load_tile(k, z_all, t * CT, CT, cols, G, B, D, ld, true);
    __syncthreads();
    float acc[4][2];
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
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t lr = row0 + warp * 4 + j;
      if (lr >= rows) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t c = t * CT + lane + 32 * h;
        if (c >= cols) continue;
        const int cv = (int)(c / G);
        const int64_t cg = c - (int64_t)cv * G;
        const float s = acc[j][h] * inv_temp;
        if (logits_ab != nullptr && rv[j] == 0 && cv == 1) {
          logits_ab[(lr) * G + cg] = s;           // lr == i for view 0
        }
        if (cv == rv[j] && cg == rg[j]) continue;  // masks * LARGE_NUM: exp underflows to exactly 0
        if (s > m[j]) { l[j] = l[j] * __expf(m[j] - s) + 1.f; m[j] = s; }
        else          { l[j] += __expf(s - m[j]); }
      }
    }
  }
  // merge the 32 per-lane (m,l) pairs of each row
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float mm = warp_max(m[j]);
    float ll = (m[j] == -INFINITY) ? 0.f : l[j] * __expf(m[j] - mm);
    ll = warp_sum(ll);
    const int64_t lr = row0 + warp * 4 + j;
    if (lane == 0 && lr < rows) {
      float* p = part + ((int64_t)split * rows + lr) * 2;
      p[0] = mm; p[1] = ll;
    }
  }
}

__global__ void fwd_finalize_kernel(const float* __restrict__ z_all, const float* __restrict__ part, int splits,
                                    int64_t B, int64_t R, int D, int64_t replica_id, float inv_temp,
                                    float* __restrict__ lse, float* __restrict__ row_loss) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t rows = 2 * B;
  const int64_t lr = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (lr >= rows) return;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, part[((int64_t)s * rows + lr) * 2]);
  float l = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float* p = part + ((int64_t)s * rows + lr) * 2;
    if (p[0] != -INFINITY) l += p[1] * expf(p[0] - m);
  }
  const float L = m + logf(l);
  const int v = (int)(lr / B);
  const int64_t g = replica_id * B + (lr - (int64_t)v * B);
  const float* a = z_all + zall_row(v, g, B) * D;
  const float* b = z_all + zall_row(1 - v, g, B) * D;
  float dot = 0.f;
  for (int d = lane; d < D; d += 32) dot = fmaf(a[d], b[d], dot);
  dot = warp_sum(dot) * inv_temp;
  if (lane == 0) { lse[lr] = L; row_loss[lr] = L - dot; }
}

__global__ void sum_scale_kernel(const float* __restrict__ x, int64_t n, float scale, float* __restrict__ out) {
  __shared__ float sh[32];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += x[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) out[0] = s * scale;
  }
}

// Backward partial: dz_a += sum_b (P_ab + P_ba - 2 Y_ab) z_b over this split's columns.
__global__ void __launch_bounds__(NT)
bwd_partial_kernel(const float* __restrict__ z_all, const float* __restrict__ lse_all, int64_t B, int64_t R,
                   int D, int64_t replica_id, float inv_temp, float* __restrict__ part /*[S][2B][D]*/,
                   int tiles_per_split) {
  extern __shared__ float sm[];
  const int ld = D + 1;
  float* q = sm;                    // [RB][ld]
  float* k = q + RB * ld;           // [CT][ld]
  float* cs = k + CT * ld;          // [RB][CT]
  float* lse_c = cs + RB * CT;      // [CT]
  const int64_t G = R * B, rows = 2 * B, cols = 2 * G;
  const int64_t row0 = (int64_t)blockIdx.x * RB;
  const int split = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int idx = threadIdx.x; idx < RB * D; idx += NT) {
    const int r = idx / D, d = idx - r * D;
    const int64_t lr = row0 + r;
    float v = 0.f;
    if (lr < rows) {
      const int vv = (int)(lr / B);
      v = z_all[zall_row(vv, replica_id * B + (lr - (int64_t)vv * B), B) * D + d];
    }
    q[r * ld + d] = v;
  }
  int rv[4];
  int64_t rg[4];
  float rl[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t lr = row0 + warp * 4 + j;
    rv[j] = (int)(lr / B);
    rg[j] = replica_id * B + (lr - (int64_t)rv[j] * B);
    rl[j] = (lr < rows) ? lse_all[zall_row(rv[j], rg[j], B)] : 0.f;
  }
  constexpr int DJ = MAXD / 32;
  float dz[4][DJ];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < DJ; ++e) dz[j][e] = 0.f;

  const int64_t n_tiles = (cols + CT - 1) / CT;
  const int64_t t0 = (int64_t)split * tiles_per_split;
  const int64_t t1 = min(n_tiles, t0 + tiles_per_split);
  for (int64_t t = t0; t < t1; ++t) {
    __syncthreads();
    load_tile(k, z_all, t * CT, CT, cols, G, B, D, ld, true);
    if (threadIdx.x < CT) {
      const int64_t c = t * CT + threadIdx.x;
      float v = 0.f;
      if (c < cols) {
        const int cv = (int)(c / G);
        v = lse_all[zall_row(cv, c - (int64_t)cv * G, B)];
      }
      lse_c[threadIdx.x] = v;
    }
    __syncthreads();
    float acc[4][2];
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
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t lr = row0 + warp * 4 + j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cl = lane + 32 * h;
        const int64_t c = t * CT + cl;
        float coef = 0.f;
        if (lr < rows && c < cols) {
          const int cv = (int)(c / G);
          const int64_t cg = c - (int64_t)cv * G;
          const bool self = (cv == rv[j] && cg == rg[j]);
          if (!self) {
            const float s = acc[j][h] * inv_temp;
            coef = __expf(s - rl[j]) + __expf(s - lse_c[cl]);
            if (cv != rv[j] && cg == rg[j]) coef -= 2.f;   // positive pair: label in both rows
          }
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
    float* p = part + ((int64_t)split * rows + lr) * D;
#pragma unroll
    for (int e = 0; e < DJ; ++e) {
      const int d = lane + 32 * e;
      if (d < D) p[d] = dz[j][e];
    }
  }
}

__global__ void bwd_finalize_kernel(const float* __restrict__ z_all, const float* __restrict__ part, int splits,
                                    const float* __restrict__ inv_norm, int hidden_norm, int64_t B, int D,
                                    int64_t replica_id, float scale, float* __restrict__ dhidden) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t rows = 2 * B;
  const int64_t lr = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (lr >= rows) return;
  const int v = (int)(lr / B);
  const float* z = z_all + zall_row(v, replica_id * B + (lr - (int64_t)v * B), B) * D;
  float g[MAXD / 32];
  float dot = 0.f;
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    float a = 0.f;
    if (d < D) {
      for (int s = 0; s < splits; ++s) a += part[((int64_t)s * rows + lr) * D + d];
      a *= scale;
      dot = fmaf(a, z[d], dot);
    }
    g[e] = a;
  }
  dot = warp_sum(dot);
  const float inv = inv_norm ? inv_norm[lr] : 1.f;
#pragma unroll
  for (int e = 0; e < MAXD / 32; ++e) {
    const int d = lane + 32 * e;
    if (d < D) {
      // l2-normalise backward: dx = (dz - z (z . dz)) / ||x||   (SURVEY A6)
      dhidden[lr * D + d] = hidden_norm ? (g[e] - z[d] * dot) * inv : g[e];
    }
  }
}

__global__ void labels_kernel(int64_t B, int64_t G, int64_t replica_id, int64_t* __restrict__ labels_idx,
                              float* __restrict__ labels, float* __restrict__ masks) {
  const int64_t i = blockIdx.x;
  const int64_t idx = i + replica_id * B;
  if (labels_idx && threadIdx.x == 0) labels_idx[i] = idx;
  if (labels)
    for (int64_t c = threadIdx.x; c < 2 * G; c += blockDim.x) labels[i * 2 * G + c] = (c == idx) ? 1.f : 0.f;
  if (masks)
    for (int64_t c = threadIdx.x; c < G; c += blockDim.x) masks[i * G + c] = (c == idx) ? 1.f : 0.f;
}

// tf2/metrics.py:23-36; one warp per row, then a single-block mean.
__global__ void metrics_rows_kernel(const float* __restrict__ logits, int64_t B, int64_t G, int64_t replica_id,
                                    float* __restrict__ acc_row, float* __restrict__ ent_row) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (i >= B) return;
  const float* x = logits + i * G;
  float m = -INFINITY; int64_t am = 0;
  for (int64_t c = lane; c < G; c += 32) if (x[c] > m) { m = x[c]; am = c; }
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int64_t oa = __shfl_xor_sync(0xffffffffu, am, o);
    if (om > m || (om == m && oa < am)) { m = om; am = oa; }   // first max, like tf.argmax
  }
  float l = 0.f;
  for (int64_t c = lane; c < G; c += 32) l += expf(x[c] - m);
  l = warp_sum(l);
  float e = 0.f;
  for (int64_t c = lane; c < G; c += 32) { const float p = expf(x[c] - m) / l; e += p * logf(p + 1e-8f); }
  e = warp_sum(e);
  if (lane == 0) { acc_row[i] = (am == i + replica_id * B) ? 1.f : 0.f; ent_row[i] = -e; }
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

}  // namespace
}  // namespace simclr

using namespace simclr;

extern "C" {

int simclr_ntxent_normalize(const float* hidden, int64_t rows, int64_t dim, int hidden_norm, float* z,
                            float* inv_norm, void* stream) {
  SIMCLR_CHECK_ARG(hidden && z && inv_norm, "ntxent_normalize: null pointer");
  SIMCLR_CHECK_ARG(rows >= 0 && dim > 0, "ntxent_normalize: bad shape rows=%lld dim=%lld", (long long)rows, (long long)dim);
  if (rows == 0) return SIMCLR_OK;
  const int warps = 8;
  normalize_kernel<<<(unsigned)((rows + warps - 1) / warps), warps * 32, 0, (cudaStream_t)stream>>>(
      hidden, rows, dim, hidden_norm, z, inv_norm);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

size_t simclr_ntxent_workspace_bytes(int64_t B, int64_t R, int64_t D) {
  if (B <= 0 || R <= 0 || D <= 0) return 0;
  int tps;
  const int splits = pick_splits(B, R, &tps);
  const size_t bwd = (size_t)splits * 2 * B * D * sizeof(float);
  const size_t fwd = (size_t)splits * 2 * B * 2 * sizeof(float);
  return (bwd > fwd ? bwd : fwd) + 2 * (size_t)B * sizeof(float) * 2;
}

int simclr_ntxent_forward(const float* z_all, int64_t B, int64_t R, int64_t D, int64_t replica_id,
                          float temperature, float* logits_ab, float* lse, float* row_loss, float* loss,
                          void* workspace, size_t workspace_bytes, void* stream) {
  SIMCLR_CHECK_ARG(z_all && lse && row_loss && loss && workspace, "ntxent_forward: null pointer");
  SIMCLR_CHECK_ARG(B > 0 && R > 0 && D > 0 && D <= MAXD, "ntxent_forward: need B,R>0 and 0<D<=%d (got B=%lld R=%lld D=%lld)", MAXD, (long long)B, (long long)R, (long long)D);
  SIMCLR_CHECK_ARG(replica_id >= 0 && replica_id < R, "ntxent_forward: replica_id %lld out of [0,%lld)", (long long)replica_id, (long long)R);
  SIMCLR_CHECK_ARG(temperature > 0.f, "ntxent_forward: temperature must be > 0");
  if (workspace_bytes < simclr_ntxent_workspace_bytes(B, R, D)) {
    set_error("ntxent_forward: workspace too small (%zu < %zu)", workspace_bytes, simclr_ntxent_workspace_bytes(B, R, D));
    return SIMCLR_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int tps;
  const int splits = pick_splits(B, R, &tps);
  const size_t smem = (size_t)(RB + CT) * (D + 1) * sizeof(float);
  // a per-device attribute: set on every call (a process may drive more than one GPU)
  SIMCLR_CHECK_CUDA(cudaFuncSetAttribute(fwd_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (RB + CT) * (MAXD + 1) * 4));
  float* part = (float*)workspace;
  dim3 grid((unsigned)((2 * B + RB - 1) / RB), splits);
  fwd_partial_kernel<<<grid, NT, smem, st>>>(z_all, B, R, (int)D, replica_id, 1.f / temperature, logits_ab, part, tps);
  SIMCLR_CHECK_LAUNCH();
  fwd_finalize_kernel<<<(unsigned)((2 * B + 7) / 8), 256, 0, st>>>(z_all, part, splits, B, R, (int)D, replica_id,
                                                                    1.f / temperature, lse, row_loss);
  SIMCLR_CHECK_LAUNCH();
  sum_scale_kernel<<<1, 1024, 0, st>>>(row_loss, 2 * B, 1.f / (float)B, loss);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_ntxent_labels(int64_t B, int64_t R, int64_t replica_id, int64_t* labels_idx, float* labels,
                         float* masks, void* stream) {
  SIMCLR_CHECK_ARG(B > 0 && R > 0 && replica_id >= 0 && replica_id < R, "ntxent_labels: bad B/R/replica_id");
  labels_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(B, R * B, replica_id, labels_idx, labels, masks);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_ntxent_backward(const float* z_all, const float* lse_all, const float* inv_norm, int hidden_norm,
                           int64_t B, int64_t R, int64_t D, int64_t replica_id, float temperature,
                           float grad_scale, float* dhidden, void* workspace, size_t workspace_bytes,
                           void* stream) {
  SIMCLR_CHECK_ARG(z_all && lse_all && dhidden && workspace, "ntxent_backward: null pointer");
  SIMCLR_CHECK_ARG(!hidden_norm || inv_norm, "ntxent_backward: inv_norm required when hidden_norm");
  SIMCLR_CHECK_ARG(B > 0 && R > 0 && D > 0 && D <= MAXD, "ntxent_backward: need B,R>0 and 0<D<=%d", MAXD);
  SIMCLR_CHECK_ARG(replica_id >= 0 && replica_id < R, "ntxent_backward: replica_id out of range");
  SIMCLR_CHECK_ARG(temperature > 0.f, "ntxent_backward: temperature must be > 0");
  if (workspace_bytes < simclr_ntxent_workspace_bytes(B, R, D)) {
    set_error("ntxent_backward: workspace too small");
    return SIMCLR_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int tps;
  const int splits = pick_splits(B, R, &tps);
  const size_t smem = ((size_t)(RB + CT) * (D + 1) + RB * CT + CT) * sizeof(float);
  SIMCLR_CHECK_CUDA(cudaFuncSetAttribute(bwd_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         ((RB + CT) * (MAXD + 1) + RB * CT + CT) * 4));
  float* part = (float*)workspace;
  dim3 grid((unsigned)((2 * B + RB - 1) / RB), splits);
  bwd_partial_kernel<<<grid, NT, smem, st>>>(z_all, lse_all, B, R, (int)D, replica_id, 1.f / temperature, part, tps);
  SIMCLR_CHECK_LAUNCH();
  bwd_finalize_kernel<<<(unsigned)((2 * B + 7) / 8), 256, 0, st>>>(z_all, part, splits, inv_norm, hidden_norm, B, (int)D,
                                                                    replica_id, grad_scale / temperature, dhidden);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_contrast_metrics(const float* logits_ab, int64_t B, int64_t G, int64_t replica_id, float* out,
                            void* stream) {
  SIMCLR_CHECK_ARG(logits_ab && out && B > 0 && G > 0, "contrast_metrics: bad args");
  // out needs 2 + 2*B floats: [acc, entropy, acc_row[B], ent_row[B]]
  cudaStream_t st = (cudaStream_t)stream;
  float* acc_row = out + 2;
  float* ent_row = out + 2 + B;
  metrics_rows_kernel<<<(unsigned)((B + 7) / 8), 256, 0, st>>>(logits_ab, B, G, replica_id, acc_row, ent_row);
  SIMCLR_CHECK_LAUNCH();
  sum_scale_kernel<<<1, 1024, 0, st>>>(acc_row, B, 1.f / (float)B, out);
  sum_scale_kernel<<<1, 1024, 0, st>>>(ent_row, B, 1.f / (float)B, out + 1);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
