// BatchNorm family (tf2/resnet.py:31-78; SURVEY.md A4).  All HBM-bound:
// 16-byte vector loads, per-thread fp32 partials, block tree in shared memory,
// one fp64 partial per channel per block, added in block order.  Tensors are [rows][C] views of
// NHWC activations; C % 8 == 0.
#include "common.cuh"

namespace simclr {
namespace {

constexpr int BT = 256;

template <typename T> __device__ __forceinline__ void load8(const T* p, float* f);
template <> __device__ __forceinline__ void load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  Vec16<__nv_bfloat16> v; v.load(p); v.unpack(f);
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float* f);
template <> __device__ __forceinline__ void store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) {
  Vec16<__nv_bfloat16> v; v.pack(f); v.store(p);
}

// Eight consecutive channels kept in their storage format until they are consumed, so that
// several rows of loads can be in flight per thread without eight fp32 registers per load.
template <typename T> struct Raw8;
template <> struct Raw8<float> {
  float4 a, b;
  __device__ __forceinline__ void ld(const float* p) { a = reinterpret_cast<const float4*>(p)[0]; b = reinterpret_cast<const float4*>(p)[1]; }
  __device__ __forceinline__ void to(float* f) const { f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w; }
};
template <> struct Raw8<__nv_bfloat16> {
  Vec16<__nv_bfloat16> v;
  __device__ __forceinline__ void ld(const __nv_bfloat16* p) { v.load(p); }
  __device__ __forceinline__ void to(float* f) const { v.unpack(f); }
};

// Thread layout shared by the reduction kernels: P threads span the
// channel vectors of a row (power of two <= 256), 256/P "row lanes".
struct RedLayout { int P, row_lanes, col_iters; };
inline RedLayout red_layout(int64_t C) {
  const int cvecs = (int)(C / 8);
  int P = 1;
  while (P * 2 <= cvecs && P * 2 <= BT) P *= 2;
  RedLayout l; l.P = P; l.row_lanes = BT / P; l.col_iters = (cvecs + P - 1) / P;
  return l;
}

// mode 0: stats (sum x, sum x^2).  mode 1: bwd reduce (sum dz, sum dz*xhat) with
// optional in-place dz <- (dz + dz2) * [z > 0].  mode 2: bwd reduce of a BN+ReLU
// without residual: the mask [scale*y + shift > 0] is recomputed from y (a2 = scale,
// zmask = shift, both fp32 [C]); dz is neither re-read from a mask tensor nor written.
// mode 3: mode 1 with the ReLU mask of the block tail as ONE BIT per element (byte i = the 8 channels
// of 16-byte vector i, written by bn_apply_kernel) instead of the output tensor z: 1/16 of the bytes.
// mode 4: mode 3 for the tail of a PROJECTION block: the masked gradient is also the gradient w.r.t. the
// output of the shortcut's BatchNorm (no ReLU), whose reduction (conv output y2, mean2, rstd2 -> sums2) is
// taken in the same pass instead of re-reading the gradient.
// The kernels are HBM-latency bound: each thread keeps 4 (modes 0, 2) or 2 (mode 1) rows of
// 16-byte loads in flight, two 256-thread CTAs per SM.
template <typename T, typename Ty, int MODE>
__global__ void __launch_bounds__(BT, 2)
bn_reduce_kernel(T* __restrict__ a, const void* __restrict__ a2_, const void* __restrict__ zmask_,
                 const Ty* __restrict__ y, int64_t rows, int C, int P, int rows_per_block,
                 const float* __restrict__ mean, const float* __restrict__ rstd, double* __restrict__ sums,
                 const Ty* __restrict__ y2 = nullptr, const float* __restrict__ mean2 = nullptr,
                 const float* __restrict__ rstd2 = nullptr, double* __restrict__ sums2 = nullptr) {
  extern __shared__ double sh[];  // [row_lanes][P*8][2]
  constexpr bool BITS = MODE == 3 || MODE == 4;      // mode 4: mode 3 for a projection block, see below
  const T* __restrict__ a2 = MODE == 2 ? nullptr : (const T*)a2_;
  const T* __restrict__ zmask = (MODE == 2 || BITS) ? nullptr : (const T*)zmask_;
  const uint8_t* __restrict__ zbits = BITS ? (const uint8_t*)zmask_ : nullptr;
  const int tx = threadIdx.x % P, ty = threadIdx.x / P;
  const int row_lanes = BT / P;
  const int cvecs = C / 8;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t r1 = min(rows, r0 + rows_per_block);
  const int64_t lane_step = (int64_t)row_lanes * C;
  for (int cv = tx; cv < cvecs + (P - 1 - ((cvecs - 1) % P)); cv += P) {   // uniform trip count across tx
    const bool active = cv < cvecs;
    // Per-thread sums are fp32 (a few hundred rows at most), everything from the block tree on is fp64.  The
    // forward statistics (mode 0) additionally fold into fp64 every few groups; doing that in the backward
    // modes costs ~13% of their bandwidth (fp32->fp64 converts are slow) for no measurable accuracy.
    float s0[8], s1[8], s2[8];
    double d0[8], d1[8], d2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s0[i] = s1[i] = s2[i] = 0.f; d0[i] = d1[i] = d2[i] = 0.0; }
    auto fold = [&]() {
#pragma unroll
      for (int i = 0; i < 8; ++i) { d0[i] += (double)s0[i]; d1[i] += (double)s1[i]; s0[i] = 0.f; s1[i] = 0.f; }
      if (MODE == 4) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { d2[i] += (double)s2[i]; s2[i] = 0.f; }
      }
    };
    int groups = 0;
    auto fold_some = [&]() { if ((++groups & 3) == 0) fold(); };   // every 4th group: fp32->fp64 converts are slow
    if (active) {
      int64_t r = r0 + ty;
      if (MODE == 0) {
        // Shifted sums: u = x - pivot with pivot = row 0 of the tensor (any sample of the channel).  The
        // fp32 squares are then O(variance) instead of O(mean^2), so var = E[x^2] - mean^2 keeps its digits
        // for nearly constant channels (|mean| >> sigma); the shift is undone in fp64 by the block tree.
        float pv[8];
        { Raw8<T> q0; q0.ld(a + (int64_t)cv * 8); q0.to(pv); }
        auto acc = [&](const Raw8<T>& q) {
          float v[8]; q.to(v);
#pragma unroll
          for (int i = 0; i < 8; ++i) { const float u = v[i] - pv[i]; s0[i] += u; s1[i] = fmaf(u, u, s1[i]); }
        };
        for (; r + 3 * row_lanes < r1; r += 4 * row_lanes) {
          const T* p = a + r * C + (int64_t)cv * 8;
          Raw8<T> q[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) q[u].ld(p + u * lane_step);
#pragma unroll
          for (int u = 0; u < 4; ++u) acc(q[u]);
          fold_some();
        }
        for (; r < r1; r += row_lanes) { Raw8<T> q; q.ld(a + r * C + (int64_t)cv * 8); acc(q); }
        fold();
      } else if (MODE == 2) {
        float mu[8], msc[8], msh[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          mu[i] = mean[cv * 8 + i];
          msc[i] = ((const float*)a2_)[cv * 8 + i];
          msh[i] = ((const float*)zmask_)[cv * 8 + i];
        }
        // s1 accumulates dz*(y - mean); rstd is applied once at the end
        auto acc = [&](const Raw8<T>& qg, const Raw8<Ty>& qy) {
          float g[8], yy[8]; qg.to(g); qy.to(yy);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float gm = fmaf(yy[i], msc[i], msh[i]) > 0.f ? g[i] : 0.f;
            s0[i] += gm;
            s1[i] = fmaf(gm, yy[i] - mu[i], s1[i]);
          }
        };
        for (; r + 3 * row_lanes < r1; r += 4 * row_lanes) {
          const int64_t off = r * C + (int64_t)cv * 8;
          Raw8<T> qg[4]; Raw8<Ty> qy[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) { qg[u].ld(a + off + u * lane_step); qy[u].ld(y + off + u * lane_step); }
#pragma unroll
          for (int u = 0; u < 4; ++u) acc(qg[u], qy[u]);
        }
        for (; r < r1; r += row_lanes) {
          const int64_t off = r * C + (int64_t)cv * 8;
          Raw8<T> qg; Raw8<Ty> qy; qg.ld(a + off); qy.ld(y + off); acc(qg, qy);
        }
        fold();
#pragma unroll
        for (int i = 0; i < 8; ++i) d1[i] *= (double)rstd[cv * 8 + i];
      } else {
        float mu[8], mu2[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { mu[i] = mean[cv * 8 + i]; mu2[i] = MODE == 4 ? mean2[cv * 8 + i] : 0.f; }
        const bool has2 = a2 != nullptr, hasz = zmask != nullptr;
        auto acc = [&](int64_t off, const Raw8<T>& qv, const Raw8<T>& qw, const Raw8<T>& qz, const Raw8<Ty>& qy, unsigned bits,
                       const Raw8<Ty>& qy2) {
          float v[8], yy[8]; qv.to(v); qy.to(yy);
          if (has2) {
            float w[8]; qw.to(w);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] += w[i];
          }
          if (hasz) {
            float z[8]; qz.to(z);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = (z[i] > 0.f) ? v[i] : 0.f;
          }
          if (BITS) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = ((bits >> i) & 1u) ? v[i] : 0.f;
          }
          if (has2 || hasz || BITS) {
            store8<T>(a + off, v);
            // keep the sums consistent with what phase 2 will read back
            if (sizeof(T) == 2) {
#pragma unroll
              for (int i = 0; i < 8; ++i) v[i] = to_f<T>(from_f<T>(v[i]));
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) { s0[i] += v[i]; s1[i] = fmaf(v[i], yy[i] - mu[i], s1[i]); }
          if (MODE == 4) {
            float y2v[8]; qy2.to(y2v);
#pragma unroll
            for (int i = 0; i < 8; ++i) s2[i] = fmaf(v[i], y2v[i] - mu2[i], s2[i]);
          }
        };
        for (; r + row_lanes < r1; r += 2 * row_lanes) {
          const int64_t off = r * C + (int64_t)cv * 8;
          Raw8<T> qv[2], qw[2], qz[2]; Raw8<Ty> qy[2], qy2[2]; unsigned qb[2] = {0u, 0u};
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            qv[u].ld(a + off + u * lane_step);
            if (has2) qw[u].ld(a2 + off + u * lane_step); else qw[u] = qv[u];
            if (hasz) qz[u].ld(zmask + off + u * lane_step); else qz[u] = qv[u];
            if (BITS) qb[u] = zbits[(off + u * lane_step) >> 3];
            qy[u].ld(y + off + u * lane_step);
            if (MODE == 4) qy2[u].ld(y2 + off + u * lane_step); else qy2[u] = qy[u];
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) acc(off + u * lane_step, qv[u], qw[u], qz[u], qy[u], qb[u], qy2[u]);
        }
        for (; r < r1; r += row_lanes) {
          const int64_t off = r * C + (int64_t)cv * 8;
          Raw8<T> qv, qw, qz; Raw8<Ty> qy, qy2;
          qv.ld(a + off);
          if (has2) qw.ld(a2 + off); else qw = qv;
          if (hasz) qz.ld(zmask + off); else qz = qv;
          const unsigned qb = BITS ? (unsigned)zbits[off >> 3] : 0u;
          qy.ld(y + off);
          if (MODE == 4) qy2.ld(y2 + off); else qy2 = qy;
          acc(off, qv, qw, qz, qy, qb, qy2);
        }
        fold();
#pragma unroll
        for (int i = 0; i < 8; ++i) d1[i] *= (double)rstd[cv * 8 + i];
        if (MODE == 4) {
#pragma unroll
          for (int i = 0; i < 8; ++i) d2[i] *= (double)rstd2[cv * 8 + i];
        }
      }
    }
    // block tree over row lanes
    __syncthreads();
    double* mine = sh + ((size_t)ty * P + tx) * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) { mine[i] = d0[i]; mine[8 + i] = d1[i]; }
    __syncthreads();
    // P*16 values to reduce over row_lanes; thread t handles value index t, t+BT, ...
    for (int idx = threadIdx.x; idx < P * 16; idx += BT) {
      const int px = idx / 16, e = idx % 16;
      const int c8 = (cv - tx + px);
      if (c8 >= cvecs) continue;
      double acc = 0.0;
      for (int l = 0; l < row_lanes; ++l) acc += sh[((size_t)l * P + px) * 16 + e];
      const int ch = c8 * 8 + (e & 7);
      if (MODE == 0) {         // undo the pivot shift: sum x = S0 + n p,  sum x^2 = S1 + 2 p S0 + n p^2
        const double pvt = (double)to_f<T>(a[ch]);
        const double n = (double)(r1 - r0);
        if (e < 8) {
          acc += n * pvt;
        } else {
          double a0 = 0.0;
          for (int l = 0; l < row_lanes; ++l) a0 += sh[((size_t)l * P + px) * 16 + e - 8];
          acc += 2.0 * pvt * a0 + n * pvt * pvt;
        }
      }
      sums[(size_t)blockIdx.x * 2 * C + (e >> 3) * C + ch] = acc;       // this block's partial (summed in block order)
    }
    if (MODE == 4) {        // second tree: (sum dz, sum dz*xhat2) of the shortcut's BatchNorm
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 8; ++i) mine[8 + i] = d2[i];
      __syncthreads();
      for (int idx = threadIdx.x; idx < P * 16; idx += BT) {
        const int px = idx / 16, e = idx % 16;
        const int c8 = (cv - tx + px);
        if (c8 >= cvecs) continue;
        double acc = 0.0;
        for (int l = 0; l < row_lanes; ++l) acc += sh[((size_t)l * P + px) * 16 + e];
        sums2[(size_t)blockIdx.x * 2 * C + (e >> 3) * C + c8 * 8 + (e & 7)] = acc;
      }
    }
  }
}

__global__ void bn_finalize_kernel(const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum,
                                   float* __restrict__ mm, float* __restrict__ mv, float* __restrict__ mean,
                                   float* __restrict__ rstd, float* __restrict__ scale, float* __restrict__ shift,
                                   int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = sums[c] / count;
  double var = sums[C + c] / count - m * m;      // biased variance (SyncBN form, A4)
  if (var < 0.0) var = 0.0;
  const float mf = (float)m, vf = (float)var;
  const float r = rsqrtf(vf + eps);
  const float g = gamma ? gamma[c] : 1.f;
  const float b = beta ? beta[c] : 0.f;
  const float sc = g * r;
  mean[c] = mf; rstd[c] = r; scale[c] = sc; shift[c] = b - mf * sc;
  if (mm) mm[c] = mm[c] - (mm[c] - mf) * (1.f - momentum);
  if (mv) mv[c] = mv[c] - (mv[c] - vf) * (1.f - momentum);
}

// The host sizes the grid so that gridDim*BT*8 is a multiple of C whenever it can: a thread then
// stays on one block of 8 channels for the whole grid-stride loop and keeps its per-channel
// coefficients in registers (reloading them per vector makes these kernels L1-bound).
template <typename Ty, typename Tz>
__global__ void __launch_bounds__(BT)
bn_apply_kernel(const Ty* __restrict__ y, const Tz* __restrict__ res, Tz* __restrict__ z, int64_t nvec, int C,
                const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                uint8_t* __restrict__ mask_bits) {
  const int64_t stride = (int64_t)gridDim.x * BT;
  int64_t i = (int64_t)blockIdx.x * BT + threadIdx.x;
  const bool fixed_c = (stride * 8) % C == 0;
  float sc[8], sh[8];
  if (fixed_c) { const int c = (int)((i * 8) % C); load8<float>(scale + c, sc); load8<float>(shift + c, sh); }
  auto body = [&](int64_t off, const Raw8<Ty>& qy, const Raw8<Tz>& qr) {
    float v[8]; qy.to(v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaf(v[k], sc[k], sh[k]);
    if (res != nullptr) {
      float r[8]; qr.to(r);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] += r[k];
    }
    if (relu) {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
    }
    store8<Tz>(z + off, v);
    if (mask_bits != nullptr) {          // [z > 0] of the stored (rounded) outputs, one bit per element
      unsigned b = 0u;
#pragma unroll
      for (int k = 0; k < 8; ++k) b |= (to_f<Tz>(from_f<Tz>(v[k])) > 0.f ? 1u : 0u) << k;
      mask_bits[off >> 3] = (uint8_t)b;
    }
  };
  if (fixed_c) {
    for (; i + stride < nvec; i += 2 * stride) {
      const int64_t o0 = i * 8, o1 = (i + stride) * 8;
      Raw8<Ty> q0, q1; Raw8<Tz> r0, r1;
      q0.ld(y + o0); q1.ld(y + o1);
      if (res != nullptr) { r0.ld(res + o0); r1.ld(res + o1); }
      body(o0, q0, r0); body(o1, q1, r1);
    }
  }
  for (; i < nvec; i += stride) {
    const int64_t off = i * 8;
    if (!fixed_c) { const int c = (int)(off % C); load8<float>(scale + c, sc); load8<float>(shift + c, sh); }
    Raw8<Ty> q; Raw8<Tz> r;
    q.ld(y + off);
    if (res != nullptr) r.ld(res + off);
    body(off, q, r);
  }
}

// dy = k1*dz + k2*y + k3 per channel, with
//   k1 = gamma*rstd, k2 = -gamma*rstd^2*S1/M, k3 = gamma*rstd*(mean*rstd*S1/M - S0/M)
// (== gamma*rstd*(dz - S0/M - xhat*S1/M), SURVEY A4).
__global__ void bn_bwd_coef_kernel(const float* __restrict__ mean, const float* __restrict__ rstd,
                                   const float* __restrict__ gamma, const double* __restrict__ sums,
                                   const double* __restrict__ sums_local, double inv_count,
                                   float* __restrict__ coef, float* __restrict__ dgamma,
                                   float* __restrict__ dbeta, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double r = rstd[c], mu = mean[c], g = gamma ? gamma[c] : 1.0;
  const double a = sums[c] * inv_count, b = sums[C + c] * inv_count;
  coef[c] = (float)(g * r);
  coef[C + c] = (float)(-g * r * r * b);
  coef[2 * C + c] = (float)(g * r * (mu * r * b - a));
  if (dbeta) dbeta[c] = (float)sums_local[c];
  if (dgamma) dgamma[c] = (float)sums_local[C + c];
}

// mask_scale / mask_shift non-null: dz is the gradient w.r.t. relu(scale*y + shift) and the
// mask is recomputed here instead of being applied to dz in memory beforehand.
template <typename T, typename Ty, typename Td, bool MASK>
__global__ void __launch_bounds__(BT, MASK ? 3 : 4)      // MASK keeps 40 coefficient registers: 64 registers spilled
bn_bwd_apply_kernel(const T* __restrict__ dz, const Ty* __restrict__ y, Td* __restrict__ dy, int64_t nvec, int C,
                    const float* __restrict__ coef, const float* __restrict__ mask_scale,
                    const float* __restrict__ mask_shift) {
  const int64_t stride = (int64_t)gridDim.x * BT;
  int64_t i = (int64_t)blockIdx.x * BT + threadIdx.x;
  const bool fixed_c = (stride * 8) % C == 0;
  float k1[8], k2[8], k3[8], ms[8], mh[8];
  auto load_coef = [&](int c) {
    load8<float>(coef + c, k1); load8<float>(coef + C + c, k2); load8<float>(coef + 2 * C + c, k3);
    if (MASK) { load8<float>(mask_scale + c, ms); load8<float>(mask_shift + c, mh); }
  };
  if (fixed_c) load_coef((int)((i * 8) % C));
  auto body = [&](int64_t off, const Raw8<T>& qg, const Raw8<Ty>& qy) {
    float g[8], yy[8], o[8]; qg.to(g); qy.to(yy);
    if (MASK) {
#pragma unroll
      for (int k = 0; k < 8; ++k) g[k] = fmaf(yy[k], ms[k], mh[k]) > 0.f ? g[k] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaf(k1[k], g[k], fmaf(k2[k], yy[k], k3[k]));
    store8<Td>(dy + off, o);
  };
  if (fixed_c) {
    for (; i + stride < nvec; i += 2 * stride) {
      const int64_t o0 = i * 8, o1 = (i + stride) * 8;
      Raw8<T> g0, g1; Raw8<Ty> y0, y1;
      g0.ld(dz + o0); g1.ld(dz + o1); y0.ld(y + o0); y1.ld(y + o1);
      body(o0, g0, y0); body(o1, g1, y1);
    }
  }
  for (; i < nvec; i += stride) {
    const int64_t off = i * 8;
    if (!fixed_c) load_coef((int)(off % C));
    Raw8<T> qg; Raw8<Ty> qy; qg.ld(dz + off); qy.ld(y + off);
    body(off, qg, qy);
  }
}

// Tail of a PROJECTION block in one pass: z = relu(scale*y + shift + zs) with zs = the shortcut's BatchNorm output
// scale2*y2 + shift2 rounded to the activation type exactly as the unfused chain would have stored it -- which
// it now never is.  Writes the ReLU bit mask like bn_apply_kernel.
template <typename Ty, typename Tz>
__global__ void __launch_bounds__(BT)
bn_apply2_tail_kernel(const Ty* __restrict__ y, const Ty* __restrict__ y2, Tz* __restrict__ z, int64_t nvec, int C,
                      const float* __restrict__ scale, const float* __restrict__ shift,
                      const float* __restrict__ scale2, const float* __restrict__ shift2,
                      uint8_t* __restrict__ mask_bits) {
  const int64_t stride = (int64_t)gridDim.x * BT;
  int64_t i = (int64_t)blockIdx.x * BT + threadIdx.x;
  const bool fixed_c = (stride * 8) % C == 0;
  float sc[8], sh[8], sc2[8], sh2[8];
  auto load_coef = [&](int c) {
    load8<float>(scale + c, sc); load8<float>(shift + c, sh); load8<float>(scale2 + c, sc2); load8<float>(shift2 + c, sh2);
  };
  if (fixed_c) load_coef((int)((i * 8) % C));
  auto body = [&](int64_t off, const Raw8<Ty>& qy, const Raw8<Ty>& qy2) {
    float v[8], w[8]; qy.to(v); qy2.to(w);
    unsigned b = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float zs = to_f<Tz>(from_f<Tz>(fmaf(w[k], sc2[k], sh2[k])));
      v[k] = fmaxf(fmaf(v[k], sc[k], sh[k]) + zs, 0.f);
      b |= (to_f<Tz>(from_f<Tz>(v[k])) > 0.f ? 1u : 0u) << k;
    }
    store8<Tz>(z + off, v);
    mask_bits[off >> 3] = (uint8_t)b;
  };
  if (fixed_c) {
    for (; i + stride < nvec; i += 2 * stride) {
      const int64_t o0 = i * 8, o1 = (i + stride) * 8;
      Raw8<Ty> q0, q1, r0, r1;
      q0.ld(y + o0); q1.ld(y + o1); r0.ld(y2 + o0); r1.ld(y2 + o1);
      body(o0, q0, r0); body(o1, q1, r1);
    }
  }
  for (; i < nvec; i += stride) {
    const int64_t off = i * 8;
    if (!fixed_c) load_coef((int)(off % C));
    Raw8<Ty> q, r; q.ld(y + off); r.ld(y2 + off);
    body(off, q, r);
  }
}

// Backward of the same tail: the masked gradient dz feeds two BatchNorms (the block's last one and the shortcut's);
// dy = k1*dz + k2*y + k3 and dy2 = m1*dz + m2*y2 + m3 in one pass over dz.
template <typename T, typename Ty, typename Td>
__global__ void __launch_bounds__(BT, 2)       // 48 coefficient registers per thread: no 64-register cap here
bn_bwd_apply2_kernel(const T* __restrict__ dz, const Ty* __restrict__ y, const Ty* __restrict__ y2, Td* __restrict__ dy,
                     Td* __restrict__ dy2, int64_t nvec, int C, const float* __restrict__ coef,
                     const float* __restrict__ coef2) {
  const int64_t stride = (int64_t)gridDim.x * BT;
  int64_t i = (int64_t)blockIdx.x * BT + threadIdx.x;
  const bool fixed_c = (stride * 8) % C == 0;
  float k1[8], k2[8], k3[8], m1[8], m2[8], m3[8];
  auto load_coef = [&](int c) {
    load8<float>(coef + c, k1); load8<float>(coef + C + c, k2); load8<float>(coef + 2 * C + c, k3);
    load8<float>(coef2 + c, m1); load8<float>(coef2 + C + c, m2); load8<float>(coef2 + 2 * C + c, m3);
  };
  if (fixed_c) load_coef((int)((i * 8) % C));
  auto body = [&](int64_t off, const Raw8<T>& qg, const Raw8<Ty>& qy, const Raw8<Ty>& qy2) {
    float g[8], a[8], o[8]; qg.to(g); qy.to(a);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaf(k1[k], g[k], fmaf(k2[k], a[k], k3[k]));
    store8<Td>(dy + off, o);
    qy2.to(a);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaf(m1[k], g[k], fmaf(m2[k], a[k], m3[k]));
    store8<Td>(dy2 + off, o);
  };
  if (fixed_c) {
    for (; i + stride < nvec; i += 2 * stride) {
      const int64_t o0 = i * 8, o1 = (i + stride) * 8;
      Raw8<T> g0, g1; Raw8<Ty> a0, a1, b0, b1;
      g0.ld(dz + o0); g1.ld(dz + o1); a0.ld(y + o0); a1.ld(y + o1); b0.ld(y2 + o0); b1.ld(y2 + o1);
      body(o0, g0, a0, b0); body(o1, g1, a1, b1);
    }
  }
  for (; i < nvec; i += stride) {
    const int64_t off = i * 8;
    if (!fixed_c) load_coef((int)(off % C));
    Raw8<T> qg; Raw8<Ty> qy, qy2;
    qg.ld(dz + off); qy.ld(y + off); qy2.ld(y2 + off);
    body(off, qg, qy, qy2);
  }
}

// grid for the element-wise kernels: as many CTAs as fit, rounded down so that gridDim*BT*8 is a
// multiple of C (see bn_apply_kernel)
inline unsigned ew_grid_c(int64_t nvec, int64_t C) {
  int64_t b = (nvec + BT - 1) / BT;
  const int64_t cap = (int64_t)num_sms() * 16;
  if (b > cap) b = cap;
  int64_t q = C, per = (int64_t)BT * 8;          // need b * per % C == 0  <=>  b % (C / gcd(C, per)) == 0
  int64_t x = q, yv = per;
  while (yv) { const int64_t t = x % yv; x = yv; yv = t; }
  const int64_t m = q / x;
  if (b >= m) b = b / m * m;
  if (b < 1) b = 1;
  return (unsigned)b;
}

template <typename T, typename Ty, int MODE>
int launch_reduce(void* a, const void* a2, const void* zmask, const void* y, int64_t rows, int64_t C,
                  const float* mean, const float* rstd, double* sums, cudaStream_t st, const void* y2 = nullptr,
                  const float* mean2 = nullptr, const float* rstd2 = nullptr, double* sums2 = nullptr) {
  const RedLayout l = red_layout(C);
  int64_t nblocks = (rows + l.row_lanes * 8 - 1) / (l.row_lanes * 8);
  // 2 CTAs of 256 threads are resident per SM (__launch_bounds__(BT, 2)): one wave of fat blocks.  Every block ends
  // with one fp64 partial per column; the partials are added in block order (the same bits every run), so fewer
  // blocks also mean less to add.
  const int64_t cap = (int64_t)num_sms() * 2;
  if (nblocks > cap) nblocks = cap;
  if (nblocks < 1) nblocks = 1;
  const int rows_per_block = (int)((rows + nblocks - 1) / nblocks);
  nblocks = (rows + rows_per_block - 1) / rows_per_block;
  const size_t smem = (size_t)BT * 16 * sizeof(double);
  if (!accumulate_prezeroed()) {
    cudaError_t e = cudaMemsetAsync(sums, 0, 2 * C * sizeof(double), st);
    if (e != cudaSuccess) { set_error("bn reduce memset: %s", cudaGetErrorString(e)); return (int)e; }
    if (sums2) {
      e = cudaMemsetAsync(sums2, 0, 2 * C * sizeof(double), st);
      if (e != cudaSuccess) { set_error("bn reduce memset: %s", cudaGetErrorString(e)); return (int)e; }
    }
  }
  const int64_t part = 2 * C;                     // doubles per block partial
  const int nsets = sums2 ? 2 : 1;
  double* ws = nullptr;
  { int rc = scratch_alloc(&ws, (size_t)nsets * nblocks * part * sizeof(double), st); if (rc) return rc; }
  double* ws2 = sums2 ? ws + nblocks * part : nullptr;
  cudaError_t e = cudaMemsetAsync(ws, 0, (size_t)nsets * nblocks * part * sizeof(double), st);
  if (e == cudaSuccess) {
    bn_reduce_kernel<T, Ty, MODE><<<(unsigned)nblocks, BT, smem, st>>>(
        (T*)a, a2, zmask, (const Ty*)y, rows, (int)C, l.P, rows_per_block, mean, rstd, ws, (const Ty*)y2, mean2, rstd2, ws2);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) { set_error("bn reduce launch: %s", cudaGetErrorString(e)); scratch_free(ws, st); return (int)e; }
  int rc = run_sum_partials_f64(ws, part, sums, part, (int)nblocks, st);
  if (!rc && sums2) rc = run_sum_partials_f64(ws2, part, sums2, part, (int)nblocks, st);
  const int rf = scratch_free(ws, st);
  return rc ? rc : rf;
}

}  // namespace
}  // namespace simclr

using namespace simclr;
typedef __nv_bfloat16 bf16;

extern "C" {

int simclr_bn_stats(const void* x, int dtype, int64_t rows, int64_t C, double* sums, void* stream) {
  SIMCLR_CHECK_ARG(x && sums, "bn_stats: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_stats: need rows>0 and C%%8==0 (rows=%lld C=%lld)", (long long)rows, (long long)C);
  SIMCLR_CHECK_ARG(aligned16(x), "bn_stats: x must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32) return launch_reduce<float, float, 0>((void*)x, nullptr, nullptr, nullptr, rows, C, nullptr, nullptr, sums, st);
  if (dtype == SIMCLR_BF16) return launch_reduce<bf16, bf16, 0>((void*)x, nullptr, nullptr, nullptr, rows, C, nullptr, nullptr, sums, st);
  set_error("bn_stats: unknown dtype %d", dtype);
  return SIMCLR_ERR_INVALID_ARG;
}

int simclr_bn_finalize(const double* sums, double count, const float* gamma, const float* beta, float eps,
                       float momentum, float* moving_mean, float* moving_var, float* mean, float* rstd,
                       float* scale, float* shift, int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(sums && mean && rstd && scale && shift, "bn_finalize: null pointer");
  SIMCLR_CHECK_ARG(C > 0 && count > 0, "bn_finalize: bad C/count");
  bn_finalize_kernel<<<(unsigned)((C + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      sums, count, gamma, beta, eps, momentum, moving_mean, moving_var, mean, rstd, scale, shift, (int)C);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

static int bn_apply_impl(const void* y, int y_dtype, const void* residual, void* z, int z_dtype, int64_t rows,
                         int64_t C, const float* scale, const float* shift, int relu, uint8_t* mask_bits, void* stream) {
  SIMCLR_CHECK_ARG(y && z && scale && shift, "bn_apply: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_apply: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(y) && aligned16(z) && aligned16(residual), "bn_apply: pointers must be 16-byte aligned");
  const int64_t nvec = rows * C / 8;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = ew_grid_c(nvec, C);
  if (y_dtype == SIMCLR_F32 && z_dtype == SIMCLR_F32)
    bn_apply_kernel<float, float><<<grid, BT, 0, st>>>((const float*)y, (const float*)residual, (float*)z, nvec, (int)C, scale, shift, relu, mask_bits);
  else if (y_dtype == SIMCLR_BF16 && z_dtype == SIMCLR_BF16)
    bn_apply_kernel<bf16, bf16><<<grid, BT, 0, st>>>((const bf16*)y, (const bf16*)residual, (bf16*)z, nvec, (int)C, scale, shift, relu, mask_bits);
  else if (y_dtype == SIMCLR_F32 && z_dtype == SIMCLR_BF16)
    bn_apply_kernel<float, bf16><<<grid, BT, 0, st>>>((const float*)y, (const bf16*)residual, (bf16*)z, nvec, (int)C, scale, shift, relu, mask_bits);
  else if (y_dtype == SIMCLR_BF16 && z_dtype == SIMCLR_F32)
    bn_apply_kernel<bf16, float><<<grid, BT, 0, st>>>((const bf16*)y, (const float*)residual, (float*)z, nvec, (int)C, scale, shift, relu, mask_bits);
  else { set_error("bn_apply: unknown dtypes %d/%d", y_dtype, z_dtype); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bn_apply(const void* y, int y_dtype, const void* residual, void* z, int z_dtype, int64_t rows,
                    int64_t C, const float* scale, const float* shift, int relu, void* stream) {
  return bn_apply_impl(y, y_dtype, residual, z, z_dtype, rows, C, scale, shift, relu, nullptr, stream);
}

int simclr_bn_apply_relu_mask(const void* y, int y_dtype, const void* residual, void* z, int z_dtype, int64_t rows,
                              int64_t C, const float* scale, const float* shift, uint8_t* relu_mask_bits,
                              void* stream) {
  SIMCLR_CHECK_ARG(relu_mask_bits, "bn_apply_relu_mask: null mask");
  return bn_apply_impl(y, y_dtype, residual, z, z_dtype, rows, C, scale, shift, 1, relu_mask_bits, stream);
}

int simclr_bn_bwd_reduce_bits(void* dz, const void* dz2, const uint8_t* relu_mask_bits, int dtype, const void* y,
                              int y_dtype, int64_t rows, int64_t C, const float* mean, const float* rstd,
                              double* sums, void* stream) {
  SIMCLR_CHECK_ARG(dz && relu_mask_bits && y && mean && rstd && sums, "bn_bwd_reduce_bits: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_reduce_bits: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(dz2) && aligned16(y), "bn_bwd_reduce_bits: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32)
    return launch_reduce<float, float, 3>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16)
    return launch_reduce<bf16, bf16, 3>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_F32)
    return launch_reduce<bf16, float, 3>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_BF16)
    return launch_reduce<float, bf16, 3>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st);
  set_error("bn_bwd_reduce_bits: unknown dtypes");
  return SIMCLR_ERR_INVALID_ARG;
}

int simclr_bn_bwd_reduce(void* dz, const void* dz2, const void* relu_mask_z, int dtype, const void* y,
                         int y_dtype, int64_t rows, int64_t C, const float* mean, const float* rstd,
                         double* sums, void* stream) {
  SIMCLR_CHECK_ARG(dz && y && mean && rstd && sums, "bn_bwd_reduce: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_reduce: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(dz2) && aligned16(relu_mask_z) && aligned16(y), "bn_bwd_reduce: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32)
    return launch_reduce<float, float, 1>(dz, dz2, relu_mask_z, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16)
    return launch_reduce<bf16, bf16, 1>(dz, dz2, relu_mask_z, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_F32)
    return launch_reduce<bf16, float, 1>(dz, dz2, relu_mask_z, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_BF16)
    return launch_reduce<float, bf16, 1>(dz, dz2, relu_mask_z, y, rows, C, mean, rstd, sums, st);
  set_error("bn_bwd_reduce: unknown dtypes");
  return SIMCLR_ERR_INVALID_ARG;
}

int simclr_bn_bwd_relu_reduce(const void* dz, int dtype, const void* y, int y_dtype, int64_t rows, int64_t C,
                              const float* mean, const float* rstd, const float* scale, const float* shift,
                              double* sums, void* stream) {
  SIMCLR_CHECK_ARG(dz && y && mean && rstd && scale && shift && sums, "bn_bwd_relu_reduce: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_relu_reduce: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(y), "bn_bwd_relu_reduce: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32)
    return launch_reduce<float, float, 2>((void*)dz, scale, shift, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16)
    return launch_reduce<bf16, bf16, 2>((void*)dz, scale, shift, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_F32)
    return launch_reduce<bf16, float, 2>((void*)dz, scale, shift, y, rows, C, mean, rstd, sums, st);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_BF16)
    return launch_reduce<float, bf16, 2>((void*)dz, scale, shift, y, rows, C, mean, rstd, sums, st);
  set_error("bn_bwd_relu_reduce: unknown dtypes");
  return SIMCLR_ERR_INVALID_ARG;
}

static int launch_bwd_apply(const void* dz, int dtype, const void* y, int y_dtype, void* dy, int dy_dtype, int64_t rows,
                            int64_t C, const float* coef_ws, const float* mask_scale, const float* mask_shift,
                            cudaStream_t st) {
  const int64_t nvec = rows * C / 8;
  const unsigned grid = ew_grid_c(nvec, C);
#define LAUNCH(T, Ty, Td)                                                                                          \
  do {                                                                                                             \
    if (mask_scale) bn_bwd_apply_kernel<T, Ty, Td, true><<<grid, BT, 0, st>>>((const T*)dz, (const Ty*)y, (Td*)dy, nvec, (int)C, coef_ws, mask_scale, mask_shift); \
    else bn_bwd_apply_kernel<T, Ty, Td, false><<<grid, BT, 0, st>>>((const T*)dz, (const Ty*)y, (Td*)dy, nvec, (int)C, coef_ws, nullptr, nullptr); \
  } while (0)
  const int key = dtype * 4 + y_dtype * 2 + dy_dtype;
  switch (key) {
    case 0: LAUNCH(float, float, float); break;
    case 1: LAUNCH(float, float, bf16); break;
    case 2: LAUNCH(float, bf16, float); break;
    case 3: LAUNCH(float, bf16, bf16); break;
    case 4: LAUNCH(bf16, float, float); break;
    case 5: LAUNCH(bf16, float, bf16); break;
    case 6: LAUNCH(bf16, bf16, float); break;
    case 7: LAUNCH(bf16, bf16, bf16); break;
    default: set_error("bn_bwd_apply: unknown dtypes"); return SIMCLR_ERR_INVALID_ARG;
  }
#undef LAUNCH
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bn_bwd_apply(const void* dz, int dtype, const void* y, int y_dtype, void* dy, int dy_dtype,
                        int64_t rows, int64_t C, const float* mean, const float* rstd, const float* gamma,
                        const double* sums, const double* sums_local, double count, float* dgamma,
                        float* dbeta, float* coef_ws, const float* mask_scale, const float* mask_shift,
                        void* stream) {
  SIMCLR_CHECK_ARG((mask_scale == nullptr) == (mask_shift == nullptr), "bn_bwd_apply: mask_scale and mask_shift go together");
  SIMCLR_CHECK_ARG(dz && y && dy && mean && rstd && sums && sums_local && coef_ws, "bn_bwd_apply: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0 && count > 0, "bn_bwd_apply: bad shape");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(y) && aligned16(dy), "bn_bwd_apply: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  SIMCLR_CHECK_ARG(aligned16(coef_ws), "bn_bwd_apply: coef_ws alignment");
  bn_bwd_coef_kernel<<<(unsigned)((C + 127) / 128), 128, 0, st>>>(mean, rstd, gamma, sums, sums_local, 1.0 / count,
                                                                   coef_ws, dgamma, dbeta, (int)C);
  SIMCLR_CHECK_LAUNCH();
  return launch_bwd_apply(dz, dtype, y, y_dtype, dy, dy_dtype, rows, C, coef_ws, mask_scale, mask_shift, st);
}

int simclr_bn_bwd_coef(const float* mean, const float* rstd, const float* gamma, const double* sums,
                       const double* sums_local, double count, float* coef, float* dgamma, float* dbeta, int64_t C,
                       void* stream) {
  SIMCLR_CHECK_ARG(mean && rstd && sums && sums_local && coef && C > 0 && count > 0, "bn_bwd_coef: bad arguments");
  bn_bwd_coef_kernel<<<(unsigned)((C + 127) / 128), 128, 0, (cudaStream_t)stream>>>(mean, rstd, gamma, sums, sums_local,
                                                                                   1.0 / count, coef, dgamma, dbeta, (int)C);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bn_bwd_apply_coef(const void* dz, int dtype, const void* y, int y_dtype, void* dy, int dy_dtype,
                             int64_t rows, int64_t C, const float* coef, const float* mask_scale,
                             const float* mask_shift, void* stream) {
  SIMCLR_CHECK_ARG((mask_scale == nullptr) == (mask_shift == nullptr), "bn_bwd_apply_coef: mask_scale and mask_shift go together");
  SIMCLR_CHECK_ARG(dz && y && dy && coef, "bn_bwd_apply_coef: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_apply_coef: bad shape");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(y) && aligned16(dy) && aligned16(coef), "bn_bwd_apply_coef: alignment");
  return launch_bwd_apply(dz, dtype, y, y_dtype, dy, dy_dtype, rows, C, coef, mask_scale, mask_shift, (cudaStream_t)stream);
}

/* Projection-block tail (see bn_apply2_tail_kernel / bn_reduce_kernel mode 4 / bn_bwd_apply2_kernel). */
int simclr_bn_apply2_relu_mask(const void* y, const void* y2, int y_dtype, void* z, int z_dtype, int64_t rows, int64_t C,
                               const float* scale, const float* shift, const float* scale2, const float* shift2,
                               uint8_t* relu_mask_bits, void* stream) {
  SIMCLR_CHECK_ARG(y && y2 && z && scale && shift && scale2 && shift2 && relu_mask_bits, "bn_apply2_relu_mask: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_apply2_relu_mask: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(y) && aligned16(y2) && aligned16(z), "bn_apply2_relu_mask: pointers must be 16-byte aligned");
  const int64_t nvec = rows * C / 8;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = ew_grid_c(nvec, C);
  if (y_dtype == SIMCLR_F32 && z_dtype == SIMCLR_F32)
    bn_apply2_tail_kernel<float, float><<<grid, BT, 0, st>>>((const float*)y, (const float*)y2, (float*)z, nvec, (int)C, scale, shift, scale2, shift2, relu_mask_bits);
  else if (y_dtype == SIMCLR_BF16 && z_dtype == SIMCLR_BF16)
    bn_apply2_tail_kernel<bf16, bf16><<<grid, BT, 0, st>>>((const bf16*)y, (const bf16*)y2, (bf16*)z, nvec, (int)C, scale, shift, scale2, shift2, relu_mask_bits);
  else { set_error("bn_apply2_relu_mask: unsupported dtypes %d/%d", y_dtype, z_dtype); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bn_bwd_reduce2_bits(void* dz, const void* dz2, const uint8_t* relu_mask_bits, int dtype, const void* y,
                               const void* y2, int y_dtype, int64_t rows, int64_t C, const float* mean,
                               const float* rstd, const float* mean2, const float* rstd2, double* sums, double* sums2,
                               void* stream) {
  SIMCLR_CHECK_ARG(dz && relu_mask_bits && y && y2 && mean && rstd && mean2 && rstd2 && sums && sums2, "bn_bwd_reduce2_bits: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_reduce2_bits: need rows>0 and C%%8==0");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(dz2) && aligned16(y) && aligned16(y2), "bn_bwd_reduce2_bits: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32)
    return launch_reduce<float, float, 4>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st, y2, mean2, rstd2, sums2);
  if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16)
    return launch_reduce<bf16, bf16, 4>(dz, dz2, relu_mask_bits, y, rows, C, mean, rstd, sums, st, y2, mean2, rstd2, sums2);
  set_error("bn_bwd_reduce2_bits: unsupported dtypes");
  return SIMCLR_ERR_INVALID_ARG;
}

int simclr_bn_bwd_apply2_coef(const void* dz, int dtype, const void* y, const void* y2, int y_dtype, void* dy, void* dy2,
                              int dy_dtype, int64_t rows, int64_t C, const float* coef, const float* coef2, void* stream) {
  SIMCLR_CHECK_ARG(dz && y && y2 && dy && dy2 && coef && coef2, "bn_bwd_apply2_coef: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "bn_bwd_apply2_coef: bad shape");
  SIMCLR_CHECK_ARG(aligned16(dz) && aligned16(y) && aligned16(y2) && aligned16(dy) && aligned16(dy2), "bn_bwd_apply2_coef: alignment");
  const int64_t nvec = rows * C / 8;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = ew_grid_c(nvec, C);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32 && dy_dtype == SIMCLR_F32)
    bn_bwd_apply2_kernel<float, float, float><<<grid, BT, 0, st>>>((const float*)dz, (const float*)y, (const float*)y2, (float*)dy, (float*)dy2, nvec, (int)C, coef, coef2);
  else if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16 && dy_dtype == SIMCLR_BF16)
    bn_bwd_apply2_kernel<bf16, bf16, bf16><<<grid, BT, 0, st>>>((const bf16*)dz, (const bf16*)y, (const bf16*)y2, (bf16*)dy, (bf16*)dy2, nvec, (int)C, coef, coef2);
  else { set_error("bn_bwd_apply2_coef: unsupported dtypes"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
