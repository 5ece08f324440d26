// Pooling kernels: MaxPooling2D(3,2,'SAME') (tf2/resnet.py:605-611, SURVEY A3:
// TF-SAME pads after first) and the global mean over H,W (tf2/resnet.py:693-696).
#include "common.cuh"

namespace simclr {
namespace {

// BNRELU: x is the conv output; relu(scale*x + shift), rounded to T exactly like the BatchNorm apply kernel would have
// stored it, is what the window maximum is taken over -- the stem's BN+ReLU output is never materialised
// (tf2/resnet.py:593-611: conv -> BatchNormRelu -> MaxPooling2D).
template <typename T, bool BNRELU>
__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint8_t* __restrict__ argmax, int64_t total,
                   int H, int W, int C, int Ho, int Wo, int pb_h, int pb_w, const float* __restrict__ scale,
                   const float* __restrict__ shift) {
  constexpr int V = Vec16<T>::N;
  const int cv = C / V;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    float sc[V], sh[V];
    if (BNRELU) {
#pragma unroll
      for (int i = 0; i < V; ++i) { sc[i] = scale[c + i]; sh[i] = shift[c + i]; }
    }
    int64_t p = idx / cv;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int64_t n = p / Ho;
    float best[V]; int arg[V];
#pragma unroll
    for (int i = 0; i < V; ++i) { best[i] = -INFINITY; arg[i] = 0; }
    bool first = true;
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int h = ho * 2 - pb_h + dh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int w = wo * 2 - pb_w + dw;
        if (w < 0 || w >= W) continue;
        Vec16<T> v; v.load(x + (((n * H + h) * W + w) * (int64_t)C + c));
        float f[V]; v.unpack(f);
        if (BNRELU) {
#pragma unroll
          for (int i = 0; i < V; ++i) f[i] = to_f<T>(from_f<T>(fmaxf(fmaf(f[i], sc[i], sh[i]), 0.f)));
        }
#pragma unroll
        for (int i = 0; i < V; ++i) {
          // first maximum in window scan order wins (matches TF / torch argmax routing)
          if (first || f[i] > best[i]) { best[i] = f[i]; arg[i] = dh * 3 + dw; }
        }
        first = false;
      }
    }
    Vec16<T> o; o.pack(best);
    const int64_t ooff = ((n * Ho + ho) * Wo + wo) * (int64_t)C + c;
    o.store(y + ooff);
    // V argmax codes packed into one 4/8-byte store (ooff is a multiple of V)
    if (V == 8) {
      uint64_t pk = 0;
#pragma unroll
      for (int i = 0; i < V; ++i) pk |= (uint64_t)(arg[i] & 0xff) << (8 * i);
      *reinterpret_cast<uint64_t*>(argmax + ooff) = pk;
    } else {
      uint32_t pk = 0;
#pragma unroll
      for (int i = 0; i < V; ++i) pk |= (uint32_t)(arg[i] & 0xff) << (8 * i);
      *reinterpret_cast<uint32_t*>(argmax + ooff) = pk;
    }
  }
}

// One thread per 2x2 block of input pixels and V channels.  With stride 2 and a 3x3 window the
// block's pixels lie in at most 2x2 pooling windows (ho, wo in {hb - 1 + pb, hb + pb}): their dy and
// argmax vectors are loaded once and routed to the four pixels.
template <typename T>
__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ argmax, T* __restrict__ dx,
                   int64_t total, int H, int W, int C, int Ho, int Wo, int pb_h, int pb_w) {
  constexpr int V = Vec16<T>::N;
  const int cv = C / V;
  const int Hb = (H + 1) / 2, Wb = (W + 1) / 2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    int64_t p = idx / cv;
    const int wb = (int)(p % Wb); p /= Wb;
    const int hb = (int)(p % Hb);
    const int64_t n = p / Hb;
    float g[2][2][V];
    uint64_t am[2][2];
    bool live[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int ho = hb - 1 + pb_h + i, wo = wb - 1 + pb_w + j;
        live[i][j] = ho >= 0 && ho < Ho && wo >= 0 && wo < Wo;
        am[i][j] = 0;
        if (live[i][j]) {
          const int64_t ooff = ((n * Ho + ho) * Wo + wo) * (int64_t)C + c;
          Vec16<T> v; v.load(dy + ooff); v.unpack(g[i][j]);
          if (V == 8) am[i][j] = *reinterpret_cast<const uint64_t*>(argmax + ooff);
          else am[i][j] = *reinterpret_cast<const uint32_t*>(argmax + ooff);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) g[i][j][k] = 0.f;
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int h = 2 * hb + a;
      if (h >= H) continue;
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int w = 2 * wb + b;
        if (w >= W) continue;
        float acc[V];
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int dh = a + 2 - pb_h - 2 * i;        // h + pb_h - 2*ho with ho = hb - 1 + pb_h + i
          if (dh < 0 || dh > 2) continue;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int dw = b + 2 - pb_w - 2 * j;
            if (dw < 0 || dw > 2 || !live[i][j]) continue;
            const int code = dh * 3 + dw;
#pragma unroll
            for (int k = 0; k < V; ++k) if ((int)((am[i][j] >> (8 * k)) & 0xff) == code) acc[k] += g[i][j][k];
          }
        }
        Vec16<T> o; o.pack(acc);
        o.store(dx + (((n * H + h) * W + w) * (int64_t)C + c));
      }
    }
  }
}

// MaxPooling2D backward fused with the backward pass of the BatchNorm + ReLU in front of it: the gradient w.r.t.
// the BN output, dz = maxpool_bwd(d [+ d2]) * [scale*y + shift > 0], is formed on the fly from the pooled-size
// gradient(s), the argmax codes and the conv output y, and never written.  PHASE 0 accumulates the BatchNorm
// reduction (sum dz, sum dz*(y - mean)) * rstd into `sums` [2][C]; PHASE 1 writes dy = k1*dz + k2*y + k3.
// Roundings are those of the unfused chain (bf16 sum d + d2, bf16 dz).  Thread -> channel block is fixed
// (gridDim*256 is a multiple of C/V), so PHASE 0 keeps per-thread partial sums in registers.
template <typename T, int PHASE>
__global__ void __launch_bounds__(256)
maxpool_bn_bwd_kernel(const T* __restrict__ d, const T* __restrict__ d2, const uint8_t* __restrict__ argmax,
                      const T* __restrict__ y, T* __restrict__ dy_out, int64_t total, int H, int W, int C, int Ho, int Wo,
                      int pb_h, int pb_w, const float* __restrict__ mean, const float* __restrict__ rstd,
                      const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ coef,
                      double* __restrict__ sums) {
  constexpr int V = Vec16<T>::N;
  const int cv = C / V;
  const int Hb = (H + 1) / 2, Wb = (W + 1) / 2;
  const int c = (int)((blockIdx.x * 256 + threadIdx.x) % cv) * V;       // fixed for the whole grid-stride loop
  float sc[V], sh[V], mu[V], k1[V], k2[V], k3[V], s0[V], s1[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    sc[i] = scale[c + i]; sh[i] = shift[c + i]; s0[i] = 0.f; s1[i] = 0.f;
    if (PHASE == 0) mu[i] = mean[c + i];
    else { k1[i] = coef[c + i]; k2[i] = coef[C + c + i]; k3[i] = coef[2 * C + c + i]; }
  }
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = idx / cv;
    const int wb = (int)(p % Wb); p /= Wb;
    const int hb = (int)(p % Hb);
    const int64_t n = p / Hb;
    float g[2][2][V];
    uint64_t am[2][2];
    bool live[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int ho = hb - 1 + pb_h + i, wo = wb - 1 + pb_w + j;
        live[i][j] = ho >= 0 && ho < Ho && wo >= 0 && wo < Wo;
        am[i][j] = 0;
        if (live[i][j]) {
          const int64_t ooff = ((n * Ho + ho) * Wo + wo) * (int64_t)C + c;
          Vec16<T> v; v.load(d + ooff); v.unpack(g[i][j]);
          if (d2 != nullptr) {
            Vec16<T> v2; v2.load(d2 + ooff); float g2[V]; v2.unpack(g2);
#pragma unroll
            for (int k = 0; k < V; ++k) g[i][j][k] = to_f<T>(from_f<T>(g[i][j][k] + g2[k]));
          }
          if (V == 8) am[i][j] = *reinterpret_cast<const uint64_t*>(argmax + ooff);
          else am[i][j] = *reinterpret_cast<const uint32_t*>(argmax + ooff);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) g[i][j][k] = 0.f;
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int h = 2 * hb + a;
      if (h >= H) continue;
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int w = 2 * wb + b;
        if (w >= W) continue;
        float acc[V];
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int dh = a + 2 - pb_h - 2 * i;
          if (dh < 0 || dh > 2) continue;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int dw = b + 2 - pb_w - 2 * j;
            if (dw < 0 || dw > 2 || !live[i][j]) continue;
            const int code = dh * 3 + dw;
#pragma unroll
            for (int k = 0; k < V; ++k) if ((int)((am[i][j] >> (8 * k)) & 0xff) == code) acc[k] += g[i][j][k];
          }
        }
        const int64_t off = ((n * H + h) * W + w) * (int64_t)C + c;
        Vec16<T> vy; vy.load(y + off); float yy[V]; vy.unpack(yy);
        float o[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float dz = fmaf(yy[k], sc[k], sh[k]) > 0.f ? to_f<T>(from_f<T>(acc[k])) : 0.f;
          if (PHASE == 0) { s0[k] += dz; s1[k] = fmaf(dz, yy[k] - mu[k], s1[k]); }
          else o[k] = fmaf(k1[k], dz, fmaf(k2[k], yy[k], k3[k]));
        }
        if (PHASE == 1) { Vec16<T> vo; vo.pack(o); vo.store(dy_out + off); }
      }
    }
  }
  if (PHASE == 0) {
    // threads t and t' with t % cv == t' % cv hold partial sums of the same channels: fold in shared memory,
    // then one fp64 atomic per channel per block
    __shared__ float sh_s[256][2 * V + 1];
#pragma unroll
    for (int k = 0; k < V; ++k) { sh_s[threadIdx.x][k] = s0[k]; sh_s[threadIdx.x][V + k] = s1[k]; }
    __syncthreads();
    for (int e = threadIdx.x; e < cv * 2 * V; e += 256) {
      const int j = e / (2 * V), q = e % (2 * V);
      double t = 0.0;
      for (int r = j; r < 256; r += cv) t += (double)sh_s[r][q];
      const int ch = j * V + (q % V);
      if (q < V) sums[(size_t)blockIdx.x * 2 * C + ch] = t;              // this block's partial (summed in block order)
      else sums[(size_t)blockIdx.x * 2 * C + C + ch] = t * (double)rstd[ch];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// bf16 specialisations of the fused stem kernels.  The generic templates above are issue-bound (~700 thread
// instructions per 16-byte vector: per-channel fp32 compares and selects); these keep the eight channels of a
// vector as four packed bf16x2 registers and do the window routing with packed compares and byte permutes.
// Arithmetic and rounding points are those of the generic kernels (z = bf16(relu(fma(y, scale, shift))),
// g = bf16(d + d2), first maximum in scan order wins).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ __nv_bfloat162 as_bf2(uint32_t u) { return *reinterpret_cast<__nv_bfloat162*>(&u); }
__device__ __forceinline__ uint32_t as_u32(__nv_bfloat162 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ uint32_t sel32(uint32_t m, uint32_t a, uint32_t b) { return (a & m) | (b & ~m); }

// Forward.  Also stores ysel = the conv output y at the argmax tap, so that the BatchNorm reduction of the backward
// pass can run over the pooled tensor (a quarter of the elements) instead of re-reading y.
// All nine loads of a window are issued unconditionally (clamped addresses, out-of-image taps masked afterwards):
// with the loads inside the bounds branches the compiler serialises them and the kernel is latency-bound.
__global__ void __launch_bounds__(256)
maxpool_bnrelu_fwd_bf16_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                               uint8_t* __restrict__ argmax, __nv_bfloat16* __restrict__ ysel, int64_t total,
                               int H, int W, int C, int Ho, int Wo, int pb_h, int pb_w,
                               const float* __restrict__ scale, const float* __restrict__ shift) {
  const int cv = C / 8;
  const int c = (int)((blockIdx.x * 256 + threadIdx.x) % cv) * 8;       // gridDim*256 is a multiple of cv
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sc[i] = scale[c + i]; sh[i] = shift[c + i]; }
  // 32-bit index arithmetic throughout (64-bit divisions cost ~100 instructions each; the host checks the sizes)
  const unsigned npix = (unsigned)(total / cv), qstep = gridDim.x * 256u / (unsigned)cv;
  for (unsigned q = (blockIdx.x * 256u + threadIdx.x) / (unsigned)cv; q < npix; q += qstep) {
    const unsigned wo_u = q % (unsigned)Wo, t_u = q / (unsigned)Wo;
    const int wo = (int)wo_u, ho = (int)(t_u % (unsigned)Ho);
    const int n = (int)(t_u / (unsigned)Ho);
    uint4 v[9];
    uint32_t ok[9];
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      const int h = ho * 2 - pb_h + dh;
      const int hc = min(max(h, 0), H - 1);
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int w = wo * 2 - pb_w + dw;
        const int wc = min(max(w, 0), W - 1);
        ok[dh * 3 + dw] = (h == hc && w == wc) ? 0xffffffffu : 0u;
        v[dh * 3 + dw] = *reinterpret_cast<const uint4*>(x + ((int64_t)((n * H + hc) * W + wc) * C + c));
      }
    }
    uint32_t best[4], arg[4], ys[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { best[i] = 0xff80ff80u; arg[i] = 0u; ys[i] = 0u; }   // -inf: the first live tap wins
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const uint32_t r[4] = {v[t].x, v[t].y, v[t].z, v[t].w};
      const uint32_t code2 = (uint32_t)t * 0x00010001u;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float lo = fmaxf(fmaf(__uint_as_float(r[i] << 16), sc[2 * i], sh[2 * i]), 0.f);
        const float hi = fmaxf(fmaf(__uint_as_float(r[i] & 0xffff0000u), sc[2 * i + 1], sh[2 * i + 1]), 0.f);
        const __nv_bfloat162 z2 = __floats2bfloat162_rn(lo, hi);
        const uint32_t m = __hgt2_mask(z2, as_bf2(best[i])) & ok[t];
        best[i] = sel32(m, as_u32(z2), best[i]);
        arg[i] = sel32(m, code2, arg[i]);
        ys[i] = sel32(m, r[i], ys[i]);
      }
    }
    const int64_t ooff = (int64_t)q * C + c;
    *reinterpret_cast<uint4*>(out + ooff) = make_uint4(best[0], best[1], best[2], best[3]);
    if (ysel != nullptr) *reinterpret_cast<uint4*>(ysel + ooff) = make_uint4(ys[0], ys[1], ys[2], ys[3]);
    // one code byte per channel: low bytes of the 16-bit lanes
    *reinterpret_cast<uint2*>(argmax + ooff) = make_uint2(__byte_perm(arg[0], arg[1], 0x6420), __byte_perm(arg[2], arg[3], 0x6420));
  }
}

// Backward, BatchNorm reduction over the POOLED tensor: sum dz = sum over windows of g * [z(argmax pixel) > 0] and
// sum dz*(y - mean) likewise with y = ysel (each window routes its gradient to exactly one pixel).  Differs from
// the per-pixel formulation only in that a pixel selected by several windows contributes the unrounded sum of
// their gradients.  Reads 3 pooled-size tensors instead of 2 + the 4x larger conv output.
__global__ void __launch_bounds__(256)
maxpool_bn_bwd_reduce_pooled_bf16_kernel(const __nv_bfloat16* __restrict__ d, const __nv_bfloat16* __restrict__ d2,
                                         const __nv_bfloat16* __restrict__ ysel, int64_t total, int C,
                                         const float* __restrict__ mean, const float* __restrict__ rstd,
                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                         double* __restrict__ sums) {
  const int cv = C / 8;
  const int c = (int)((blockIdx.x * 256 + threadIdx.x) % cv) * 8;
  float sc[8], sh[8], mu[8], s0[8], s1[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sc[i] = scale[c + i]; sh[i] = shift[c + i]; mu[i] = mean[c + i]; s0[i] = 0.f; s1[i] = 0.f; }
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += 2 * step) {
    // two vectors in flight per thread
    uint4 vd[2], v2[2], vy[2];
    bool on[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int64_t j = idx + u * step;
      on[u] = j < total;
      if (on[u]) {
        vd[u] = *reinterpret_cast<const uint4*>(d + j * 8);
        if (d2 != nullptr) v2[u] = *reinterpret_cast<const uint4*>(d2 + j * 8);
        vy[u] = *reinterpret_cast<const uint4*>(ysel + j * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (!on[u]) continue;
      const uint32_t a[4] = {vd[u].x, vd[u].y, vd[u].z, vd[u].w};
      const uint32_t b[4] = {v2[u].x, v2[u].y, v2[u].z, v2[u].w};
      const uint32_t yv[4] = {vy[u].x, vy[u].y, vy[u].z, vy[u].w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t g = a[i];
        if (d2 != nullptr) g = as_u32(__hadd2(as_bf2(a[i]), as_bf2(b[i])));
        const float g0 = __uint_as_float(g << 16), g1 = __uint_as_float(g & 0xffff0000u);
        const float y0 = __uint_as_float(yv[i] << 16), y1 = __uint_as_float(yv[i] & 0xffff0000u);
        const float m0 = fmaf(y0, sc[2 * i], sh[2 * i]) > 0.f ? g0 : 0.f;
        const float m1 = fmaf(y1, sc[2 * i + 1], sh[2 * i + 1]) > 0.f ? g1 : 0.f;
        s0[2 * i] += m0; s1[2 * i] = fmaf(m0, y0 - mu[2 * i], s1[2 * i]);
        s0[2 * i + 1] += m1; s1[2 * i + 1] = fmaf(m1, y1 - mu[2 * i + 1], s1[2 * i + 1]);
      }
    }
  }
  __shared__ float sh_s[256][17];
#pragma unroll
  for (int k = 0; k < 8; ++k) { sh_s[threadIdx.x][k] = s0[k]; sh_s[threadIdx.x][8 + k] = s1[k]; }
  __syncthreads();
  for (int e = threadIdx.x; e < cv * 16; e += 256) {
    const int j = e / 16, q = e % 16;
    double t = 0.0;
    for (int r = j; r < 256; r += cv) t += (double)sh_s[r][q];
    const int ch = j * 8 + (q % 8);
    if (q < 8) sums[(size_t)blockIdx.x * 2 * C + ch] = t;                // this block's partial (summed in block order)
    else sums[(size_t)blockIdx.x * 2 * C + C + ch] = t * (double)rstd[ch];
  }
}

// Backward, apply: one thread per 2x2 block of conv-output pixels and 8 channels (see maxpool_bwd_kernel).  The
// window -> pixel routing is a packed compare of the argmax codes (expanded to 16-bit lanes) with the code the pixel
// has in that window, an AND and a packed add per channel pair.  The SAME-padding offsets are template parameters so
// that the routing is branch-free, and every load is unconditional (clamped address, dead windows zeroed afterwards).
template <int PBH, int PBW>
__global__ void __launch_bounds__(256)
maxpool_bn_bwd_apply_bf16_kernel(const __nv_bfloat16* __restrict__ d, const __nv_bfloat16* __restrict__ d2,
                                 const uint8_t* __restrict__ argmax, const __nv_bfloat16* __restrict__ y,
                                 __nv_bfloat16* __restrict__ dy_out, int64_t total, int H, int W, int C, int Ho, int Wo,
                                 const float* __restrict__ scale, const float* __restrict__ shift,
                                 const float* __restrict__ coef) {
  const int cv = C / 8;
  const int Hb = (H + 1) / 2, Wb = (W + 1) / 2;
  const int c = (int)((blockIdx.x * 256 + threadIdx.x) % cv) * 8;
  float sc[8], sh[8], k1[8], k2[8], k3[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = scale[c + i]; sh[i] = shift[c + i];
    k1[i] = coef[c + i]; k2[i] = coef[C + c + i]; k3[i] = coef[2 * C + c + i];
  }
  const unsigned nblk = (unsigned)(total / cv), qstep = gridDim.x * 256u / (unsigned)cv;
  for (unsigned q = (blockIdx.x * 256u + threadIdx.x) / (unsigned)cv; q < nblk; q += qstep) {
    const unsigned t_u = q / (unsigned)Wb;
    const int wb = (int)(q % (unsigned)Wb), hb = (int)(t_u % (unsigned)Hb);
    const int n = (int)(t_u / (unsigned)Hb);
    uint4 vd[2][2], v2[2][2], vy[2][2];
    uint2 va[2][2];
    uint32_t live[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int ho = hb - 1 + PBH + i, wo = wb - 1 + PBW + j;
        const int hc = min(max(ho, 0), Ho - 1), wc = min(max(wo, 0), Wo - 1);
        live[i][j] = (ho == hc && wo == wc) ? 0xffffffffu : 0u;
        const int64_t ooff = (int64_t)((n * Ho + hc) * Wo + wc) * C + c;
        vd[i][j] = *reinterpret_cast<const uint4*>(d + ooff);
        if (d2 != nullptr) v2[i][j] = *reinterpret_cast<const uint4*>(d2 + ooff);
        va[i][j] = *reinterpret_cast<const uint2*>(argmax + ooff);
        const int h = min(2 * hb + i, H - 1), w = min(2 * wb + j, W - 1);
        vy[i][j] = *reinterpret_cast<const uint4*>(y + ((int64_t)((n * H + h) * W + w) * C + c));
      }
    }
    uint32_t g[2][2][4], am[2][2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint32_t a4[4] = {vd[i][j].x, vd[i][j].y, vd[i][j].z, vd[i][j].w};
        const uint32_t b4[4] = {v2[i][j].x, v2[i][j].y, v2[i][j].z, v2[i][j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          uint32_t t = a4[k];
          if (d2 != nullptr) t = as_u32(__hadd2(as_bf2(a4[k]), as_bf2(b4[k])));
          g[i][j][k] = t & live[i][j];
        }
        // code bytes -> 16-bit lanes holding code * 0x0101 (bf16 bit patterns: zero or normal, never NaN)
        am[i][j][0] = __byte_perm(va[i][j].x, 0, 0x1100); am[i][j][1] = __byte_perm(va[i][j].x, 0, 0x3322);
        am[i][j][2] = __byte_perm(va[i][j].y, 0, 0x1100); am[i][j][3] = __byte_perm(va[i][j].y, 0, 0x3322);
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int h = 2 * hb + a, w = 2 * wb + b;
        // windows this pixel lies in (compile-time after unrolling): with one or two, a packed bf16 add IS the
        // rounded exact sum; with more, accumulate in fp32 and round once (the unfused pooling backward's rounding)
        const int nwin = ((a + 2 - PBH <= 2) + (a - PBH >= 0)) * ((b + 2 - PBW <= 2) + (b - PBW >= 0));
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        float accf[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int dh = a + 2 - PBH - 2 * i;          // compile-time after unrolling
          if (dh < 0 || dh > 2) continue;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int dw = b + 2 - PBW - 2 * j;
            if (dw < 0 || dw > 2) continue;
            const uint32_t code2 = (uint32_t)(dh * 3 + dw) * 0x01010101u;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t gm = g[i][j][k] & __heq2_mask(as_bf2(am[i][j][k]), as_bf2(code2));
              if (nwin <= 2) acc[k] = as_u32(__hadd2(as_bf2(acc[k]), as_bf2(gm)));
              else { accf[2 * k] += __uint_as_float(gm << 16); accf[2 * k + 1] += __uint_as_float(gm & 0xffff0000u); }
            }
          }
        }
        if (nwin > 2) {
#pragma unroll
          for (int k = 0; k < 4; ++k) acc[k] = as_u32(__floats2bfloat162_rn(accf[2 * k], accf[2 * k + 1]));
        }
        const uint32_t yv[4] = {vy[a][b].x, vy[a][b].y, vy[a][b].z, vy[a][b].w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float y0 = __uint_as_float(yv[k] << 16), y1 = __uint_as_float(yv[k] & 0xffff0000u);
          const float d0 = fmaf(y0, sc[2 * k], sh[2 * k]) > 0.f ? __uint_as_float(acc[k] << 16) : 0.f;
          const float d1 = fmaf(y1, sc[2 * k + 1], sh[2 * k + 1]) > 0.f ? __uint_as_float(acc[k] & 0xffff0000u) : 0.f;
          const float o0 = fmaf(k1[2 * k], d0, fmaf(k2[2 * k], y0, k3[2 * k]));
          const float o1 = fmaf(k1[2 * k + 1], d1, fmaf(k2[2 * k + 1], y1, k3[2 * k + 1]));
          o[k] = as_u32(__floats2bfloat162_rn(o0, o1));
        }
        if (h < H && w < W)
          *reinterpret_cast<uint4*>(dy_out + ((int64_t)((n * H + h) * W + w) * C + c)) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// x [N][HW][C] -> y [N][C] mean.  One thread per (n, channel); HW strided reads are
// coalesced across channels.
template <typename T, typename To>
__global__ void avgpool_fwd_kernel(const T* __restrict__ x, To* __restrict__ y, int64_t N, int HW, int C) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * C) return;
  const int64_t n = idx / C; const int c = (int)(idx % C);
  const T* p = x + n * HW * (int64_t)C + c;
  float s = 0.f;
  for (int i = 0; i < HW; ++i) s += to_f<T>(p[(int64_t)i * C]);
  y[idx] = from_f<To>(s / (float)HW);
}

template <typename Ti, typename T>
__global__ void avgpool_bwd_kernel(const Ti* __restrict__ dy, T* __restrict__ dx, int64_t total, int HW, int C) {
  const float inv = 1.f / (float)HW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const int64_t n = idx / ((int64_t)HW * C);
    dx[idx] = from_f<T>(to_f<Ti>(dy[n * C + c]) * inv);
  }
}

// bf16 output, C % 8 == 0: one thread per (n, hw, 8 channels), a 16-byte store each (the scalar kernel above
// issues 2-byte stores and runs at a tenth of the HBM rate).
template <typename Ti>
__global__ void avgpool_bwd_vec8_kernel(const Ti* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int64_t total8,
                                        int HW, int C) {
  const float inv = 1.f / (float)HW;
  const int cv = C / 8;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total8;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * 8;
    const int64_t n = idx / ((int64_t)HW * cv);
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = to_f<Ti>(dy[n * C + c + i]) * inv;
    Vec16<__nv_bfloat16> o; o.pack(f);
    o.store(dx + idx * 8);
  }
}

inline void same_pad(int64_t H, int64_t* Ho, int* pb) {
  *Ho = (H + 1) / 2;
  int64_t total = (*Ho - 1) * 2 + 3 - H;
  if (total < 0) total = 0;
  *pb = (int)(total / 2);
}
inline unsigned grid_for(int64_t total, int threads) {
  int64_t b = (total + threads - 1) / threads;
  const int64_t cap = (int64_t)num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace
}  // namespace simclr

using namespace simclr;
typedef __nv_bfloat16 bf16;

extern "C" {

int simclr_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int dtype, int64_t N, int64_t H, int64_t W,
                            int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(x && y && argmax, "maxpool_fwd: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "maxpool_fwd: need C%%8==0 and positive dims");
  int64_t Ho, Wo; int pbh, pbw;
  same_pad(H, &Ho, &pbh); same_pad(W, &Wo, &pbw);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32) {
    const int64_t total = N * Ho * Wo * (C / 4);
    maxpool_fwd_kernel<float, false><<<grid_for(total, 256), 256, 0, st>>>((const float*)x, (float*)y, argmax, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, nullptr, nullptr);
  } else if (dtype == SIMCLR_BF16) {
    const int64_t total = N * Ho * Wo * (C / 8);
    maxpool_fwd_kernel<bf16, false><<<grid_for(total, 256), 256, 0, st>>>((const bf16*)x, (bf16*)y, argmax, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, nullptr, nullptr);
  } else { set_error("maxpool_fwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, void* dx, int dtype, int64_t N, int64_t H,
                            int64_t W, int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(dy && dx && argmax, "maxpool_bwd: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "maxpool_bwd: need C%%8==0 and positive dims");
  int64_t Ho, Wo; int pbh, pbw;
  same_pad(H, &Ho, &pbh); same_pad(W, &Wo, &pbw);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32) {
    const int64_t total = N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 4);
    maxpool_bwd_kernel<float><<<grid_for(total, 256), 256, 0, st>>>((const float*)dy, argmax, (float*)dx, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw);
  } else if (dtype == SIMCLR_BF16) {
    const int64_t total = N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
    maxpool_bwd_kernel<bf16><<<grid_for(total, 256), 256, 0, st>>>((const bf16*)dy, argmax, (bf16*)dx, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw);
  } else { set_error("maxpool_bwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bn_relu_maxpool_fwd(const void* y, int dtype, const float* scale, const float* shift, void* out,
                               uint8_t* argmax, void* ysel, int64_t N, int64_t H, int64_t W, int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(y && scale && shift && out && argmax, "bn_relu_maxpool_fwd: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "bn_relu_maxpool_fwd: need C%%8==0 and positive dims");
  int64_t Ho, Wo; int pbh, pbw;
  same_pad(H, &Ho, &pbh); same_pad(W, &Wo, &pbw);
  cudaStream_t st = (cudaStream_t)stream;
  SIMCLR_CHECK_ARG(ysel == nullptr || dtype == SIMCLR_BF16, "bn_relu_maxpool_fwd: ysel is a bf16-path output");
  if (dtype == SIMCLR_F32) {
    const int64_t total = N * Ho * Wo * (C / 4);
    maxpool_fwd_kernel<float, true><<<grid_for(total, 256), 256, 0, st>>>((const float*)y, (float*)out, argmax, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, scale, shift);
  } else if (dtype == SIMCLR_BF16) {
    const int64_t total = N * Ho * Wo * (C / 8);
    if (256 % (C / 8) == 0 && N * H * W < (int64_t(1) << 31))
      maxpool_bnrelu_fwd_bf16_kernel<<<grid_for(total, 256), 256, 0, st>>>((const bf16*)y, (bf16*)out, argmax, (bf16*)ysel, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, scale, shift);
    else {
      SIMCLR_CHECK_ARG(ysel == nullptr, "bn_relu_maxpool_fwd: ysel needs C/8 dividing 256");
      maxpool_fwd_kernel<bf16, true><<<grid_for(total, 256), 256, 0, st>>>((const bf16*)y, (bf16*)out, argmax, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, scale, shift);
    }
  } else { set_error("bn_relu_maxpool_fwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

static int maxpool_bn_bwd(int phase, const void* d, const void* d2, const uint8_t* argmax, const void* y,
                          const void* ysel, int dtype, void* dy, int64_t N, int64_t H, int64_t W, int64_t C, const float* mean, const float* rstd,
                          const float* scale, const float* shift, const float* coef, double* sums, void* stream) {
  const int V = dtype == SIMCLR_BF16 ? 8 : 4;
  const int64_t cv = C / V;
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && 256 % cv == 0,
                   "maxpool_bn_bwd: need C%%8==0 and C/%d dividing 256 (C=%lld)", V, (long long)C);
  int64_t Ho, Wo; int pbh, pbw;
  same_pad(H, &Ho, &pbh); same_pad(W, &Wo, &pbw);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = N * ((H + 1) / 2) * ((W + 1) / 2) * cv;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * (phase == 0 ? 4 : 16);       // phase 0 ends with one partial per channel per block
  if (blocks > cap) blocks = cap;
  if (phase == 0 && !accumulate_prezeroed()) SIMCLR_CHECK_CUDA(cudaMemsetAsync(sums, 0, 2 * C * sizeof(double), st));
  // phase 0: every block writes its partial [2][C] to scratch; the partials are added into `sums` in block order
  double* ws = nullptr;
  int nparts = 0;
  if (phase == 0) {
    nparts = (int)blocks;
    if (dtype == SIMCLR_BF16 && ysel != nullptr) {
      const int64_t pb = (N * Ho * Wo * cv + 511) / 512;
      nparts = (int)(pb > cap ? cap : pb);
    }
    int rc = scratch_alloc(&ws, (size_t)nparts * 2 * C * sizeof(double), st);
    if (rc) return rc;
    const cudaError_t e = cudaMemsetAsync(ws, 0, (size_t)nparts * 2 * C * sizeof(double), st);
    if (e != cudaSuccess) { set_error("maxpool_bn_bwd: memset: %s", cudaGetErrorString(e)); scratch_free(ws, st); return (int)e; }
  }
  auto finish = [&]() -> int {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_error("maxpool_bn_bwd: launch: %s", cudaGetErrorString(e));
      if (ws) scratch_free(ws, st);
      return (int)e;
    }
    if (!ws) return SIMCLR_OK;
    const int rc = run_sum_partials_f64(ws, 2 * C, sums, 2 * C, nparts, st);
    const int rf = scratch_free(ws, st);
    return rc ? rc : rf;
  };
  if (dtype == SIMCLR_BF16 && phase == 0 && ysel != nullptr) {
    const int64_t ptotal = N * Ho * Wo * cv;
    maxpool_bn_bwd_reduce_pooled_bf16_kernel<<<(unsigned)nparts, 256, 0, st>>>((const bf16*)d, (const bf16*)d2, (const bf16*)ysel, ptotal, (int)C, mean, rstd, scale, shift, ws);
    return finish();
  }
  if (dtype == SIMCLR_BF16 && phase == 1 && N * H * W < (int64_t(1) << 31)) {
#define MPA(PH, PW) maxpool_bn_bwd_apply_bf16_kernel<PH, PW><<<(unsigned)blocks, 256, 0, st>>>((const bf16*)d, (const bf16*)d2, argmax, (const bf16*)y, (bf16*)dy, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, scale, shift, coef)
    if (pbh == 0 && pbw == 0) MPA(0, 0); else if (pbh == 0) MPA(0, 1); else if (pbw == 0) MPA(1, 0); else MPA(1, 1);
#undef MPA
    SIMCLR_CHECK_LAUNCH();
    return SIMCLR_OK;
  }
#define MPB(T, PH) maxpool_bn_bwd_kernel<T, PH><<<(unsigned)blocks, 256, 0, st>>>((const T*)d, (const T*)d2, argmax, (const T*)y, (T*)dy, total, (int)H, (int)W, (int)C, (int)Ho, (int)Wo, pbh, pbw, mean, rstd, scale, shift, coef, ws)
  if (dtype == SIMCLR_F32) { if (phase == 0) MPB(float, 0); else MPB(float, 1); }
  else if (dtype == SIMCLR_BF16) { if (phase == 0) MPB(bf16, 0); else MPB(bf16, 1); }
  else { set_error("maxpool_bn_bwd: unknown dtype"); if (ws) scratch_free(ws, st); return SIMCLR_ERR_INVALID_ARG; }
#undef MPB
  return finish();
}

int simclr_maxpool_bn_bwd_reduce(const void* d, const void* d2, const uint8_t* argmax, const void* y,
                                 const void* ysel, int dtype, int64_t N, int64_t H, int64_t W, int64_t C, const float* mean, const float* rstd,
                                 const float* scale, const float* shift, double* sums, void* stream) {
  SIMCLR_CHECK_ARG(d && argmax && y && mean && rstd && scale && shift && sums, "maxpool_bn_bwd_reduce: null pointer");
  return maxpool_bn_bwd(0, d, d2, argmax, y, ysel, dtype, nullptr, N, H, W, C, mean, rstd, scale, shift, nullptr, sums, stream);
}

int simclr_maxpool_bn_bwd_apply(const void* d, const void* d2, const uint8_t* argmax, const void* y, int dtype, void* dy,
                                int64_t N, int64_t H, int64_t W, int64_t C, const float* coef, const float* scale,
                                const float* shift, void* stream) {
  SIMCLR_CHECK_ARG(d && argmax && y && dy && coef && scale && shift, "maxpool_bn_bwd_apply: null pointer");
  return maxpool_bn_bwd(1, d, d2, argmax, y, nullptr, dtype, dy, N, H, W, C, nullptr, nullptr, scale, shift, coef, nullptr, stream);
}

int simclr_global_avgpool_fwd(const void* x, int dtype, void* y, int y_dtype, int64_t N, int64_t HW, int64_t C,
                              void* stream) {
  SIMCLR_CHECK_ARG(x && y && N > 0 && HW > 0 && C > 0, "avgpool_fwd: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((N * C + 255) / 256);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32) avgpool_fwd_kernel<float, float><<<grid, 256, 0, st>>>((const float*)x, (float*)y, N, (int)HW, (int)C);
  else if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16) avgpool_fwd_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)y, N, (int)HW, (int)C);
  else if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_F32) avgpool_fwd_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)x, (float*)y, N, (int)HW, (int)C);
  else if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_BF16) avgpool_fwd_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)x, (bf16*)y, N, (int)HW, (int)C);
  else { set_error("avgpool_fwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_global_avgpool_bwd(const void* dy, int dy_dtype, void* dx, int dtype, int64_t N, int64_t HW, int64_t C,
                              void* stream) {
  SIMCLR_CHECK_ARG(dy && dx && N > 0 && HW > 0 && C > 0, "avgpool_bwd: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = N * HW * C;
  const unsigned grid = grid_for(total, 256);
  if (dtype == SIMCLR_BF16 && C % 8 == 0) {
    const unsigned g8 = grid_for(total / 8, 256);
    if (dy_dtype == SIMCLR_F32) avgpool_bwd_vec8_kernel<float><<<g8, 256, 0, st>>>((const float*)dy, (bf16*)dx, total / 8, (int)HW, (int)C);
    else if (dy_dtype == SIMCLR_BF16) avgpool_bwd_vec8_kernel<bf16><<<g8, 256, 0, st>>>((const bf16*)dy, (bf16*)dx, total / 8, (int)HW, (int)C);
    else { set_error("avgpool_bwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
    SIMCLR_CHECK_LAUNCH();
    return SIMCLR_OK;
  }
  if (dy_dtype == SIMCLR_F32 && dtype == SIMCLR_F32) avgpool_bwd_kernel<float, float><<<grid, 256, 0, st>>>((const float*)dy, (float*)dx, total, (int)HW, (int)C);
  else if (dy_dtype == SIMCLR_BF16 && dtype == SIMCLR_BF16) avgpool_bwd_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)dy, (bf16*)dx, total, (int)HW, (int)C);
  else if (dy_dtype == SIMCLR_F32 && dtype == SIMCLR_BF16) avgpool_bwd_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)dy, (bf16*)dx, total, (int)HW, (int)C);
  else if (dy_dtype == SIMCLR_BF16 && dtype == SIMCLR_F32) avgpool_bwd_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)dy, (float*)dx, total, (int)HW, (int)C);
  else { set_error("avgpool_bwd: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
