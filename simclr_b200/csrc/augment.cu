// Train-time augmentation on device (tf2/data_util.py:443-475): crop + bicubic
// resize (tf.image.resize BICUBIC: half-pixel centres, Keys a=-0.5, 1024-entry
// coefficient table indexed by lrintf(frac * 1024) of the fp32 sample position,
// out-of-range taps dropped and weights renormalised), flip,
// colour jitter in a drawn order with a clip after each op, grayscale, final clip.
// All random draws are inputs.  One CTA per output image; every thread owns the
// same output pixels in every pass, only the contrast mean needs a block reduction.
#include "common.cuh"

namespace simclr {
namespace {

constexpr int AT = 512;

__device__ __forceinline__ double keys_inner(double x) { return ((1.5 * x - 2.5) * x) * x + 1.0; }          // |x| <= 1, A=-0.5
__device__ __forceinline__ double keys_outer(double x) { return ((-0.5 * x + 2.5) * x - 4.0) * x + 2.0; }   // 1 < |x| < 2

// weights/indices of the 4 taps for output index o (TF GetWeightsAndIndices, half-pixel scaler).  The sample
// position, its floor and the table offset are TF's fp32 arithmetic, each operation rounded on its own (no FMA
// contraction): scale = in/out, src = (o + 0.5) * scale - 0.5, offset = lrintf((src - floor(src)) * 1024).  In
// fp64 the offset differs for large crops (first at crop side 898 for a 224 output).
__device__ __forceinline__ void bicubic_taps(int o, int in_size, int out_size, int* idx, float* w) {
  const float scale = __fdiv_rn((float)in_size, (float)out_size);
  const float src = __fsub_rn(__fmul_rn(__fadd_rn((float)o, 0.5f), scale), 0.5f);
  const float fl = floorf(src);
  const int off = (int)lrintf(__fmul_rn(__fsub_rn(src, fl), 1024.f));
  const double x = (double)off / 1024.0;
  double ww[4] = {keys_outer(x + 1.0), keys_inner(x), keys_inner(1.0 - x), keys_outer(2.0 - x)};
  double tot = 0.0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int ii = (int)fl - 1 + t;
    if (ii < 0 || ii >= in_size) ww[t] = 0.0; else tot += ww[t];
    idx[t] = min(max(ii, 0), in_size - 1);
  }
  const double inv = (fabs(tot) >= 1000.0 * 1.17549435e-38) ? 1.0 / tot : 1.0;
#pragma unroll
  for (int t = 0; t < 4; ++t) w[t] = (float)(ww[t] * inv);
}

__device__ __forceinline__ float clip01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

__device__ __forceinline__ void rgb_to_hsv(float r, float g, float b, float& h, float& s, float& v) {
  v = fmaxf(fmaxf(r, g), b);
  const float mn = fminf(fminf(r, g), b);
  const float rng = v - mn;
  s = v > 0.f ? rng / v : 0.f;
  const float norm = 1.f / (6.f * (rng > 0.f ? rng : 1.f));
  if (r == v) h = norm * (g - b);
  else if (g == v) h = norm * (b - r) + 2.f / 6.f;
  else h = norm * (r - g) + 4.f / 6.f;
  if (!(rng > 0.f)) h = 0.f;
  if (h < 0.f) h += 1.f;
}
__device__ __forceinline__ void hsv_to_rgb(float h, float s, float v, float& r, float& g, float& b) {
  const float dh = h * 6.f;
  const float dr = fminf(fmaxf(fabsf(dh - 3.f) - 1.f, 0.f), 1.f);
  const float dg = fminf(fmaxf(2.f - fabsf(dh - 2.f), 0.f), 1.f);
  const float db = fminf(fmaxf(2.f - fabsf(dh - 4.f), 0.f), 1.f);
  const float oms = 1.f - s;
  r = (oms + s * dr) * v; g = (oms + s * dg) * v; b = (oms + s * db) * v;
}

__global__ void __launch_bounds__(AT)
augment_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ src_offset, const int32_t* __restrict__ src_hw,
               const int32_t* __restrict__ box, const uint8_t* __restrict__ flip, const float* __restrict__ colour,
               float* __restrict__ out, int height, int width, int64_t pix_stride, int ch_off) {
  __shared__ float red[3][AT / 32];
  __shared__ float mean_s[3];
  const int img = blockIdx.x;
  const uint8_t* im = src + src_offset[img];
  const int Ws = src_hw[img * 2 + 1];
  const int by = box[img * 4 + 0], bx = box[img * 4 + 1], bh = box[img * 4 + 2], bw = box[img * 4 + 3];
  const bool fl = flip[img] != 0;
  const float* col = colour + img * 8;
  float* o = out + (int64_t)img * height * width * pix_stride + ch_off;
  const int npix = height * width;

  // pass 0: crop + bicubic resize (+ flip: this thread owns the *output* pixel)
  for (int p = threadIdx.x; p < npix; p += AT) {
    const int oy = p / width, ox_out = p - oy * width;
    const int ox = fl ? width - 1 - ox_out : ox_out;
    int iy[4], ix[4]; float wy[4], wx[4];
    bicubic_taps(oy, bh, height, iy, wy);
    bicubic_taps(ox, bw, width, ix, wx);
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const uint8_t* row = im + ((int64_t)(by + iy[a]) * Ws + bx) * 3;
      float racc[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint8_t* px = row + ix[b] * 3;
        // convert_image_dtype(uint8 -> float32): x / 255
        racc[0] = fmaf(wx[b], (float)px[0] * (1.f / 255.f), racc[0]);
        racc[1] = fmaf(wx[b], (float)px[1] * (1.f / 255.f), racc[1]);
        racc[2] = fmaf(wx[b], (float)px[2] * (1.f / 255.f), racc[2]);
      }
      acc[0] = fmaf(wy[a], racc[0], acc[0]); acc[1] = fmaf(wy[a], racc[1], acc[1]); acc[2] = fmaf(wy[a], racc[2], acc[2]);
    }
    float* d = o + (int64_t)p * pix_stride;
    d[0] = acc[0]; d[1] = acc[1]; d[2] = acc[2];
  }

  if (col[0] != 0.f) {        // random_apply(color_jitter, p=0.8)
    const int perm = (int)col[1];
    for (int t = 0; t < 4; ++t) {
      const int op = (perm >> (2 * t)) & 3;
      if (op == 1) {          // contrast: (x - mean_hw) * f + mean_hw per channel
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
        for (int p = threadIdx.x; p < npix; p += AT) {
          const float* d = o + (int64_t)p * pix_stride;
          s0 += d[0]; s1 += d[1]; s2 += d[2];
        }
        s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s0; red[1][threadIdx.x >> 5] = s1; red[2][threadIdx.x >> 5] = s2; }
        __syncthreads();
        if (threadIdx.x < 3) {
          float tot = 0.f;
          for (int k = 0; k < AT / 32; ++k) tot += red[threadIdx.x][k];
          mean_s[threadIdx.x] = tot / (float)npix;
        }
        __syncthreads();
      }
      for (int p = threadIdx.x; p < npix; p += AT) {
        float* d = o + (int64_t)p * pix_stride;
        float r = d[0], g = d[1], b = d[2];
        if (op == 0) { const float f = col[2]; r *= f; g *= f; b *= f; }
        else if (op == 1) { const float f = col[3]; r = (r - mean_s[0]) * f + mean_s[0]; g = (g - mean_s[1]) * f + mean_s[1]; b = (b - mean_s[2]) * f + mean_s[2]; }
        else if (op == 2) { float h, s, v; rgb_to_hsv(r, g, b, h, s, v); s = clip01(s * col[4]); hsv_to_rgb(h, s, v, r, g, b); }
        else { float h, s, v; rgb_to_hsv(r, g, b, h, s, v); h += col[5]; h -= floorf(h); hsv_to_rgb(h, s, v, r, g, b); }
        d[0] = clip01(r); d[1] = clip01(g); d[2] = clip01(b);       // clip_by_value after each op
      }
    }
  }
  const bool gray = col[6] != 0.f;
  for (int p = threadIdx.x; p < npix; p += AT) {
    float* d = o + (int64_t)p * pix_stride;
    float r = d[0], g = d[1], b = d[2];
    if (gray) { const float y = 0.2989f * r + 0.5870f * g + 0.1140f * b; r = g = b = y; }   // rgb_to_grayscale, tiled
    d[0] = clip01(r); d[1] = clip01(g); d[2] = clip01(b);           // final clip (tf2/data_util.py:474)
  }
}

}  // namespace
}  // namespace simclr

using namespace simclr;

extern "C" int simclr_augment(const uint8_t* src, const int64_t* src_offset, const int32_t* src_hw, const int32_t* box,
                              const uint8_t* flip, const float* colour, float* out, int64_t n, int64_t height,
                              int64_t width, int64_t out_pixel_stride, int64_t out_channel_offset, void* stream) {
  SIMCLR_CHECK_ARG(src && src_offset && src_hw && box && flip && colour && out, "augment: null pointer");
  SIMCLR_CHECK_ARG(n > 0 && height > 0 && width > 0 && out_pixel_stride >= 3 && out_channel_offset >= 0 &&
                       out_channel_offset + 3 <= out_pixel_stride, "augment: bad shape");
  augment_kernel<<<(unsigned)n, AT, 0, (cudaStream_t)stream>>>(src, src_offset, src_hw, box, flip, colour, out, (int)height,
                                                               (int)width, out_pixel_stride, (int)out_channel_offset);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}
