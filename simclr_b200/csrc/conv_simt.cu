// CUDA-core fp32 convolution engine reading the fp32 HWIO master weights.
// Deliberately simple (one thread per output element, fp32 FMA): it is the
// on-device verification engine for the tensor-core path and the fp32 parity path
// of the small configs; it is never the default engine.
// Semantics: tf2/resnet.py:183-208 (stride 1 'SAME', stride>1 FixedPadding +
// 'VALID'  ==  pad_beg = (k-1)/2 for odd k).
#include "common.cuh"

namespace simclr {
namespace {

struct Geo { int N, H, W, Cs, Cin, Cout, R, S, stride, pad_h, pad_w, Ho, Wo; };

template <typename T, typename To>
__global__ void __launch_bounds__(256)
fprop_kernel(const T* __restrict__ x, const float* __restrict__ w, To* __restrict__ y, Geo g) {
  const int64_t total = (int64_t)g.N * g.Ho * g.Wo * g.Cout;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(idx % g.Cout);
    int64_t m = idx / g.Cout;
    const int wo = (int)(m % g.Wo); m /= g.Wo;
    const int ho = (int)(m % g.Ho);
    const int64_t n = m / g.Ho;
    float acc = 0.f;
    for (int r = 0; r < g.R; ++r) {
      const int h = ho * g.stride - g.pad_h + r;
      if (h < 0 || h >= g.H) continue;
      for (int s = 0; s < g.S; ++s) {
        const int ww = wo * g.stride - g.pad_w + s;
        if (ww < 0 || ww >= g.W) continue;
        const T* xp = x + ((n * g.H + h) * g.W + ww) * (int64_t)g.Cs;
        const float* wp = w + ((int64_t)(r * g.S + s) * g.Cin) * g.Cout + co;
        for (int c = 0; c < g.Cin; ++c) acc = fmaf(to_f<T>(xp[c]), wp[(int64_t)c * g.Cout], acc);
      }
    }
    y[idx] = from_f<To>(acc);
  }
}

template <typename T, typename To>
__global__ void __launch_bounds__(256)
dgrad_kernel(const T* __restrict__ dy, const float* __restrict__ w, To* __restrict__ dx, Geo g) {
  const int64_t total = (int64_t)g.N * g.H * g.W * g.Cin;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int ci = (int)(idx % g.Cin);
    int64_t m = idx / g.Cin;
    const int ww = (int)(m % g.W); m /= g.W;
    const int h = (int)(m % g.H);
    const int64_t n = m / g.H;
    float acc = 0.f;
    for (int r = 0; r < g.R; ++r) {
      const int t = h + g.pad_h - r;
      if (t < 0 || t % g.stride) continue;
      const int ho = t / g.stride;
      if (ho >= g.Ho) continue;
      for (int s = 0; s < g.S; ++s) {
        const int u = ww + g.pad_w - s;
        if (u < 0 || u % g.stride) continue;
        const int wo = u / g.stride;
        if (wo >= g.Wo) continue;
        const T* dp = dy + ((n * g.Ho + ho) * g.Wo + wo) * (int64_t)g.Cout;
        const float* wp = w + ((int64_t)(r * g.S + s) * g.Cin + ci) * g.Cout;
        for (int co = 0; co < g.Cout; ++co) acc = fmaf(to_f<T>(dp[co]), wp[co], acc);
      }
    }
    dx[idx] = from_f<To>(acc);
  }
}

// dw[(r,s,ci),co] = sum_m x[m@(r,s), ci] * dy[m, co]; the M reduction is split
// over blockIdx.y and combined with fp32 atomics (dw zeroed by the caller).
template <typename T>
__global__ void __launch_bounds__(256)
wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ dw, Geo g, int64_t m_per_split) {
  const int64_t total = (int64_t)g.R * g.S * g.Cin * g.Cout;
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  const int64_t m0 = (int64_t)blockIdx.y * m_per_split;
  const int64_t m1 = min(M, m0 + m_per_split);
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(idx % g.Cout);
    int64_t k = idx / g.Cout;
    const int ci = (int)(k % g.Cin); k /= g.Cin;
    const int s = (int)(k % g.S);
    const int r = (int)(k / g.S);
    float acc = 0.f;
    for (int64_t m = m0; m < m1; ++m) {
      const int wo = (int)(m % g.Wo);
      const int64_t t = m / g.Wo;
      const int ho = (int)(t % g.Ho);
      const int64_t n = t / g.Ho;
      const int h = ho * g.stride - g.pad_h + r;
      const int ww = wo * g.stride - g.pad_w + s;
      if (h < 0 || h >= g.H || ww < 0 || ww >= g.W) continue;
      acc = fmaf(to_f<T>(x[((n * g.H + h) * g.W + ww) * (int64_t)g.Cs + ci]), to_f<T>(dy[m * g.Cout + co]), acc);
    }
    atomicAdd(dw + idx, acc);
  }
}

inline int make_geo(Geo* g, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                    int64_t S, int64_t stride) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cs < Cin || Cout <= 0 || R <= 0 || S <= 0 || stride <= 0 ||
      (R % 2) == 0 || (S % 2) == 0) {
    set_error("conv: bad geometry N=%lld H=%lld W=%lld Cs=%lld Cin=%lld Cout=%lld R=%lld S=%lld stride=%lld",
              (long long)N, (long long)H, (long long)W, (long long)Cs, (long long)Cin, (long long)Cout,
              (long long)R, (long long)S, (long long)stride);
    return SIMCLR_ERR_INVALID_ARG;
  }
  g->N = (int)N; g->H = (int)H; g->W = (int)W; g->Cs = (int)Cs; g->Cin = (int)Cin; g->Cout = (int)Cout;
  g->R = (int)R; g->S = (int)S; g->stride = (int)stride;
  g->pad_h = (int)((R - 1) / 2); g->pad_w = (int)((S - 1) / 2);
  g->Ho = (int)((H + 2 * g->pad_h - R) / stride + 1);      // == H for stride 1; FixedPadding+VALID otherwise
  g->Wo = (int)((W + 2 * g->pad_w - S) / stride + 1);
  return SIMCLR_OK;
}

inline unsigned grid_for(int64_t total) {
  int64_t b = (total + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 32;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace
}  // namespace simclr

using namespace simclr;
typedef __nv_bfloat16 bf16;

extern "C" {

int simclr_conv2d_fprop_simt(const void* x, const float* w_hwio, void* y, int dtype, int y_dtype, int64_t N,
                             int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R, int64_t S,
                             int64_t stride, void* stream) {
  SIMCLR_CHECK_ARG(x && w_hwio && y, "conv2d_fprop_simt: null pointer");
  Geo g; int rc = make_geo(&g, N, H, W, Cs, Cin, Cout, R, S, stride); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = grid_for((int64_t)g.N * g.Ho * g.Wo * g.Cout);
  if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_F32) fprop_kernel<float, float><<<grid, 256, 0, st>>>((const float*)x, w_hwio, (float*)y, g);
  else if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_BF16) fprop_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)x, w_hwio, (bf16*)y, g);
  else if (dtype == SIMCLR_BF16 && y_dtype == SIMCLR_F32) fprop_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)x, w_hwio, (float*)y, g);
  else if (dtype == SIMCLR_F32 && y_dtype == SIMCLR_BF16) fprop_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)x, w_hwio, (bf16*)y, g);
  else { set_error("conv2d_fprop_simt: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_conv2d_dgrad_simt(const void* dy, const float* w_hwio, void* dx, int dtype, int dx_dtype, int64_t N,
                             int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride,
                             void* stream) {
  SIMCLR_CHECK_ARG(dy && w_hwio && dx, "conv2d_dgrad_simt: null pointer");
  Geo g; int rc = make_geo(&g, N, H, W, Cin, Cin, Cout, R, S, stride); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = grid_for((int64_t)g.N * g.H * g.W * g.Cin);
  if (dtype == SIMCLR_F32 && dx_dtype == SIMCLR_F32) dgrad_kernel<float, float><<<grid, 256, 0, st>>>((const float*)dy, w_hwio, (float*)dx, g);
  else if (dtype == SIMCLR_BF16 && dx_dtype == SIMCLR_BF16) dgrad_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)dy, w_hwio, (bf16*)dx, g);
  else if (dtype == SIMCLR_BF16 && dx_dtype == SIMCLR_F32) dgrad_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)dy, w_hwio, (float*)dx, g);
  else if (dtype == SIMCLR_F32 && dx_dtype == SIMCLR_BF16) dgrad_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)dy, w_hwio, (bf16*)dx, g);
  else { set_error("conv2d_dgrad_simt: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_conv2d_wgrad_simt(const void* x, const void* dy, float* dw, int dtype, int64_t N, int64_t H, int64_t W,
                             int64_t Cs, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride,
                             void* stream) {
  SIMCLR_CHECK_ARG(x && dy && dw, "conv2d_wgrad_simt: null pointer");
  Geo g; int rc = make_geo(&g, N, H, W, Cs, Cin, Cout, R, S, stride); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = (int64_t)g.R * g.S * g.Cin * g.Cout;
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  SIMCLR_CHECK_CUDA(cudaMemsetAsync(dw, 0, total * sizeof(float), st));
  int64_t bx = (total + 255) / 256;
  int64_t splits = (4 * num_sms() + bx - 1) / bx; if (splits < 1) splits = 1; if (splits > M) splits = M;
  if (splits > 1024) splits = 1024;
  const int64_t mps = (M + splits - 1) / splits;
  splits = (M + mps - 1) / mps;
  dim3 grid((unsigned)(bx > 65535 ? 65535 : bx), (unsigned)splits);
  if (dtype == SIMCLR_F32) wgrad_kernel<float><<<grid, 256, 0, st>>>((const float*)x, (const float*)dy, dw, g, mps);
  else if (dtype == SIMCLR_BF16) wgrad_kernel<bf16><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)dy, dw, g, mps);
  else { set_error("conv2d_wgrad_simt: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
