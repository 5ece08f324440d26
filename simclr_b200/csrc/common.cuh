// Shared helpers for the simclr_b200 sm_90a kernels (internal header).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/simclr_b200.h"

namespace simclr {

// ---- error reporting (thread-local text, SURVEY.md 8b) ---------------------
void set_error(const char* fmt, ...);
// true: the caller has zeroed the accumulation outputs (BN sums, dW) itself (simclr_set_accumulate_prezeroed)
bool accumulate_prezeroed();

#define SIMCLR_CHECK_ARG(cond, ...)                                   \
  do {                                                                \
    if (!(cond)) {                                                    \
      ::simclr::set_error(__VA_ARGS__);                               \
      return SIMCLR_ERR_INVALID_ARG;                                  \
    }                                                                 \
  } while (0)

#define SIMCLR_CHECK_LAUNCH()                                         \
  do {                                                                \
    cudaError_t e__ = cudaGetLastError();                             \
    if (e__ != cudaSuccess) {                                         \
      ::simclr::set_error("%s:%d launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return (int)e__;                                                \
    }                                                                 \
  } while (0)

#define SIMCLR_CHECK_CUDA(expr)                                       \
  do {                                                                \
    cudaError_t e__ = (expr);                                         \
    if (e__ != cudaSuccess) {                                         \
      ::simclr::set_error("%s:%d %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
      return (int)e__;                                                \
    }                                                                 \
  } while (0)

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Scratch for the partial sums of split reductions: stream-ordered, so it is legal inside CUDA-graph capture
// (the graph then owns the allocation) and costs no device synchronisation.  Freed memory stays in the pool.
template <typename T>
inline int scratch_alloc(T** p, size_t bytes, cudaStream_t st) {
  static bool pool_kept[64] = {};
  int dev = 0;
  SIMCLR_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !pool_kept[dev]) {
    cudaMemPool_t pool;
    uint64_t keep = UINT64_MAX;
    SIMCLR_CHECK_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
    SIMCLR_CHECK_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    pool_kept[dev] = true;
  }
  SIMCLR_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(p), bytes, st));
  return SIMCLR_OK;
}
inline int scratch_free(void* p, cudaStream_t st) {
  SIMCLR_CHECK_CUDA(cudaFreeAsync(p, st));
  return SIMCLR_OK;
}
// dst[i] += the sum of parts[p][i] (part p at ws + p * stride) in an order fixed by `parts` alone: the split reductions of the
// weight gradients go through it instead of atomics, so that a step computes the same bits every run (defined in tc_conv.cu)
int run_sum_partials(const float* ws, int64_t stride, float* dst, int64_t n, int parts, cudaStream_t st);
// the same for the fp64 BatchNorm statistic sums (bn.cu, pool.cu, the fused statistics of the conv epilogues)
int run_sum_partials_f64(const double* ws, int64_t stride, double* dst, int64_t n, int parts, cudaStream_t st);


// ---- device helpers --------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// BatchNorm finalize of channel c from the (global) sums s0 = sum x, s1 = sum x^2 over `count` rows: mean, rstd,
// scale, shift and the moving-average update.  bn_finalize_kernel (bn.cu) and the SyncBN exchange (comm.cu) both
// call it, so the peer-memory and NCCL paths of a multi-GPU step give the same bits.  The fused operations are
// spelled out: left to the compiler, E[x^2] - mean^2 was contracted in one kernel and not in the other.
__device__ __forceinline__ void bn_finalize_channel(double s0, double s1, double count, const float* gamma,
                                                    const float* beta, float eps, float momentum, float* mm, float* mv,
                                                    float* mean, float* rstd, float* scale, float* shift, int c) {
  const double m = s0 / count;
  double var = fma(-m, m, s1 / count);          // biased variance (SyncBN form, SURVEY A4)
  if (var < 0.0) var = 0.0;
  const float mf = (float)m, vf = (float)var;
  const float r = rsqrtf(vf + eps);
  const float g = gamma ? gamma[c] : 1.f;
  const float b = beta ? beta[c] : 0.f;
  const float sc = __fmul_rn(g, r);
  const float om = 1.f - momentum;
  mean[c] = mf; rstd[c] = r; scale[c] = sc; shift[c] = fmaf(-mf, sc, b);
  if (mm) mm[c] = fmaf(-(mm[c] - mf), om, mm[c]);
  if (mv) mv[c] = fmaf(-(mv[c] - vf), om, mv[c]);
}

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// A 16-byte vector of activations: 4 fp32 or 8 bf16.
template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  float4 raw;
  __device__ __forceinline__ void load(const float* p) { raw = *reinterpret_cast<const float4*>(p); }
  __device__ __forceinline__ void store(float* p) const { *reinterpret_cast<float4*>(p) = raw; }
  __device__ __forceinline__ void unpack(float* f) const { f[0] = raw.x; f[1] = raw.y; f[2] = raw.z; f[3] = raw.w; }
  __device__ __forceinline__ void pack(const float* f) { raw = make_float4(f[0], f[1], f[2], f[3]); }
};
template <> struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  uint4 raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { *reinterpret_cast<uint4*>(p) = raw; }
  __device__ __forceinline__ void unpack(float* f) const {
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ __forceinline__ void pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    raw = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

}  // namespace simclr
