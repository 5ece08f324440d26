// Knowledge distillation loss of SimCLRv2 (the distillation colab's `add_kd_loss`): the student is trained on the
// temperature-softened predictions of a frozen teacher.
//
//   p = softmax(teacher / T),  log q = log_softmax(student / T),  l_r = -sum_c p_c log q_c
//   loss = T^2 * mean_r l_r,   dstudent = (q - p) * grad_scale   (d loss / d student = (T / rows) (q - p))
//
// One block per row, three passes over the row: maxima (and the argmaxes of the raw logits), the two partition
// functions, then the row loss and the gradient.  Every exponent is max-subtracted before the division by T, so the
// kernel stays finite for logits of +-1e4 at small T.  Sums are fp64 in a fixed order; the count of rows whose
// argmaxes agree is an integer sum.  A second, single-block kernel forms the mean in a fixed order, so the result has
// the same bits on every run.
#include "common.cuh"

namespace simclr {
namespace {

constexpr int kRowThreads = 256;
constexpr int kRowWarps = kRowThreads / 32;

__device__ __forceinline__ void argmax_merge(float& v, int& i, float v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    argmax_merge(v, i, v2, i2);
  }
}

// block-wide sum of two doubles, the same order on every run; every thread gets the result
__device__ __forceinline__ void block_sum2(double& a, double& b, double (*sh)[kRowWarps]) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  a = warp_sum(a); b = warp_sum(b);
  if (lane == 0) { sh[0][w] = a; sh[1][w] = b; }
  __syncthreads();
  a = 0.0; b = 0.0;
#pragma unroll
  for (int k = 0; k < kRowWarps; ++k) { a += sh[0][k]; b += sh[1][k]; }
  __syncthreads();
}

__global__ void __launch_bounds__(kRowThreads)
distill_rows_kernel(const float* __restrict__ student, const float* __restrict__ teacher, int classes, float T,
                    float grad_scale, float* __restrict__ row_loss, float* __restrict__ dstudent,
                    unsigned* __restrict__ agree) {
  __shared__ float sh_v[2][kRowWarps];
  __shared__ int sh_i[2][kRowWarps];
  __shared__ double sh_d[2][kRowWarps];
  const int64_t r = blockIdx.x;
  const float* s = student + r * classes;
  const float* t = teacher + r * classes;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // pass 1: maxima with the lowest index among equal values (each thread walks its columns in increasing order)
  float ms = -INFINITY, mt = -INFINITY;
  int is = classes, it = classes;
  for (int c = threadIdx.x; c < classes; c += kRowThreads) {
    const float a = s[c], b = t[c];
    if (a > ms) { ms = a; is = c; }
    if (b > mt) { mt = b; it = c; }
  }
  warp_argmax(ms, is); warp_argmax(mt, it);
  if (lane == 0) { sh_v[0][w] = ms; sh_i[0][w] = is; sh_v[1][w] = mt; sh_i[1][w] = it; }
  __syncthreads();
  ms = sh_v[0][0]; is = sh_i[0][0]; mt = sh_v[1][0]; it = sh_i[1][0];
#pragma unroll
  for (int k = 1; k < kRowWarps; ++k) { argmax_merge(ms, is, sh_v[0][k], sh_i[0][k]); argmax_merge(mt, it, sh_v[1][k], sh_i[1][k]); }

  // pass 2: partition functions of the max-subtracted, temperature-scaled logits
  double zs = 0.0, zt = 0.0;
  for (int c = threadIdx.x; c < classes; c += kRowThreads) {
    zs += (double)expf((s[c] - ms) / T);
    zt += (double)expf((t[c] - mt) / T);
  }
  block_sum2(zs, zt, sh_d);
  const float log_zs = (float)log(zs);
  const float inv_zt = (float)(1.0 / zt);

  // pass 3: row cross-entropy -sum p log q and the gradient (q - p) * grad_scale
  double acc = 0.0, unused = 0.0;
  for (int c = threadIdx.x; c < classes; c += kRowThreads) {
    const float log_q = (s[c] - ms) / T - log_zs;
    const float p = expf((t[c] - mt) / T) * inv_zt;
    acc -= (double)p * (double)log_q;
    if (dstudent) dstudent[r * classes + c] = (expf(log_q) - p) * grad_scale;
  }
  block_sum2(acc, unused, sh_d);
  if (threadIdx.x == 0) {
    row_loss[r] = (float)acc;
    if (is == it) atomicAdd(agree, 1u);        // an integer count: the same result in any order
  }
}

// out[0] = T^2 * mean of the row losses (fp64, fixed order); out[1]: the agreement count -> its fraction of the rows
__global__ void distill_mean_kernel(int64_t rows, float T, float* __restrict__ out) {
  __shared__ double sh[32];
  const float* row_loss = out + 2;
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < rows; i += blockDim.x) a += (double)row_loss[i];
  a = warp_sum(a);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) total += sh[k];
    const unsigned agree = *reinterpret_cast<const unsigned*>(out + 1);
    out[0] = (float)((double)T * (double)T * total / (double)rows);
    out[1] = (float)((double)agree / (double)rows);
  }
}

}  // namespace
}  // namespace simclr

using namespace simclr;

extern "C" {

int simclr_distill_xent(const float* student, const float* teacher, int64_t rows, int64_t classes, float temperature,
                        float grad_scale, float* out, float* dstudent, void* stream) {
  SIMCLR_CHECK_ARG(student && teacher && out, "distill_xent: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && rows <= INT32_MAX && classes > 0 && classes <= INT32_MAX,
                   "distill_xent: bad shape (rows %lld, classes %lld)", (long long)rows, (long long)classes);
  SIMCLR_CHECK_ARG(temperature > 0.f && temperature <= 3.0e38f, "distill_xent: temperature must be positive and finite (got %g)",
                   (double)temperature);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* agree = reinterpret_cast<unsigned*>(out + 1);
  SIMCLR_CHECK_CUDA(cudaMemsetAsync(agree, 0, sizeof(unsigned), st));
  distill_rows_kernel<<<(unsigned)rows, kRowThreads, 0, st>>>(student, teacher, (int)classes, temperature, grad_scale,
                                                              out + 2, dstudent, agree);
  SIMCLR_CHECK_LAUNCH();
  distill_mean_kernel<<<1, 1024, 0, st>>>(rows, temperature, out);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
