// Small kernels around the hot path: supervised-head loss, bias, weight
// packing for the tensor-core engine, input preparation (view split + Gaussian
// blur + cast + channel pad), error plumbing.
#include "common.cuh"

namespace simclr {

// Accumulation outputs (BN statistic sums, dW of the tensor-core wgrad) are normally zeroed by the call that
// fills them -- one cudaMemsetAsync per call, ~170 per ResNet-50 step.  A caller that zeroes them itself (one
// memset per step over pooled buffers) switches that off with simclr_set_accumulate_prezeroed(1).
static bool g_prezeroed = false;
bool accumulate_prezeroed() { return g_prezeroed; }

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

// one warp per row: loss_row = lse - sum(labels*logits); dlogits = (softmax - labels)*scale
__global__ void softmax_xent_kernel(const float* __restrict__ logits, const float* __restrict__ labels,
                                    int64_t rows, int64_t label_rows, int classes, float grad_scale,
                                    float* __restrict__ row_loss, float* __restrict__ dlogits) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* x = logits + r * classes;
  const float* l = labels + (r % label_rows) * classes;
  float m = -INFINITY;
  for (int c = lane; c < classes; c += 32) m = fmaxf(m, x[c]);
  m = warp_max(m);
  float s = 0.f, dot = 0.f;
  for (int c = lane; c < classes; c += 32) { s += expf(x[c] - m); dot = fmaf(l[c], x[c], dot); }
  s = warp_sum(s); dot = warp_sum(dot);
  const float lse = m + logf(s);
  if (lane == 0) row_loss[r] = lse - dot;
  if (dlogits) {
    const float inv = 1.f / s;
    for (int c = lane; c < classes; c += 32)
      dlogits[r * classes + c] = (expf(x[c] - m) * inv - l[c]) * grad_scale;
  }
}

__global__ void mean_kernel(const float* __restrict__ x, int64_t n, float scale, float* __restrict__ out) {
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

__global__ void bias_add_kernel(float* __restrict__ y, const float* __restrict__ b, int64_t total, int C) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    y[i] += b[i % C];
}

__global__ void bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ db, int64_t rows, int C) {
  // block per 32 channels, 8 row lanes; fixed reduction order
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ry = threadIdx.x >> 5;
  float s = 0.f;
  if (c < C) for (int64_t r = ry; r < rows; r += 8) s += dy[r * C + c];
  sh[ry][threadIdx.x & 31] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += sh[k][threadIdx.x & 31];
    db[c] = t;
  }
}

__global__ void axpy_kernel(float a, const float* __restrict__ x, float* __restrict__ y, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = fmaf(a, x[i], y[i]);
}

__global__ void l2_partial_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ part) {
  __shared__ float sh[32];
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s = fmaf(x[i], x[i], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
  }
}

template <typename Ts, typename Td>
__global__ void cast_kernel(const Ts* __restrict__ s, Td* __restrict__ d, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    d[i] = from_f<Td>(to_f<Ts>(s[i]));
}

template <typename T>
__global__ void add_inplace_kernel(T* __restrict__ a, const T* __restrict__ b, int64_t nvec) {
  constexpr int V = Vec16<T>::N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Vec16<T> x, y; x.load(a + i * V); y.load(b + i * V);
    float fx[V], fy[V]; x.unpack(fx); y.unpack(fy);
#pragma unroll
    for (int k = 0; k < V; ++k) fx[k] += fy[k];
    x.pack(fx); x.store(a + i * V);
  }
}

// fp32 HWIO [R][S][Cin][Cout] -> wf [Cout][Kp] (k=(r*S+s)*Cs+c, zero padded) and
// wd [Cin][Kdp] (k=(r*S+s)*Cout+co, zero padded to the K block).
// bf16 with 4 stored channels (the stem): k = (r*(S+1) + s+1)*4 + c, slot s' = 0 of every filter
// row zero -- S+1 slots make a filter row a whole number of 16-byte pixel pairs.
// Three-way bf16 split of an fp32 value: v = a + b + c exactly up to 2^-25 |v| (8 + 8 + 8 mantissa bits),
// a = bf16(v), b = bf16(v - a), c = bf16(v - a - b).  PART selects the term (0: the value itself).
template <typename T, int PART> __device__ __forceinline__ T pack_part(float v) {
  if (PART == 0) return from_f<T>(v);
  const float r1 = v - __bfloat162float(__float2bfloat16_rn(v));
  if (PART == 1) return from_f<T>(r1);
  return from_f<T>(r1 - __bfloat162float(__float2bfloat16_rn(r1)));
}

__global__ void split_bf16x3_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ a,
                                    __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ c, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const float r1 = v - __bfloat162float(h);
    const __nv_bfloat16 m = __float2bfloat16_rn(r1);
    a[i] = h; b[i] = m;
    c[i] = __float2bfloat16_rn(r1 - __bfloat162float(m));
  }
}

// All conv / dense layers in one launch (table row of 10 int64: w, wf, wd, R, S, Cin, Cs, Cout, Kp, Kdp).  The work
// of every layer is cut into units -- a 32x32 tile of the [K][Cout] -> [Cout][Kp] transposition (through shared
// memory, so that both the fp32 reads and the bf16 writes are coalesced), or 1024 consecutive elements of the dgrad
// operand wd (a row copy) -- and the units of all layers are dealt round-robin to the CTAs: layers differ in size by
// four orders of magnitude, one-grid-row-per-layer left the launch waiting for the blocks of the largest ones.
constexpr int PACK_MAX_LAYERS = 1024;
__device__ __forceinline__ void pack_elementwise(const long long* t, int64_t i0, int64_t i1) {
  const float* __restrict__ w = reinterpret_cast<const float*>(t[0]);
  __nv_bfloat16* __restrict__ wf = reinterpret_cast<__nv_bfloat16*>(t[1]);
  __nv_bfloat16* __restrict__ wd = reinterpret_cast<__nv_bfloat16*>(t[2]);
  const int R = (int)t[3], S = (int)t[4], Cin = (int)t[5], Cs = (int)t[6], Cout = (int)t[7], Kp = (int)t[8], Kdp = (int)t[9];
  const int64_t nf = (int64_t)Cout * Kp;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
    if (i < nf) {
      const int co = (int)(i / Kp), k = (int)(i % Kp);
      const int tap = k / Cs, c = k % Cs;
      float v = 0.f;
      if (Cs == 4) {
        const int r = tap / (S + 1), sp = tap % (S + 1);
        if (r < R && sp >= 1 && c < Cin) v = w[((int64_t)(r * S + sp - 1) * Cin + c) * Cout + co];
      } else if (tap < R * S && c < Cin) {
        v = w[((int64_t)tap * Cin + c) * Cout + co];
      }
      wf[i] = __float2bfloat16_rn(v);
    } else {
      const int64_t j = i - nf;
      const int ci = (int)(j / Kdp), k = (int)(j % Kdp);
      const int tap = k / Cout, co = k % Cout;
      wd[j] = __float2bfloat16_rn(tap < R * S ? w[((int64_t)tap * Cin + ci) * Cout + co] : 0.f);
    }
  }
}

__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const long long* __restrict__ table, int n_layers) {
  __shared__ long long ustart[PACK_MAX_LAYERS + 1];
  __shared__ float tile[32][33];
  for (int l = threadIdx.x; l < n_layers; l += blockDim.x) {
    const long long* t = table + (long long)l * 10;
    const long long Cin = t[5], Cs = t[6], Cout = t[7], Kp = t[8], Kdp = t[9];
    const long long nd = t[2] ? Cin * Kdp : 0;
    long long units;
    if (Cs == 4) units = (Cout * Kp + nd + 1023) / 1024;                    // stem layout: element-wise
    else units = ((Kp + 31) / 32) * ((Cout + 31) / 32) + (nd + 1023) / 1024;
    ustart[l + 1] = units;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ustart[0] = 0;
    for (int l = 0; l < n_layers; ++l) ustart[l + 1] += ustart[l];
  }
  __syncthreads();
  const long long total = ustart[n_layers];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (long long u = blockIdx.x; u < total; u += gridDim.x) {
    int lo = 0, hi = n_layers;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ustart[mid] <= u) lo = mid; else hi = mid; }
    const long long* t = table + (long long)lo * 10;
    const long long local = u - ustart[lo];
    const int R = (int)t[3], S = (int)t[4], Cin = (int)t[5], Cs = (int)t[6], Cout = (int)t[7], Kp = (int)t[8], Kdp = (int)t[9];
    const int64_t nf = (int64_t)Cout * Kp;
    const int64_t nd = t[2] ? (int64_t)Cin * Kdp : 0;
    if (Cs == 4) {
      const int64_t i0 = local * 1024;
      pack_elementwise(t, i0, min(i0 + 1024, nf + nd));
      continue;
    }
    const long long tiles_k = (Kp + 31) / 32, tiles_c = (Cout + 31) / 32;
    if (local < tiles_k * tiles_c) {
      const float* __restrict__ w = reinterpret_cast<const float*>(t[0]);
      __nv_bfloat16* __restrict__ wf = reinterpret_cast<__nv_bfloat16*>(t[1]);
      const int k0 = (int)(local % tiles_k) * 32, c0 = (int)(local / tiles_k) * 32;
#pragma unroll
      for (int r = ty; r < 32; r += 8) {
        const int k = k0 + r, co = c0 + tx;
        const int tap = k / Cs, c = k % Cs;
        float v = 0.f;
        if (k < Kp && tap < R * S && c < Cin && co < Cout) v = w[((int64_t)tap * Cin + c) * Cout + co];
        tile[r][tx] = v;
      }
      __syncthreads();
#pragma unroll
      for (int r = ty; r < 32; r += 8) {
        const int co = c0 + r, k = k0 + tx;
        if (co < Cout && k < Kp) wf[(int64_t)co * Kp + k] = __float2bfloat16_rn(tile[tx][r]);
      }
      __syncthreads();
    } else {
      const int64_t i0 = nf + (local - tiles_k * tiles_c) * 1024;
      pack_elementwise(t, i0, min(i0 + 1024, nf + nd));
    }
  }
}

template <typename T, int PART = 0>
__global__ void pack_weight_kernel(const float* __restrict__ w, T* __restrict__ wf, T* __restrict__ wd, int R,
                                   int S, int Cin, int Cs, int Cout, int Kp, int Kdp) {
  const int64_t nf = (int64_t)Cout * Kp;
  const int64_t nd = wd ? (int64_t)Cin * Kdp : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nf + nd; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < nf) {
      const int co = (int)(i / Kp), k = (int)(i % Kp);
      const int tap = k / Cs, c = k % Cs;
      float v = 0.f;
      if (sizeof(T) == 2 && Cs == 4) {
        const int r = tap / (S + 1), sp = tap % (S + 1);
        if (r < R && sp >= 1 && c < Cin) v = w[((int64_t)(r * S + sp - 1) * Cin + c) * Cout + co];
      } else if (tap < R * S && c < Cin) {
        v = w[((int64_t)tap * Cin + c) * Cout + co];
      }
      wf[i] = pack_part<T, PART>(v);
    } else {
      const int64_t j = i - nf;
      const int ci = (int)(j / Kdp), k = (int)(j % Kdp);
      const int tap = k / Cout, co = k % Cout;
      wd[j] = pack_part<T, PART>(tap < R * S ? w[((int64_t)tap * Cin + ci) * Cout + co] : 0.f);
    }
  }
}

// ---- input prep ------------------------------------------------------------
constexpr int MAX_TAPS = 65;
// outputs per thread along the blurred axis: (2*radius + OUT) / OUT loads per output.  The vertical pass gains from 8,
// the horizontal one loses (its lanes are OUT pixels apart)
constexpr int BLUR_OUT_H = 4, BLUR_OUT_V = 8;
constexpr int TAP_PAD = BLUR_OUT_V - 1;

// taps at wsm[TAP_PAD + i], i in [0, 2*radius]; zeros on both sides so that the sliding window of
// BLUR_OUT_H outputs can read one tap per input position without bound checks
__device__ __forceinline__ void make_taps(float* wsm, int radius, float sigma) {
  // tf2/data_util.py:338-343: exp(-x^2 / (2 sigma^2)), normalised
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < MAX_TAPS + 2 * TAP_PAD; ++i) wsm[i] = 0.f;
    for (int i = 0; i <= 2 * radius; ++i) {
      const float x = (float)(i - radius);
      const float v = expf(-(x * x) / (2.f * sigma * sigma));
      wsm[TAP_PAD + i] = v; tot += v;
    }
    for (int i = 0; i <= 2 * radius; ++i) wsm[TAP_PAD + i] /= tot;
  }
  __syncthreads();
}

// Each thread produces BLUR_OUT_H consecutive outputs along the blurred axis from one pass over the
// 2*radius + BLUR_OUT_H inputs they touch: an input is loaded once and feeds up to BLUR_OUT_H
// accumulators, the tap register file slides by one per input (the one-output-per-thread form was
// bound by its 3 loads per FMA triple).

// horizontal pass: features [B,H,W,3T] view t -> tmp [T*B,H,W,3].  One CTA per image row: the row's 3W floats of view t
// are staged in shared memory once (with `radius` zero pixels on both sides: the 'SAME' padding), then every thread
// slides BLUR_OUT_H accumulators of one channel over it -- output (w, c) is sum_j k[j] * row[(w + j)*3 + c], so in the
// flat row the window of a channel advances by 3 floats per tap.  The first version read the row straight from global
// memory: 32 lanes, 12 pixels apart, 24-byte pixels -- a different sector per lane and load (0.70 ms, L1-bound).
constexpr int BLUR_ROW_MAX = 4096;      // floats of one staged row: 3 * (W + 2*radius + BLUR_OUT_H)
__global__ void __launch_bounds__(256)
blur_h_kernel(const float* __restrict__ f, float* __restrict__ tmp, int64_t B, int H, int W, int T,
              int radius, const float* __restrict__ sigma, const uint8_t* __restrict__ sel) {
  __shared__ float wsm[MAX_TAPS + 2 * TAP_PAD];
  __shared__ float srow[BLUR_ROW_MAX];
  const int t = blockIdx.y;
  make_taps(wsm, radius, sigma[t]);
  const int64_t rows = B * H;
  const int padded = 3 * (W + 2 * radius + BLUR_OUT_H);
  const int groups = (W + BLUR_OUT_H - 1) / BLUR_OUT_H;       // per channel
  for (int64_t bh = blockIdx.x; bh < rows; bh += gridDim.x) {
    const int64_t b = bh / H;
    if (!sel[(int64_t)t * B + b]) continue;                   // uniform per CTA
    const float* row = f + bh * W * (int64_t)(3 * T) + 3 * t;
    __syncthreads();                                          // the previous row's readers are done
    for (int i = threadIdx.x; i < padded; i += blockDim.x) {
      const int w = i / 3 - radius, c = i - (i / 3) * 3;
      srow[i] = (w >= 0 && w < W) ? row[(int64_t)w * (3 * T) + c] : 0.f;
    }
    __syncthreads();
    float* dst = tmp + ((int64_t)t * rows + bh) * W * 3;
    for (int g = threadIdx.x; g < 3 * groups; g += blockDim.x) {
      const int c = g % 3, w0 = (g / 3) * BLUR_OUT_H;
      float acc[BLUR_OUT_H], k[BLUR_OUT_H];
#pragma unroll
      for (int o = 0; o < BLUR_OUT_H; ++o) { acc[o] = 0.f; k[o] = 0.f; }
      const float* src = srow + w0 * 3 + c;                   // padded pixel w0 + j  <->  image pixel w0 + j - radius
#pragma unroll 4
      for (int j = 0; j <= 2 * radius + BLUR_OUT_H - 1; ++j) {
        // output o sees input j through tap index j - o
#pragma unroll
        for (int o = BLUR_OUT_H - 1; o > 0; --o) k[o] = k[o - 1];
        k[0] = wsm[TAP_PAD + j];
        const float v = src[3 * j];
#pragma unroll
        for (int o = 0; o < BLUR_OUT_H; ++o) acc[o] = fmaf(k[o], v, acc[o]);
      }
#pragma unroll
      for (int o = 0; o < BLUR_OUT_H; ++o)
        if (w0 + o < W) dst[(w0 + o) * 3 + c] = acc[o];
    }
  }
}

// vertical pass + per-sample select + clip + cast + pad to 4 channels
template <typename To>
__global__ void blur_v_kernel(const float* __restrict__ f, const float* __restrict__ tmp, To* __restrict__ out,
                              int64_t B, int H, int W, int T, int radius, const float* __restrict__ sigma,
                              const uint8_t* __restrict__ sel, int use_blur) {
  __shared__ float wsm[MAX_TAPS + 2 * TAP_PAD];
  const int t = blockIdx.y;
  if (use_blur) make_taps(wsm, radius, sigma[t]);
  const int Hq = (H + BLUR_OUT_V - 1) / BLUR_OUT_V;
  const int64_t total = B * Hq * W;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int w = (int)(p % W);
    const int64_t bq = p / W;
    const int h0 = (int)(bq % Hq) * BLUR_OUT_V;
    const int64_t b = bq / Hq;
    float acc[BLUR_OUT_V][3];
    if (use_blur && sel[(int64_t)t * B + b]) {
      float k[BLUR_OUT_V];
#pragma unroll
      for (int o = 0; o < BLUR_OUT_V; ++o) { acc[o][0] = acc[o][1] = acc[o][2] = 0.f; k[o] = 0.f; }
      const float* col = tmp + ((((int64_t)t * B + b) * H) * W + w) * 3;
#pragma unroll 8
      for (int j = -radius; j <= radius + BLUR_OUT_V - 1; ++j) {
#pragma unroll
        for (int o = BLUR_OUT_V - 1; o > 0; --o) k[o] = k[o - 1];
        k[0] = wsm[TAP_PAD + j + radius];
        const int hh = h0 + j;
        if (hh < 0 || hh >= H) continue;
        const float* src = col + (int64_t)hh * W * 3;
        const float v0 = src[0], v1 = src[1], v2 = src[2];
#pragma unroll
        for (int o = 0; o < BLUR_OUT_V; ++o) {
          acc[o][0] = fmaf(k[o], v0, acc[o][0]); acc[o][1] = fmaf(k[o], v1, acc[o][1]); acc[o][2] = fmaf(k[o], v2, acc[o][2]);
        }
      }
    } else {
#pragma unroll
      for (int o = 0; o < BLUR_OUT_V; ++o) {
        if (h0 + o < H) {
          const float* src = f + ((b * H + h0 + o) * W + w) * (int64_t)(3 * T) + 3 * t;
          acc[o][0] = src[0]; acc[o][1] = src[1]; acc[o][2] = src[2];
        } else { acc[o][0] = acc[o][1] = acc[o][2] = 0.f; }
      }
    }
#pragma unroll
    for (int o = 0; o < BLUR_OUT_V; ++o) {
      if (h0 + o >= H) continue;
      float a0 = acc[o][0], a1 = acc[o][1], a2 = acc[o][2];
      if (use_blur) {   // tf.clip_by_value(images, 0., 1.)  (tf2/data_util.py:437)
        a0 = fminf(fmaxf(a0, 0.f), 1.f); a1 = fminf(fmaxf(a1, 0.f), 1.f); a2 = fminf(fmaxf(a2, 0.f), 1.f);
      }
      To* dst = out + ((((int64_t)t * B + b) * H + h0 + o) * W + w) * 4;
      dst[0] = from_f<To>(a0); dst[1] = from_f<To>(a1); dst[2] = from_f<To>(a2); dst[3] = from_f<To>(0.f);
    }
  }
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

int simclr_version(void) { return 100; }
const char* simclr_last_error(void) { return g_err; }

int simclr_softmax_xent(const float* logits, const float* labels, int64_t rows, int64_t label_rows,
                        int64_t classes, float grad_scale, float* loss, float* dlogits, void* stream) {
  SIMCLR_CHECK_ARG(logits && labels && loss, "softmax_xent: null pointer");
  SIMCLR_CHECK_ARG(rows > 0 && label_rows > 0 && classes > 0, "softmax_xent: bad shape");
  // row losses are staged in dlogits' tail?  No: use a small static scratch via loss+1.. -> caller gives loss[1+rows]
  cudaStream_t st = (cudaStream_t)stream;
  float* row_loss = loss + 1;
  softmax_xent_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(logits, labels, rows, label_rows, (int)classes, grad_scale, row_loss, dlogits);
  SIMCLR_CHECK_LAUNCH();
  mean_kernel<<<1, 1024, 0, st>>>(row_loss, rows, 1.f / (float)rows, loss);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bias_add(float* y, const float* bias, int64_t rows, int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(y && bias && rows > 0 && C > 0, "bias_add: bad args");
  bias_add_kernel<<<grid_for(rows * C, 256), 256, 0, (cudaStream_t)stream>>>(y, bias, rows * C, (int)C);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_bias_grad(const float* dy, float* dbias, int64_t rows, int64_t C, void* stream) {
  SIMCLR_CHECK_ARG(dy && dbias && rows > 0 && C > 0, "bias_grad: bad args");
  bias_grad_kernel<<<(unsigned)((C + 31) / 32), 256, 0, (cudaStream_t)stream>>>(dy, dbias, rows, (int)C);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_axpy(float a, const float* x, float* y, int64_t n, void* stream) {
  SIMCLR_CHECK_ARG(x && y && n > 0, "axpy: bad args");
  axpy_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(a, x, y, n);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_l2_loss(const float* x, int64_t n, float* out, void* stream) {
  SIMCLR_CHECK_ARG(x && out && n > 0, "l2_loss: bad args");
  // out needs 1 + 256 floats: out[0] result, out[1..] per-block partials
  cudaStream_t st = (cudaStream_t)stream;
  int64_t blocks = (n + 1023) / 1024; if (blocks > 256) blocks = 256;
  l2_partial_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, n, out + 1);
  SIMCLR_CHECK_LAUNCH();
  mean_kernel<<<1, 256, 0, st>>>(out + 1, blocks, 0.5f, out);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream) {
  SIMCLR_CHECK_ARG(src && dst && n > 0, "cast: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = grid_for(n, 256);
  if (src_dtype == SIMCLR_F32 && dst_dtype == SIMCLR_BF16) cast_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)src, (bf16*)dst, n);
  else if (src_dtype == SIMCLR_BF16 && dst_dtype == SIMCLR_F32) cast_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)src, (float*)dst, n);
  else if (src_dtype == SIMCLR_F32 && dst_dtype == SIMCLR_F32) cast_kernel<float, float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, n);
  else if (src_dtype == SIMCLR_BF16 && dst_dtype == SIMCLR_BF16) cast_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)src, (bf16*)dst, n);
  else { set_error("cast: unknown dtypes"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_add_inplace(void* a, const void* b, int dtype, int64_t n, void* stream) {
  SIMCLR_CHECK_ARG(a && b && n > 0, "add_inplace: bad args");
  SIMCLR_CHECK_ARG(aligned16(a) && aligned16(b), "add_inplace: pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32) {
    SIMCLR_CHECK_ARG(n % 4 == 0, "add_inplace: n must be a multiple of 4");
    add_inplace_kernel<float><<<grid_for(n / 4, 256), 256, 0, st>>>((float*)a, (const float*)b, n / 4);
  } else if (dtype == SIMCLR_BF16) {
    SIMCLR_CHECK_ARG(n % 8 == 0, "add_inplace: n must be a multiple of 8");
    add_inplace_kernel<bf16><<<grid_for(n / 8, 256), 256, 0, st>>>((bf16*)a, (const bf16*)b, n / 8);
  } else { set_error("add_inplace: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_pack_conv_weight(const float* w_hwio, void* wf, void* wd, int dtype, int64_t R, int64_t S, int64_t Cin,
                            int64_t Cs, int64_t Cout, int64_t Kp, void* stream) {
  SIMCLR_CHECK_ARG(w_hwio && wf, "pack_conv_weight: null pointer");
  const int64_t Sk = (dtype == SIMCLR_BF16 && Cs == 4) ? S + 1 : S;      // bf16 stem: S+1 slots per filter row
  SIMCLR_CHECK_ARG(R > 0 && S > 0 && Cin > 0 && Cs >= Cin && Cout > 0 && Kp >= R * Sk * Cs,
                   "pack_conv_weight: bad shape (Kp=%lld < %lld)", (long long)Kp, (long long)(R * Sk * Cs));
  SIMCLR_CHECK_ARG(wd == nullptr || Cs == Cin, "pack_conv_weight: dgrad copy needs Cs == Cin");
  cudaStream_t st = (cudaStream_t)stream;
  const int kbe = dtype == SIMCLR_BF16 ? 64 : 32;
  const int64_t Kdp = (R * S * Cout + kbe - 1) / kbe * kbe;
  SIMCLR_CHECK_ARG(Kp % kbe == 0, "pack_conv_weight: Kp must be a multiple of %d", kbe);
  const int64_t total = Cout * Kp + (wd ? Cin * Kdp : 0);
  const unsigned grid = grid_for(total, 256);
  if (dtype == SIMCLR_BF16) pack_weight_kernel<bf16><<<grid, 256, 0, st>>>(w_hwio, (bf16*)wf, (bf16*)wd, (int)R, (int)S, (int)Cin, (int)Cs, (int)Cout, (int)Kp, (int)Kdp);
  else if (dtype == SIMCLR_F32) pack_weight_kernel<float><<<grid, 256, 0, st>>>(w_hwio, (float*)wf, (float*)wd, (int)R, (int)S, (int)Cin, (int)Cs, (int)Cout, (int)Kp, (int)Kdp);
  else { set_error("pack_conv_weight: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_pack_conv_weights_multi(const void* table_dev, int64_t n_layers, void* stream) {
  SIMCLR_CHECK_ARG(table_dev && n_layers > 0 && n_layers <= PACK_MAX_LAYERS, "pack_conv_weights_multi: 1..%d layers", PACK_MAX_LAYERS);
  pack_weights_multi_kernel<<<(unsigned)(num_sms() * 8), 256, 0, (cudaStream_t)stream>>>((const long long*)table_dev, (int)n_layers);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_set_accumulate_prezeroed(int on) {
  const int prev = simclr::g_prezeroed ? 1 : 0;
  simclr::g_prezeroed = on != 0;
  return prev;
}

int simclr_memset_zero(void* p, int64_t bytes, void* stream) {
  SIMCLR_CHECK_ARG(p && bytes > 0, "memset_zero: bad arguments");
  SIMCLR_CHECK_CUDA(cudaMemsetAsync(p, 0, (size_t)bytes, (cudaStream_t)stream));
  return SIMCLR_OK;
}

int simclr_pack_conv_weight_part(const float* w_hwio, void* wf, void* wd, int part, int64_t R, int64_t S, int64_t Cin,
                                 int64_t Cs, int64_t Cout, int64_t Kp, void* stream) {
  SIMCLR_CHECK_ARG(w_hwio && wf, "pack_conv_weight_part: null pointer");
  SIMCLR_CHECK_ARG(part >= 0 && part <= 2, "pack_conv_weight_part: part must be 0, 1 or 2");
  SIMCLR_CHECK_ARG(R > 0 && S > 0 && Cin > 0 && Cs >= Cin && Cout > 0 && Kp % 64 == 0, "pack_conv_weight_part: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t Kdp = (R * S * Cout + 63) / 64 * 64;
  const int64_t total = Cout * Kp + (wd ? Cin * Kdp : 0);
  const unsigned grid = grid_for(total, 256);
#define PACK(P) pack_weight_kernel<bf16, P><<<grid, 256, 0, st>>>(w_hwio, (bf16*)wf, (bf16*)wd, (int)R, (int)S, (int)Cin, (int)Cs, (int)Cout, (int)Kp, (int)Kdp)
  if (part == 0) PACK(0); else if (part == 1) PACK(1); else PACK(2);
#undef PACK
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_split_bf16x3(const float* x, void* a, void* b, void* c, int64_t n, void* stream) {
  SIMCLR_CHECK_ARG(x && a && b && c && n > 0, "split_bf16x3: bad arguments");
  split_bf16x3_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, (bf16*)a, (bf16*)b, (bf16*)c, n);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_input_prep(const float* features, void* out, int dtype, int64_t B, int64_t H, int64_t W, int64_t T,
                      int use_blur, int64_t blur_kernel_size, const float* sigma, const uint8_t* selector,
                      float* tmp, void* stream) {
  SIMCLR_CHECK_ARG(features && out, "input_prep: null pointer");
  SIMCLR_CHECK_ARG(B > 0 && H > 0 && W > 0 && T > 0, "input_prep: bad shape");
  const int radius = (int)(blur_kernel_size / 2);     // tf.cast(kernel_size / 2, int32), tf2/data_util.py:338
  if (use_blur) {
    SIMCLR_CHECK_ARG(sigma && selector && tmp, "input_prep: blur needs sigma, selector, tmp");
    SIMCLR_CHECK_ARG(2 * radius + 1 <= MAX_TAPS, "input_prep: blur kernel too large (%d taps > %d)", 2 * radius + 1, MAX_TAPS);
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = B * H * W / BLUR_OUT_H + 1;
  int64_t bx = (total + 255) / 256; const int64_t cap = (int64_t)num_sms() * 8; if (bx > cap) bx = cap;
  dim3 grid((unsigned)bx, (unsigned)T);
  if (use_blur) {
    SIMCLR_CHECK_ARG(3 * (W + 2 * radius + BLUR_OUT_H) <= BLUR_ROW_MAX, "input_prep: image too wide for the blur row buffer (W=%lld)", (long long)W);
    int64_t rows_x = B * H; if (rows_x > (int64_t)num_sms() * 16) rows_x = (int64_t)num_sms() * 16;
    blur_h_kernel<<<dim3((unsigned)rows_x, (unsigned)T), 256, 0, st>>>(features, tmp, B, (int)H, (int)W, (int)T, radius, sigma, selector);
    SIMCLR_CHECK_LAUNCH();
  }
  if (dtype == SIMCLR_F32) blur_v_kernel<float><<<grid, 256, 0, st>>>(features, tmp, (float*)out, B, (int)H, (int)W, (int)T, radius, sigma, selector, use_blur);
  else if (dtype == SIMCLR_BF16) blur_v_kernel<bf16><<<grid, 256, 0, st>>>(features, tmp, (bf16*)out, B, (int)H, (int)W, (int)T, radius, sigma, selector, use_blur);
  else { set_error("input_prep: unknown dtype"); return SIMCLR_ERR_INVALID_ARG; }
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"
