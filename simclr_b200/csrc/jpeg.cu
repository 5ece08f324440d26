// Baseline JPEG decode on the device, bit-exact with libjpeg-turbo's default decompression as Pillow runs it
// (JDCT_ISLOW, fancy upsampling, jdcolor.c tables); the arithmetic is restated in oracle/jpeg.py.  Three kernels:
//   1. Huffman: one thread per entropy-coded segment (an image, or one restart interval), int16 coefficients in
//      natural order into a zeroed workspace.  The bit reader never reads outside [start, end) of its segment: past
//      the end, or at a marker, it supplies zero bits, and consuming any of them sets the image's error flag.
//   2. Dequantise + jpeg_idct_islow: one thread per 8x8 block, uint8 component planes padded to whole MCUs.
//   3. Fancy upsampling + YCbCr -> RGB: one thread per output pixel, into the caller's packed HWC buffer.
// The host (simclr_b200/jpeg.py) parses and validates the headers, builds the Huffman lookup tables and the image /
// segment descriptors; field layouts are in include/simclr_b200.h.
#include "common.cuh"

namespace simclr {
namespace {

// image descriptor fields (int64 each), see simclr_jpeg_decode in the header
enum {
  D_OUT = 0, D_H, D_W, D_NCOMP, D_HMAX, D_VMAX, D_MCUX, D_MCUY, D_BLK, D_NBLK,
  D_COFF = 10, D_BW = 13, D_BH = 16, D_HS = 19, D_VS = 22, D_QT = 25, D_DC = 28, D_AC = 31, D_FIELDS = 40
};
enum { S_IMG = 0, S_START, S_END, S_MCU0, S_NMCU, S_FIELDS = 8 };
// Huffman table: uint16 look[512] ((length << 8) | symbol for codes of <= 9 bits, 0 otherwise), int32 maxcode[18],
// int32 valoff[18] (index of the first symbol of each length minus its first code), uint8 vals[256]
constexpr int HT_MAXCODE = 1024, HT_VALOFF = 1096, HT_VALS = 1168;

__constant__ uint8_t kNatural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63};

struct BitReader {
  const uint8_t* p;
  int64_t pos, end;
  uint64_t buf;                 // MSB-aligned
  int nbits;
  int64_t real, used;           // bits of segment data appended / bits consumed

  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t b = 0;
      if (pos < end) {
        const uint32_t c = p[pos];
        if (c != 0xFF) { b = c; ++pos; real += 8; }
        else if (pos + 1 < end && p[pos + 1] == 0) { b = 0xFF; pos += 2; real += 8; }   // stuffed 0xFF
        else pos = end;                                 // a marker (or a lone 0xFF at the end): the data ends
      }
      buf |= (uint64_t)b << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)(buf >> (64 - n)); }
  __device__ __forceinline__ void skip(int n) { buf <<= n; nbits -= n; used += n; }
};

__device__ __forceinline__ int extend(uint32_t v, int s) { return v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

__device__ __forceinline__ int huff_decode(BitReader& br, const uint8_t* __restrict__ t, bool& bad) {
  const uint32_t pk = br.peek(16);
  const uint32_t e = reinterpret_cast<const uint16_t*>(t)[pk >> 7];
  if (e >> 8) { br.skip(e >> 8); return e & 255; }
  const int32_t* maxcode = reinterpret_cast<const int32_t*>(t + HT_MAXCODE);
  const int32_t* valoff = reinterpret_cast<const int32_t*>(t + HT_VALOFF);
#pragma unroll 1
  for (int l = 10; l <= 16; ++l) {
    const int32_t c = (int32_t)(pk >> (16 - l));
    if (c <= maxcode[l]) { br.skip(l); return t[HT_VALS + ((c + valoff[l]) & 255)]; }
  }
  bad = true;
  return 0;
}

__global__ void __launch_bounds__(32)
huffman_kernel(const int64_t* __restrict__ images, const int64_t* __restrict__ segs, int64_t nseg, int lanes,
               const uint8_t* __restrict__ tables, const uint8_t* __restrict__ data, int16_t* __restrict__ coef,
               uint8_t* __restrict__ error) {
  if ((int)threadIdx.x >= lanes) return;
  const int64_t sid = (int64_t)blockIdx.x * lanes + threadIdx.x;
  if (sid >= nseg) return;
  const int64_t* s = segs + sid * S_FIELDS;
  const int64_t img = s[S_IMG];
  const int64_t* d = images + img * D_FIELDS;
  BitReader br{data, s[S_START], s[S_END], 0, 0, 0, 0};
  const int ncomp = (int)d[D_NCOMP], mcux = (int)d[D_MCUX];
  const int64_t blk0 = d[D_BLK];
  int pred[3] = {0, 0, 0};
  bool bad = false;
  const int64_t m_end = s[S_MCU0] + s[S_NMCU];
  for (int64_t m = s[S_MCU0]; m < m_end && !bad; ++m) {
    const int my = (int)(m / mcux), mx = (int)(m - (int64_t)my * mcux);
    for (int c = 0; c < ncomp && !bad; ++c) {
      const int hs = (int)d[D_HS + c], vs = (int)d[D_VS + c], bw = (int)d[D_BW + c];
      const uint8_t* dc = tables + d[D_DC + c];
      const uint8_t* ac = tables + d[D_AC + c];
      for (int v = 0; v < vs && !bad; ++v) {
        for (int h = 0; h < hs && !bad; ++h) {
          int16_t* blk = coef + (blk0 + d[D_COFF + c] + (int64_t)(my * vs + v) * bw + mx * hs + h) * 64;
          if (br.nbits < 32) br.fill();
          const int t = huff_decode(br, dc, bad) & 15;
          if (t) { pred[c] += extend(br.peek(t), t); br.skip(t); }
          blk[0] = (int16_t)pred[c];
          for (int k = 1; k < 64; ++k) {
            if (br.nbits < 32) br.fill();
            const int rs = huff_decode(br, ac, bad);
            const int r = rs >> 4, sz = rs & 15;
            if (sz) {
              k += r;
              if (k > 63) { bad = true; break; }
              blk[kNatural[k]] = (int16_t)extend(br.peek(sz), sz);
              br.skip(sz);
            } else {
              if (r != 15) break;
              k += 15;
            }
          }
        }
      }
    }
  }
  if (bad || br.used > br.real) error[img] = 1;
}

// ---- jpeg_idct_islow (jidctint.c) ------------------------------------------------------------------------------
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172

template <int SHIFT>
__device__ __forceinline__ void idct_1d(const int* x, int* o) {
  int z2 = x[2], z3 = x[6];
  int z1 = (z2 + z3) * FIX_0_541196100;
  const int tmp2 = z1 + z3 * -FIX_1_847759065;
  const int tmp3 = z1 + z2 * FIX_0_765366865;
  const int tmp0 = (x[0] + x[4]) * (1 << CONST_BITS);
  const int tmp1 = (x[0] - x[4]) * (1 << CONST_BITS);
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  int t0 = x[7], t1 = x[5], t2 = x[3], t3 = x[1];
  z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2;
  int z4 = t1 + t3;
  const int z5 = (z3 + z4) * FIX_1_175875602;
  t0 *= FIX_0_298631336; t1 *= FIX_2_053119869; t2 *= FIX_3_072711026; t3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5; z4 = z4 * -FIX_0_390180644 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  constexpr int R = 1 << (SHIFT - 1);
  o[0] = (tmp10 + t3 + R) >> SHIFT; o[7] = (tmp10 - t3 + R) >> SHIFT;
  o[1] = (tmp11 + t2 + R) >> SHIFT; o[6] = (tmp11 - t2 + R) >> SHIFT;
  o[2] = (tmp12 + t1 + R) >> SHIFT; o[5] = (tmp12 - t1 + R) >> SHIFT;
  o[3] = (tmp13 + t0 + R) >> SHIFT; o[4] = (tmp13 - t0 + R) >> SHIFT;
}

// the post-IDCT range-limit table of jdmaster.c: 10-bit wrap-around, then clamp(x + 128) to [0, 255]
__device__ __forceinline__ uint32_t range_limit(int v) { return (uint32_t)min(max((((v + 512) & 1023) - 512) + 128, 0), 255); }

constexpr int IDCT_T = 128;

__global__ void __launch_bounds__(IDCT_T)
idct_kernel(const int64_t* __restrict__ images, const uint8_t* __restrict__ tables, const int16_t* __restrict__ coef,
            uint8_t* __restrict__ planes) {
  const int64_t* d = images + (int64_t)blockIdx.y * D_FIELDS;
  const int64_t b = (int64_t)blockIdx.x * IDCT_T + threadIdx.x;
  if (b >= d[D_NBLK]) return;
  const int c = (d[D_NCOMP] == 3 && b >= d[D_COFF + 2]) ? 2 : (d[D_NCOMP] == 3 && b >= d[D_COFF + 1]) ? 1 : 0;
  const int64_t lb = b - d[D_COFF + c];
  const int bw = (int)d[D_BW + c];
  const int by = (int)(lb / bw), bx = (int)(lb - (int64_t)by * bw);
  const uint16_t* q = reinterpret_cast<const uint16_t*>(tables + d[D_QT + c]);
  const int64_t gb = d[D_BLK] + b;
  const uint4* src = reinterpret_cast<const uint4*>(coef + gb * 64);
  int ws[64];
#pragma unroll
  for (int r = 0; r < 8; ++r) {                      // dequantise (natural order: row r = vertical frequency)
    const uint4 v = src[r];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ws[r * 8 + 2 * k] = (int)(int16_t)(w[k] & 0xffff) * (int)q[r * 8 + 2 * k];
      ws[r * 8 + 2 * k + 1] = (int)(int16_t)(w[k] >> 16) * (int)q[r * 8 + 2 * k + 1];
    }
  }
#pragma unroll
  for (int col = 0; col < 8; ++col) {                // pass 1: columns (an all-zero AC column gives DC << PASS1_BITS,
    int x[8], o[8];                                  //  which the full pass computes exactly as well)
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = ws[k * 8 + col];
    idct_1d<CONST_BITS - PASS1_BITS>(x, o);
#pragma unroll
    for (int k = 0; k < 8; ++k) ws[k * 8 + col] = o[k];
  }
  uint8_t* out = planes + (d[D_BLK] + d[D_COFF + c]) * 64 + (int64_t)by * 8 * (bw * 8) + bx * 8;
#pragma unroll
  for (int r = 0; r < 8; ++r) {                      // pass 2: rows, descale by 3 more bits, range limit
    int o[8];
    idct_1d<CONST_BITS + PASS1_BITS + 3>(ws + r * 8, o);
    const uint32_t lo = range_limit(o[0]) | range_limit(o[1]) << 8 | range_limit(o[2]) << 16 | range_limit(o[3]) << 24;
    const uint32_t hi = range_limit(o[4]) | range_limit(o[5]) << 8 | range_limit(o[6]) << 16 | range_limit(o[7]) << 24;
    *reinterpret_cast<uint2*>(out + (int64_t)r * bw * 8) = make_uint2(lo, hi);
  }
}

// ---- fancy upsampling (jdsample.c) + YCbCr -> RGB (jdcolor.c) --------------------------------------------------
constexpr int COLOR_T = 256;

struct Plane {
  const uint8_t* p;
  int stride, w, h;           // w, h: the component's downsampled size (its real samples)
  __device__ __forceinline__ int at(int y, int x) const { return p[(int64_t)min(max(y, 0), h - 1) * stride + min(max(x, 0), w - 1)]; }
};

// chroma sample of output pixel (y, x) for luma sampling (hmax, vmax) over 1x1 chroma
__device__ __forceinline__ int upsample(const Plane& c, int hmax, int vmax, int y, int x) {
  if (hmax == 1 && vmax == 1) return c.at(y, x);
  if (hmax == 1) {                                  // h1v2: always the triangle filter, biases +1 / +2
    const int j = y >> 1;
    return (y & 1) ? (3 * c.at(j, x) + c.at(j + 1, x) + 2) >> 2 : (3 * c.at(j, x) + c.at(j - 1, x) + 1) >> 2;
  }
  const int i = x >> 1;
  if (c.w <= 2) return c.at(vmax == 2 ? y >> 1 : y, i);            // libjpeg-turbo's plain upsampler
  if (vmax == 1) {                                  // h2v1: biases +1 / +2, edge columns copied
    if (x & 1) return i == c.w - 1 ? c.at(y, i) : (3 * c.at(y, i) + c.at(y, i + 1) + 2) >> 2;
    return i == 0 ? c.at(y, 0) : (3 * c.at(y, i) + c.at(y, i - 1) + 1) >> 2;
  }
  const int j = y >> 1, jf = (y & 1) ? j + 1 : j - 1;               // h2v2: column sums 3 * near + far row
  const int s = 3 * c.at(j, i) + c.at(jf, i);
  if (x & 1) return i == c.w - 1 ? (4 * s + 7) >> 4 : (3 * s + 3 * c.at(j, i + 1) + c.at(jf, i + 1) + 7) >> 4;
  return i == 0 ? (4 * s + 8) >> 4 : (3 * s + 3 * c.at(j, i - 1) + c.at(jf, i - 1) + 8) >> 4;
}

__global__ void __launch_bounds__(COLOR_T)
color_kernel(const int64_t* __restrict__ images, const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  const int64_t* d = images + (int64_t)blockIdx.y * D_FIELDS;
  const int H = (int)d[D_H], W = (int)d[D_W];
  const int64_t p = (int64_t)blockIdx.x * COLOR_T + threadIdx.x;
  if (p >= (int64_t)H * W) return;
  const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
  const uint8_t* base = planes + d[D_BLK] * 64;
  const int yv = base[(int64_t)y * (d[D_BW] * 8) + x];
  uint8_t* o = out + d[D_OUT] + p * 3;
  if (d[D_NCOMP] == 1) { o[0] = o[1] = o[2] = (uint8_t)yv; return; }
  const int hmax = (int)d[D_HMAX], vmax = (int)d[D_VMAX];
  const int cw = (W + hmax - 1) / hmax, ch = (H + vmax - 1) / vmax;
  const Plane cb{base + d[D_COFF + 1] * 64, (int)d[D_BW + 1] * 8, cw, ch};
  const Plane cr{base + d[D_COFF + 2] * 64, (int)d[D_BW + 2] * 8, cw, ch};
  const int xb = upsample(cb, hmax, vmax, y, x) - 128, xr = upsample(cr, hmax, vmax, y, x) - 128;
  constexpr int HALF = 1 << 15;
  o[0] = (uint8_t)min(max(yv + ((91881 * xr + HALF) >> 16), 0), 255);
  o[1] = (uint8_t)min(max(yv + ((-46802 * xr - 22554 * xb + HALF) >> 16), 0), 255);
  o[2] = (uint8_t)min(max(yv + ((116130 * xb + HALF) >> 16), 0), 255);
}

}  // namespace
}  // namespace simclr

using namespace simclr;

extern "C" int simclr_jpeg_decode(const int64_t* images, int64_t n, const int64_t* segments, int64_t nseg,
                                  const uint8_t* tables, const uint8_t* data, int64_t total_blocks, int64_t max_blocks,
                                  int64_t max_pixels, void* workspace, size_t workspace_bytes, uint8_t* out,
                                  uint8_t* error, void* stream) {
  SIMCLR_CHECK_ARG(images && segments && tables && data && workspace && out && error, "jpeg_decode: null pointer");
  SIMCLR_CHECK_ARG(n > 0 && n <= 65535 && nseg >= n && total_blocks > 0 && max_blocks > 0 && max_pixels > 0,
                   "jpeg_decode: bad sizes");
  SIMCLR_CHECK_ARG(workspace_bytes >= (size_t)total_blocks * 192 && aligned16(workspace), "jpeg_decode: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int16_t* coef = reinterpret_cast<int16_t*>(workspace);
  uint8_t* planes = reinterpret_cast<uint8_t*>(workspace) + total_blocks * 128;
  SIMCLR_CHECK_CUDA(cudaMemsetAsync(coef, 0, (size_t)total_blocks * 128, st));
  SIMCLR_CHECK_CUDA(cudaMemsetAsync(error, 0, (size_t)n, st));
  // Spread the segments over as many warps as the GPU can issue from at once: the decode of one segment is a
  // serial chain, so a warp with fewer active lanes finishes its lanes sooner.
  const int64_t slots = 4LL * num_sms();
  const int lanes = (int)std::min<int64_t>(32, std::max<int64_t>(1, (nseg + slots - 1) / slots));
  huffman_kernel<<<(unsigned)((nseg + lanes - 1) / lanes), 32, 0, st>>>(images, segments, nseg, lanes, tables, data,
                                                                       coef, error);
  SIMCLR_CHECK_LAUNCH();
  idct_kernel<<<dim3((unsigned)((max_blocks + IDCT_T - 1) / IDCT_T), (unsigned)n), IDCT_T, 0, st>>>(images, tables, coef, planes);
  SIMCLR_CHECK_LAUNCH();
  color_kernel<<<dim3((unsigned)((max_pixels + COLOR_T - 1) / COLOR_T), (unsigned)n), COLOR_T, 0, st>>>(images, planes, out);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}
