// wgmma implicit-GEMM engine for conv fprop / dgrad / wgrad and the dense
// layers (tf2/resnet.py:183-208, tf2/model.py:143-151).
//
// One persistent, warp-specialised kernel per GEMM flavour:
//   warps 0-3  consumer     one warpgroup issues wgmma (two m64 halves per 128-row tile, fp32
//                           accumulators in registers) and runs the epilogue -> global
//   warp  4    TMA producer weights / dY tiles (and activations for 1x1 stride-1)
//   warps 5-8  gather       im2col rows of NHWC activations -> 128B-swizzled smem
// Pipeline: smem full/empty mbarriers (producers <-> consumer); the producers run ahead into
// the next tile while the consumer drains the accumulators.  Tiles: 128 x BN x 128 bytes of K
// per stage, BN <= 128 (a 128 x 128 fp32 accumulator is 128 registers per consumer thread).
#include "tc_common.cuh"

namespace simclr {
namespace tc {
namespace {

constexpr int A_STAGE_BYTES = 128 * 128;     // 128 rows x 128 B
constexpr int PIPE_BYTES = 192 * 1024;
constexpr int EPI_THREADS = 128;     // the consumer warpgroup
constexpr int AUX_T0 = 160;          // first thread after the consumer warpgroup and the TMA warp
constexpr int GATHER_THREADS = 128;  // 4 gather warps (the consumer's accumulators need the register file)
constexpr int STATS_THREADS = 128;   // 4 statistics warps (TMA-fed fprop)
constexpr int GROWS = GATHER_THREADS / 8;   // tile rows covered by one pass of the gather threads (8 threads per row)
constexpr int GPT = 128 / GROWS;            // 16-byte pieces per gather thread per stage
constexpr int igemm_threads(bool a_tma, bool stats) { return a_tma ? (stats ? AUX_T0 + STATS_THREADS : AUX_T0) : AUX_T0 + GATHER_THREADS; }
constexpr int wgrad_threads(bool a_tma) { return a_tma ? AUX_T0 : AUX_T0 + GATHER_THREADS; }
// A CTA's warps are spread over the SM's four 16K-register sub-partitions: with the 9 warps of the gather-fed kernels
// one sub-partition holds 3, which caps a thread at 168 registers, and their 128-column accumulators spill a little.

template <int BN> struct Tile {
  static constexpr int B_STAGE_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = PIPE_BYTES / STAGE_BYTES;
  static constexpr int EPI_BYTES = 2 * A_STAGE_BYTES;           // two [128 rows][128 B] store staging tiles
  static constexpr int GATHER_DEPTH = STAGES > 4 ? 4 : STAGES - 1;   // cp.async groups in flight per thread
  static constexpr size_t SMEM_BYTES = 1024 /*align*/ + (size_t)STAGES * STAGE_BYTES + EPI_BYTES + 256 /*barriers*/;
};

// wgrad work item: 128 k-rows x BN output channels x a run of pixel blocks
template <int BN> struct WTile {
  static constexpr int A_BYTES = A_STAGE_BYTES;
  static constexpr int B_STAGE_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = PIPE_BYTES / STAGE_BYTES;
  static constexpr int GATHER_DEPTH = STAGES > 4 ? 4 : STAGES - 1;
  static constexpr size_t SMEM_BYTES = 1024 + (size_t)STAGES * STAGE_BYTES + 2 * A_STAGE_BYTES + 256;
};

struct Geom {
  const void* src;     // gathered tensor: X (fprop/wgrad) or dY (dgrad), NHWC
  void* out;
  int mode;            // 0: out pixel -> in pixel = p*stride - pad + r ; 1 (dgrad): (p + pad - r)/stride
  int H, W, C;         // dims of the gathered tensor
  int R, S, RS, stride, stride_w, pad_h, pad_w;   // stride: rows (and columns unless stride_w differs: stem pixel pairs)
  int s2;              // stem K order: S+1 slots of 4 channels per filter row (0: ordinary (r, s, c) order)
  FastDiv dPQ, dQ, dC, dS;
  long long M;         // GEMM rows (pixels)
  int n_out, ldc;      // valid output columns, output row stride (elements)
  int num_kb;          // K blocks (fprop/dgrad) or pixel blocks (wgrad)
  int tiles_m, tiles_n;
  // wgrad only
  int Cin, Cout, splits, kb_per_split;
  float* ws;           // splits > 1: per-split partials ([splits][ws_rows][Cout] or [splits][dW]), summed in split order
  long long ws_stride; // floats per split partial
  // strided-dgrad parity classes: taps from a table, output rows scattered with stride `os`
  int use_tab, cblocks;
  int P, Q;            // GEMM-row pixel grid (wgrad: incremental pixel walk)
  int adv_p, adv_q;    // pixels-per-stage / Q and % Q
  int tap_sign;        // +1: source = base + (r, s) (fprop / wgrad / tables); -1: base - (r, s) (stride-1 dgrad)
  int tab_r[9], tab_s[9], tab_kcol[9];
  int os, oh0, ow0, OH, OW;
  // TMA im2col feed of the gathered operand: base pixel of GEMM row (n, p, q) is
  // (q*stride + im_base, p*stride + im_base); the tap goes into the instruction's filter offsets
  int im2col, im_base, im_nimg;
  int accum;           // fp32 outputs only: add into `out` (TMA reduce-add / atomics) instead of storing (tc3 passes)
};

template <typename T> struct Elt;
template <> struct Elt<__nv_bfloat16> { static constexpr bool TF32 = false; static constexpr int KBE = 64; static constexpr int CH = 8; };
template <> struct Elt<float> { static constexpr bool TF32 = true; static constexpr int KBE = 32; static constexpr int CH = 4; };

struct Pipe { int stage; uint32_t phase; };
template <int STAGES> __device__ __forceinline__ void advance(Pipe& p) {
  if (++p.stage == STAGES) { p.stage = 0; p.phase ^= 1; }
}

// Per-K-block tap decode shared by the gather loops: K index -> (tap, channel) -> source offset
// (dr, ds) relative to the row's base pixel.  Done once per stage per thread; the per-row work is
// then two adds, two unsigned bound checks and one 64-bit multiply-add.
struct TapRef { int dr, ds; bool ok; };
__device__ __forceinline__ TapRef decode_tap(const Geom& g, uint32_t tap) {
  TapRef t;
  t.ok = (int)tap < g.RS;
  if (g.use_tab) {
    const int ti = t.ok ? (int)tap : 0;
    t.dr = g.tab_r[ti]; t.ds = g.tab_s[ti];
  } else {
    uint32_t r, s; g.dS.divmod(tap, r, s);
    t.dr = g.tap_sign * (int)r; t.ds = g.tap_sign * (int)s;
  }
  return t;
}

template <typename To>
__device__ __forceinline__ void store_row32(To* dst, const uint32_t* acc, int valid, bool vec_ok);
template <>
__device__ __forceinline__ void store_row32<float>(float* dst, const uint32_t* acc, int valid, bool vec_ok) {
  if (valid >= 32 && vec_ok) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      reinterpret_cast<uint4*>(dst)[i] = make_uint4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) if (i < valid) dst[i] = __uint_as_float(acc[i]);
  }
}
template <>
__device__ __forceinline__ void store_row32<__nv_bfloat16>(__nv_bfloat16* dst, const uint32_t* acc, int valid, bool vec_ok) {
  if (valid >= 32 && vec_ok) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 h = __floats2bfloat162_rn(__uint_as_float(acc[8 * i + 2 * j]), __uint_as_float(acc[8 * i + 2 * j + 1]));
        w[j] = *reinterpret_cast<uint32_t*>(&h);
      }
      reinterpret_cast<uint4*>(dst)[i] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) if (i < valid) dst[i] = __float2bfloat16_rn(__uint_as_float(acc[i]));
  }
}

// One arrival per warp: 32 lanes arriving on the same mbarrier serialise in the LSU.
__device__ __forceinline__ void warp_arrive(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

struct SmemCtl {
  uint64_t* full; uint64_t* empty;
  uint64_t* sfull; uint64_t* sfree;   // staging tile handed to / returned by the statistics warps
  uint8_t* epi;     // 2 x [128][128 B] staging tiles for the TMA-store epilogue
};
template <int STAGES>
__device__ __forceinline__ SmemCtl carve(uint8_t* base, int stage_bytes) {
  SmemCtl c;
  c.epi = base + (size_t)STAGES * stage_bytes;
  uint64_t* b = reinterpret_cast<uint64_t*>(c.epi + 2 * A_STAGE_BYTES);
  c.full = b; c.empty = b + STAGES;
  c.sfull = b + 2 * STAGES; c.sfree = b + 2 * STAGES + 2;
  return c;
}

// ===========================================================================
// fprop / dgrad / dense:  out[M][n_out] = gather(src)[M][K] * Wk[n_out][K]^T
// ===========================================================================
template <typename T, typename To, int BN, bool A_TMA, bool SMALLC, bool TMA_EPI, bool STATS>
__global__ void __launch_bounds__(igemm_threads(A_TMA, STATS), 1)
igemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
             const __grid_constant__ CUtensorMap tmap_out, const Geom g, double* __restrict__ bn_sums) {
  using TL = Tile<BN>;
  constexpr int STAGES = TL::STAGES;
  constexpr bool TF32 = Elt<T>::TF32;
  constexpr int KBE = Elt<T>::KBE;
  constexpr int CH = Elt<T>::CH;
  constexpr int NF = BN / 2;                          // accumulator registers per thread and m64 half

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const SmemCtl ctl = carve<STAGES>(smem, TL::STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&ctl.full[s], A_TMA ? 1 : 1 + GATHER_THREADS / 32);
      mbar_init(&ctl.empty[s], EPI_THREADS / 32);
    }
    for (int a = 0; a < 2; ++a) { mbar_init(&ctl.sfull[a], 1); mbar_init(&ctl.sfree[a], STATS_THREADS / 32); }
    fence_barrier_init();
  }
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmap_b);
    if (A_TMA) tma_prefetch_desc(&tmap_a);
    if (TMA_EPI) tma_prefetch_desc(&tmap_out);
  }
  // With TMA-fed activations warps 5-8 have no gather to do: they take the BatchNorm statistics off the
  // epilogue's critical path (short-K 1x1 layers are epilogue-bound).
  constexpr bool STATS_WARPS = STATS && A_TMA;
  constexpr int BOX_COLS = 128 / (int)sizeof(To);     // 64 (bf16) / 32 (fp32) output columns per staged tile
  constexpr int BOXES = BN / BOX_COLS;
  constexpr int CPC = 16 / (int)sizeof(To);           // columns per 16-byte chunk: 8 (bf16) / 4 (fp32)
  __syncthreads();
  const int num_tiles = g.tiles_m * g.tiles_n;

  if (warp < 4) {
    // ------------------------------ consumer: MMA + epilogue ------------------------------
    // Descriptor low words are running 32-bit sums (one uniform add per MMA); a stage is handed back to the
    // producers once the wgmma group after it has been issued and it has retired (one group in flight).
    constexpr uint32_t HI = desc_hi_sw128(1024);
    const uint32_t smem_lo = uniform_u32(desc_lo(smem_u32(smem), 16));
    const bool all_rows[2][2] = {{true, true}, {true, true}};   // rows >= M hold exact zeros / are clipped
    float acc[2][NF];
    Pipe pp{0, 0};
    To* out = reinterpret_cast<To*>(g.out);
    uint32_t box_ctr = 0;                                // counts staged ("live") boxes only
    // fused BatchNorm statistics (tf2/resnet.py:50-72): per-column sum / sum of squares of the
    // *stored* (rounded) outputs, accumulated in registers over all tiles of this CTA (the host
    // makes gridDim a multiple of tiles_n so a CTA keeps one column block) and flushed once.
    // Thread t owns 16-byte chunk (t & 7) -- CPC consecutive columns -- of rows (t >> 3)*8 .. +7 of
    // every staged tile: 8 conflict-free LDS.128 per box, partial sums kept in registers.
    const int sj = threadIdx.x & 7, srg = threadIdx.x >> 3;
    float st_sum[BOXES][CPC], st_sq[BOXES][CPC];
#pragma unroll
    for (int b = 0; b < BOXES; ++b)
#pragma unroll
      for (int c = 0; c < CPC; ++c) { st_sum[b][c] = 0.f; st_sq[b][c] = 0.f; }
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(out) & 15) == 0) && ((g.ldc * (int)sizeof(To)) % 16 == 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int tm = tile / g.tiles_n, tn = tile - tm * g.tiles_n;
      int prev = 0;
      for (int kb = 0; kb < g.num_kb; ++kb) {
        mbar_wait(&ctl.full[pp.stage], pp.phase);
        const uint32_t a_lo = smem_lo + (uint32_t)pp.stage * (TL::STAGE_BYTES >> 4);
        const uint32_t b_lo = a_lo + (A_STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)          // 4 x (32 bytes of K) per stage
#pragma unroll
          for (int h = 0; h < 2; ++h)        // rows 64h .. 64h + 63: 64 rows x 128 B further
            wgmma<BN, TF32, false, false>(acc[h], desc_pack(a_lo + h * (64 * 128 >> 4) + 2 * k, HI), desc_pack(b_lo + 2 * k, HI),
                                          (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (kb > 0) { wgmma_wait<1>(); warp_arrive(&ctl.empty[prev]); }
        prev = pp.stage;
        advance<STAGES>(pp);
      }
      wgmma_wait<0>(acc);
      warp_arrive(&ctl.empty[prev]);

      if (TMA_EPI) {
        // registers -> 128B-swizzled smem tile [128 rows][128 B] -> TMA store (coalesced, rows >= M and
        // columns >= n_out clipped by the tensor map).  Two staging tiles alternate.
#pragma unroll
        for (int b = 0; b < BOXES; ++b) {
          uint8_t* stage = ctl.epi + (box_ctr & 1) * A_STAGE_BYTES;
          const int n0 = tn * BN + b * BOX_COLS;
          if (n0 >= g.n_out) continue;                     // uniform across the CTA
          if (threadIdx.x == 0) {
            tma_store_wait_read<1>();   // the store issued two boxes ago has read its tile
            if (STATS_WARPS) mbar_wait(&ctl.sfree[box_ctr & 1], ((box_ctr >> 1) & 1) ^ 1);   // ... and so have the stats warps
          }
          named_barrier_sync(1, EPI_THREADS);
          stage_frag<To>(smem_u32(stage), acc, b * BOX_COLS / 8, all_rows);
          fence_proxy_async();
          named_barrier_sync(1, EPI_THREADS);
          if (threadIdx.x == 0) {
            if (sizeof(To) == 4 && g.accum) tma_reduce_add_2d(&tmap_out, stage, n0, tm * 128);
            else tma_store_2d(&tmap_out, stage, n0, tm * 128);
            tma_store_commit();
            if (STATS_WARPS) mbar_arrive(&ctl.sfull[box_ctr & 1]);
          }
          if (STATS && !STATS_WARPS) {
            float a0[CPC], a1[CPC];
#pragma unroll
            for (int c = 0; c < CPC; ++c) { a0[c] = 0.f; a1[c] = 0.f; }
#pragma unroll
            for (int i = 0; i < 8; ++i) {                 // rows srg*8 + i (rows >= M hold exact zeros)
              const uint4 raw = *reinterpret_cast<const uint4*>(stage + (srg * 8 + i) * 128 + ((sj ^ i) << 4));
              float v[CPC];
              if (sizeof(To) == 2) {
                const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) { v[(2 * e) % CPC] = __uint_as_float(w[e] << 16); v[(2 * e + 1) % CPC] = __uint_as_float(w[e] & 0xffff0000u); }
              } else {
                v[0] = __uint_as_float(raw.x); v[1] = __uint_as_float(raw.y); v[2 % CPC] = __uint_as_float(raw.z); v[3 % CPC] = __uint_as_float(raw.w);
              }
#pragma unroll
              for (int c = 0; c < CPC; ++c) { a0[c] += v[c]; a1[c] = fmaf(v[c], v[c], a1[c]); }
            }
#pragma unroll
            for (int c = 0; c < CPC; ++c) { st_sum[b][c] += a0[c]; st_sq[b][c] += a1[c]; }
          }
          ++box_ctr;
        }
      } else {
        // 32-column slices through one smem tile: thread t then holds row t of the slice
        const long long m = (long long)tm * 128 + threadIdx.x;
        long long row_off = m * g.ldc;
        if (g.os && m < g.M) {       // scattered rows (strided-dgrad parity class)
          uint32_t n, rem, p, q;
          g.dPQ.divmod((uint32_t)m, n, rem);
          g.dQ.divmod(rem, p, q);
          row_off = (((long long)n * g.OH + p * g.os + g.oh0) * g.OW + q * g.os + g.ow0) * g.ldc;
        }
#pragma unroll
        for (int c = 0; c < BN / 32; ++c) {
          const int n0 = tn * BN + c * 32;
          const int valid = g.n_out - n0;
          if (valid <= 0) continue;                        // uniform across the CTA
          named_barrier_sync(1, EPI_THREADS);              // the previous slice has been read
          stage_frag<float>(smem_u32(ctl.epi), acc, c * 4, all_rows);
          named_barrier_sync(1, EPI_THREADS);
          uint32_t r32[32];
          load_row32(ctl.epi, threadIdx.x, r32);
          if (m < g.M) {
            if (sizeof(To) == 4 && g.accum) {
              float* o = reinterpret_cast<float*>(out) + row_off + n0;
#pragma unroll
              for (int i = 0; i < 32; ++i) if (i < valid) atomicAdd(o + i, __uint_as_float(r32[i]));
            } else {
              store_row32<To>(out + row_off + n0, r32, valid, vec_ok);
            }
          }
        }
      }
    }
    if (TMA_EPI && STATS && !STATS_WARPS) {
      const int tn0 = blockIdx.x % g.tiles_n;            // constant for this CTA (gridDim % tiles_n == 0)
#pragma unroll
      for (int b = 0; b < BOXES; ++b) {
#pragma unroll
        for (int c = 0; c < CPC; ++c) {
          // fold the 4 row groups of the warp (lane >> 3) onto lanes 0-7
          float s0 = st_sum[b][c], s1 = st_sq[b][c];
          s0 += __shfl_xor_sync(0xffffffffu, s0, 8);  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
          s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
          const int col = tn0 * BN + b * BOX_COLS + sj * CPC + c;
          if (lane < 8 && col < g.n_out && (int)blockIdx.x < num_tiles) {     // partial of (CTA, warp): summed in order
            double* part = bn_sums + ((size_t)blockIdx.x * 4 + warp) * 2 * g.n_out;
            part[col] = (double)s0;
            part[g.n_out + col] = (double)s1;
          }
        }
      }
    }
    if (TMA_EPI && threadIdx.x == 0) tma_store_wait_all<0>();
  } else if (warp == 4) {
    // ------------------------------ TMA producer --------------------------
    if (lane == 0) {
      Pipe pp{0, 0};
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tm = tile / g.tiles_n, tn = tile - tm * g.tiles_n;
        // im2col feed: base pixel of the tile's first row; taps advance in K order, cblocks channel blocks each
        int im_n = 0, im_w = 0, im_h = 0, tap = 0, cb = 0, tr = 0, ts = 0;
        if (A_TMA && g.im2col) {
          uint32_t n, rem, p, q;
          g.dPQ.divmod((uint32_t)(tm * 128), n, rem);
          g.dQ.divmod(rem, p, q);
          im_n = (int)n; im_w = (int)q * g.stride + g.im_base; im_h = (int)p * g.stride + g.im_base;
        }
        for (int kb = 0; kb < g.num_kb; ++kb) {
          mbar_wait(&ctl.empty[pp.stage], pp.phase ^ 1);
          uint8_t* a_dst = smem + (size_t)pp.stage * TL::STAGE_BYTES;
          mbar_arrive_expect_tx(&ctl.full[pp.stage], TL::B_STAGE_BYTES + (A_TMA ? A_STAGE_BYTES : 0));
          if (A_TMA) {
            if (g.im2col) {
              int ow, oh;
              if (g.use_tab) { ow = g.tab_s[tap] - g.im_base; oh = g.tab_r[tap] - g.im_base; }
              else if (g.tap_sign > 0) { ow = ts; oh = tr; }
              else { ow = g.S - 1 - ts; oh = g.R - 1 - tr; }
              tma_load_im2col(a_dst, &tmap_a, &ctl.full[pp.stage], cb * KBE, im_w, im_h, im_n, ow, oh);
              if (++cb == g.cblocks) { cb = 0; ++tap; if (++ts == g.S) { ts = 0; ++tr; } }
            } else {
              tma_load_2d(a_dst, &tmap_a, &ctl.full[pp.stage], kb * KBE, tm * 128);
            }
          }
          int kcol = kb * KBE;
          if (g.use_tab) { const int t = kb / g.cblocks; kcol = g.tab_kcol[t] + (kb - t * g.cblocks) * KBE; }
          tma_load_2d(a_dst + A_STAGE_BYTES, &tmap_b, &ctl.full[pp.stage], kcol, tn * BN);
          advance<STAGES>(pp);
        }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------ statistics warps (TMA-fed kernels) -----
    if (STATS_WARPS) {
      const int st_t = threadIdx.x - AUX_T0;
      const int sj = st_t & 7, srg = st_t >> 3;
      // packed fp32 pairs: (sum, sum) and (sumsq, sumsq) of two adjacent columns per register pair
      constexpr int CP2 = CPC / 2;
      uint64_t st_sum[BOXES][CP2], st_sq[BOXES][CP2];
#pragma unroll
      for (int b = 0; b < BOXES; ++b)
#pragma unroll
        for (int c = 0; c < CP2; ++c) { st_sum[b][c] = 0ull; st_sq[b][c] = 0ull; }
      uint32_t ctr = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tn = tile % g.tiles_n;
#pragma unroll
        for (int b = 0; b < BOXES; ++b) {
          if (tn * BN + b * BOX_COLS >= g.n_out) continue;
          const uint8_t* stage = ctl.epi + (ctr & 1) * A_STAGE_BYTES;
          mbar_wait(&ctl.sfull[ctr & 1], (ctr >> 1) & 1);
#pragma unroll
          for (int i = 0; i < 8; ++i) {                     // rows srg*8 + i (rows >= M hold exact zeros)
            const uint4 raw = *reinterpret_cast<const uint4*>(stage + (srg * 8 + i) * 128 + ((sj ^ i) << 4));
            if (sizeof(To) == 2) {
              const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint64_t v = f2_pack(__uint_as_float(w[e] << 16), __uint_as_float(w[e] & 0xffff0000u));
                st_sum[b][e % CP2] = f2_add(st_sum[b][e % CP2], v);
                st_sq[b][e % CP2] = f2_fma(v, v, st_sq[b][e % CP2]);
              }
            } else {
              const uint64_t v0 = f2_pack(__uint_as_float(raw.x), __uint_as_float(raw.y));
              const uint64_t v1 = f2_pack(__uint_as_float(raw.z), __uint_as_float(raw.w));
              st_sum[b][0] = f2_add(st_sum[b][0], v0); st_sq[b][0] = f2_fma(v0, v0, st_sq[b][0]);
              st_sum[b][1 % CP2] = f2_add(st_sum[b][1 % CP2], v1); st_sq[b][1 % CP2] = f2_fma(v1, v1, st_sq[b][1 % CP2]);
            }
          }
          warp_arrive(&ctl.sfree[ctr & 1]);
          ++ctr;
        }
      }
      // Flush: fold the row groups of a warp by shuffles, the four warps through shared memory (the
      // operand ring is idle by now: every MMA of this CTA has retired before its last box was staged), then ONE fp64 partial
      // per column per CTA into the CTA's slot of the partials, which the host adds in CTA order.
      const int tn0 = blockIdx.x % g.tiles_n;
      float* red = reinterpret_cast<float*>(smem);          // [4 warps][BN columns][2]
      const int sw = st_t >> 5;
#pragma unroll
      for (int b = 0; b < BOXES; ++b) {
#pragma unroll
        for (int c = 0; c < CPC; ++c) {
          float lo0, hi0, lo1, hi1;
          f2_unpack(st_sum[b][c / 2], lo0, hi0); f2_unpack(st_sq[b][c / 2], lo1, hi1);
          float s0 = (c & 1) ? hi0 : lo0, s1 = (c & 1) ? hi1 : lo1;
          s0 += __shfl_xor_sync(0xffffffffu, s0, 8);  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
          s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
          const int lc = b * BOX_COLS + sj * CPC + c;
          if (lane < 8) { red[(sw * BN + lc) * 2] = s0; red[(sw * BN + lc) * 2 + 1] = s1; }
        }
      }
      named_barrier_sync(2, STATS_THREADS);
      for (int lc = st_t; lc < BN; lc += STATS_THREADS) {
        const int col = tn0 * BN + lc;
        if (col < g.n_out && (int)blockIdx.x < num_tiles) {
          double s0 = 0.0, s1 = 0.0;
#pragma unroll
          for (int w = 0; w < 4; ++w) { s0 += (double)red[(w * BN + lc) * 2]; s1 += (double)red[(w * BN + lc) * 2 + 1]; }
          double* part = bn_sums + (size_t)blockIdx.x * 4 * 2 * g.n_out;
          part[col] = s0;
          part[g.n_out + col] = s1;
        }
      }
    }
    // ------------------------------ gather producers ----------------------
    // cp.async keeps GATHER_DEPTH K blocks of loads in flight per thread; a stage is handed to the
    // MMA warp (fence.proxy.async + mbarrier arrive) once its group has landed.
    if (!A_TMA) {
      constexpr int D = TL::GATHER_DEPTH;
      const int gt = threadIdx.x - AUX_T0;
      const int j = gt & 7;              // 16-byte chunk within the 128-byte K block
      const int row0 = gt >> 3;          // rows row0 + GROWS*i
      Pipe pi{0, 0}, pa{0, 0};
      int inflight = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tm = tile / g.tiles_n;
        int rpix[GPT], rbh[GPT], rbw[GPT];     // rpix: n*H*W of the gathered tensor (-1: row beyond M)
#pragma unroll
        for (int i = 0; i < GPT; ++i) {
          const long long m = (long long)tm * 128 + row0 + GROWS * i;
          if (m < g.M) {
            uint32_t n, rem, p, q;
            g.dPQ.divmod((uint32_t)m, n, rem);
            g.dQ.divmod(rem, p, q);
            rpix[i] = (int)n * g.H * g.W;
            rbh[i] = g.mode == 0 ? (int)p * g.stride - g.pad_h : (int)p + g.pad_h;
            rbw[i] = g.mode == 0 ? (int)q * g.stride_w - g.pad_w : (int)q + g.pad_w;
          } else { rpix[i] = -1; rbh[i] = 0; rbw[i] = 0; }
        }
        const T* src = reinterpret_cast<const T*>(g.src);
        for (int kb = 0; kb < g.num_kb; ++kb) {
          const uint32_t k0 = (uint32_t)(kb * KBE + j * CH);
          mbar_wait(&ctl.empty[pi.stage], pi.phase ^ 1);
          const uint32_t a_addr = smem_u32(smem + (size_t)pi.stage * TL::STAGE_BYTES);
          if (!SMALLC) {
            uint32_t tap, c; g.dC.divmod(k0, tap, c);
            const TapRef t = decode_tap(g, tap);
#pragma unroll
            for (int i = 0; i < GPT; ++i) {
              const int h = rbh[i] + t.dr, w = rbw[i] + t.ds;
              const bool ok = t.ok && rpix[i] >= 0 && (unsigned)h < (unsigned)g.H && (unsigned)w < (unsigned)g.W;
              const T* p = src + (long long)(rpix[i] + h * g.W + w) * g.C + c;
              cp_async16(a_addr + sw128_offset(row0 + GROWS * i, j), ok ? (const void*)p : (const void*)src, ok ? 16u : 0u);
            }
          } else {
            // stem: 4 stored channels, so a 16-byte chunk covers two taps (8 bytes each)
            const TapRef t0 = decode_tap(g, k0 >> 2), t1 = decode_tap(g, (k0 >> 2) + 1);
#pragma unroll
            for (int i = 0; i < GPT; ++i) {
              const uint32_t dst = a_addr + sw128_offset(row0 + GROWS * i, j);
              const int h0 = rbh[i] + t0.dr, w0 = rbw[i] + t0.ds, h1 = rbh[i] + t1.dr, w1 = rbw[i] + t1.ds;
              const bool ok0 = t0.ok && rpix[i] >= 0 && (unsigned)h0 < (unsigned)g.H && (unsigned)w0 < (unsigned)g.W;
              const bool ok1 = t1.ok && rpix[i] >= 0 && (unsigned)h1 < (unsigned)g.H && (unsigned)w1 < (unsigned)g.W;
              const T* p0 = src + (long long)(rpix[i] + h0 * g.W + w0) * 4;
              const T* p1 = src + (long long)(rpix[i] + h1 * g.W + w1) * 4;
              cp_async8(dst, ok0 ? (const void*)p0 : (const void*)src, ok0 ? 8u : 0u);
              cp_async8(dst + 8, ok1 ? (const void*)p1 : (const void*)src, ok1 ? 8u : 0u);
            }
          }
          cp_async_commit();
          advance<STAGES>(pi);
          if (++inflight == D) {
            cp_async_wait<D - 1>();
            fence_proxy_async();
            warp_arrive(&ctl.full[pa.stage]);
            advance<STAGES>(pa);
            --inflight;
          }
        }
      }
      cp_async_wait<0>();
      fence_proxy_async();
      for (; inflight > 0; --inflight) { warp_arrive(&ctl.full[pa.stage]); advance<STAGES>(pa); }
    }
  }

  __syncthreads();
}

// ===========================================================================
// wgrad:  dW[(r,s,c)][co] = sum_pixels X[pixel@(r,s)][c] * dY[pixel][co]
// A^T (activations) and B (dY) are both MN-major: the reduction runs over pixels.
// Work item = (128 k-rows) x (BN couts) x (pixel split).  With one split every dW element is written once; with
// several, each split writes its partial to scratch and run_sum_partials adds them in split order (deterministic).
// ===========================================================================
template <typename T, int BN, bool SMALLC, bool A_TMA, bool TMA_RED>
__global__ void __launch_bounds__(wgrad_threads(A_TMA), 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy,
             const __grid_constant__ CUtensorMap tmap_dw, const Geom g, float* __restrict__ dw) {
  using TL = WTile<BN>;
  constexpr int STAGES = TL::STAGES;
  static_assert(!Elt<T>::TF32, "MN-major fp32 operands: not supported by wgmma");
  constexpr int ATOM_E = Elt<T>::KBE;            // elements along MN per 128-byte atom row
  constexpr int CH = Elt<T>::CH;
  constexpr int A_ATOMS = 128 / ATOM_E;          // 2
  constexpr int PXS = A_STAGE_BYTES / (A_ATOMS * 128);   // pixels per stage: 64
  constexpr int MMA_K = 32 / (int)sizeof(T);    // 16 pixels per MMA
  constexpr int ATOM_BYTES = PXS * 128;
  constexpr int B_ATOMS = BN / ATOM_E;
  constexpr int NF = BN / 2;
  static_assert(PXS / MMA_K == 4, "4 MMAs per stage");
  static_assert(A_ATOMS == 2, "one 64-row atom per m64 half");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const SmemCtl ctl = carve<STAGES>(smem, TL::STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&ctl.full[s], A_TMA ? 1 : 1 + GATHER_THREADS / 32); mbar_init(&ctl.empty[s], EPI_THREADS / 32); }
    fence_barrier_init();
  }
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmap_dy);
    if (A_TMA) tma_prefetch_desc(&tmap_x);
    if (TMA_RED) tma_prefetch_desc(&tmap_dw);
  }
  __syncthreads();
  const int num_items = g.tiles_m * g.tiles_n * g.splits;   // tiles_m = k-row tiles

  // item -> (tk, tn, split); splits of one tile are adjacent so their dY reads share L2
  auto decode = [&](int item, int& tk, int& tn, int& kb0, int& kb1) {
    const int split = item % g.splits;
    const int t = item / g.splits;
    tk = t / g.tiles_n; tn = t - tk * g.tiles_n;
    kb0 = split * g.kb_per_split;
    kb1 = min(g.num_kb, kb0 + g.kb_per_split);
  };

  if (warp < 4) {
    // ------------------------------ consumer: MMA + epilogue ------------------------------
    // MN-major operands: LBO = distance between 128-byte-wide atoms along M/N, SBO = 8 pixel rows; the m64 half h
    // of the A tile is atom h
    constexpr uint32_t HI = desc_hi_sw128(1024);
    const uint32_t smem_lo = uniform_u32(desc_lo(smem_u32(smem), ATOM_BYTES));
    const bool all_rows[2][2] = {{true, true}, {true, true}};
    float acc[2][NF];
    Pipe pp{0, 0};
    uint32_t box_ctr = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int tk, tn, kb0, kb1; decode(item, tk, tn, kb0, kb1);
      if (kb0 >= kb1) continue;
      const int split = item % g.splits;
      int prev = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&ctl.full[pp.stage], pp.phase);
        const uint32_t a_lo = smem_lo + (uint32_t)pp.stage * (TL::STAGE_BYTES >> 4);
        const uint32_t b_lo = a_lo + (TL::A_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            wgmma<BN, false, true, true>(acc[h], desc_pack(a_lo + h * (ATOM_BYTES >> 4) + k * (MMA_K * 128 >> 4), HI),
                                         desc_pack(b_lo + k * (MMA_K * 128 >> 4), HI), (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        if (kb > kb0) { wgmma_wait<1>(); warp_arrive(&ctl.empty[prev]); }
        prev = pp.stage;
        advance<STAGES>(pp);
      }
      wgmma_wait<0>(acc);
      warp_arrive(&ctl.empty[prev]);
      if (TMA_RED) {
        // partial tile -> swizzled smem [128 k-rows][32 fp32] -> TMA reduce-add into dW, or TMA store into this
        // split's rows of the scratch partials
#pragma unroll
        for (int cc = 0; cc < BN / 32; ++cc) {
          uint8_t* stage = ctl.epi + (box_ctr & 1) * A_STAGE_BYTES;
          const int n0 = tn * BN + cc * 32;
          if (n0 >= g.Cout) continue;                      // uniform across the CTA
          if (threadIdx.x == 0) tma_store_wait_read<1>();
          named_barrier_sync(1, EPI_THREADS);
          stage_frag<float>(smem_u32(stage), acc, cc * 4, all_rows);
          fence_proxy_async();
          named_barrier_sync(1, EPI_THREADS);
          if (threadIdx.x == 0) {
            if (g.ws) tma_store_2d(&tmap_dw, stage, n0, split * g.tiles_m * 128 + tk * 128);
            else tma_reduce_add_2d(&tmap_dw, stage, n0, tk * 128);
            tma_store_commit();
          }
          ++box_ctr;
        }
      } else {
        const int k = tk * 128 + threadIdx.x;              // row of the [R*S*Cs][Cout] matrix
        uint32_t tap, c; bool row_ok;
        if (g.s2) {          // stem K order: (r, s' in [0, S], c in [0, 4)); s' = 0 is the zero slot
          const int t4 = k >> 2, r = t4 / g.s2, sp = t4 - r * g.s2;
          c = (uint32_t)(k & 3);
          row_ok = r < g.R && sp >= 1 && (int)c < g.Cin;
          tap = (uint32_t)(r * (g.s2 - 1) + sp - 1);
        } else {
          g.dC.divmod((uint32_t)k, tap, c);
          row_ok = (int)tap < g.RS && (int)c < g.Cin;
        }
        // dW layout either way; several splits write their own copy of it
        float* drow = (g.ws ? g.ws + split * g.ws_stride : dw) + ((long long)tap * g.Cin + c) * g.Cout;
#pragma unroll
        for (int cc = 0; cc < BN / 32; ++cc) {
          named_barrier_sync(1, EPI_THREADS);              // the previous slice has been read
          stage_frag<float>(smem_u32(ctl.epi), acc, cc * 4, all_rows);
          named_barrier_sync(1, EPI_THREADS);
          uint32_t r32[32];
          load_row32(ctl.epi, threadIdx.x, r32);
          const int n0 = tn * BN + cc * 32;
          if (row_ok) {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              if (n0 + i >= g.Cout) continue;
              if (g.ws) drow[n0 + i] = __uint_as_float(r32[i]);
              else atomicAdd(drow + n0 + i, __uint_as_float(r32[i]));     // the only write to this element
            }
          }
        }
      }
    }
    if (TMA_RED && threadIdx.x == 0) tma_store_wait_all<0>();
  } else if (warp == 4) {
    if (lane == 0) {
      Pipe pp{0, 0};
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        int tk, tn, kb0, kb1; decode(item, tk, tn, kb0, kb1);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&ctl.empty[pp.stage], pp.phase ^ 1);
          uint8_t* a_dst = smem + (size_t)pp.stage * TL::STAGE_BYTES;
          uint8_t* b_dst = a_dst + TL::A_BYTES;
          mbar_arrive_expect_tx(&ctl.full[pp.stage], TL::B_STAGE_BYTES + (A_TMA ? TL::A_BYTES : 0));
          if (A_TMA) {
            if (g.im2col) {  // one im2col column of PXS pixels per atom: the atom's tap is the filter offset
              uint32_t n, rem, p, q;
              g.dPQ.divmod((uint32_t)(kb * PXS), n, rem);
              g.dQ.divmod(rem, p, q);
#pragma unroll
              for (int a = 0; a < A_ATOMS; ++a) {
                uint32_t tap, c, r, s2;
                g.dC.divmod((uint32_t)(tk * 128 + a * ATOM_E), tap, c);
                g.dS.divmod(tap, r, s2);
                const bool live = (int)tap < g.RS;     // k-rows past R*S*C: read a non-existent image (zeros)
                tma_load_im2col(a_dst + a * ATOM_BYTES, &tmap_x, &ctl.full[pp.stage], (int)c,
                                (int)q * g.stride + g.im_base, (int)p * g.stride + g.im_base,
                                live ? (int)n : g.im_nimg, live ? (int)s2 : 0, live ? (int)r : 0);
              }
            } else {         // 1x1 stride-1: the activation tile is a plain [pixels][channels] box
#pragma unroll
              for (int a = 0; a < A_ATOMS; ++a)
                tma_load_2d(a_dst + a * ATOM_BYTES, &tmap_x, &ctl.full[pp.stage], tk * 128 + a * ATOM_E, kb * PXS);
            }
          }
#pragma unroll
          for (int a = 0; a < B_ATOMS; ++a)
            tma_load_2d(b_dst + a * ATOM_BYTES, &tmap_dy, &ctl.full[pp.stage], tn * BN + a * ATOM_E, kb * PXS);
          advance<STAGES>(pp);
        }
      }
    }
    __syncwarp();
  } else if (!A_TMA) {
    constexpr int D = TL::GATHER_DEPTH;
    const int gt = threadIdx.x - AUX_T0;
    const int j = gt & 7;
    Pipe pi{0, 0}, pa{0, 0};
    int inflight = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int tk, tn, kb0, kb1; decode(item, tk, tn, kb0, kb1);
      // piece i of this thread: q = gt/8 + GROWS*i -> atom q / PXS, pixel q % PXS; its (tap, c) is fixed per item
      int pdr[GPT], pds[GPT], pc[GPT]; bool pk[GPT];
      int pdr2[GPT], pds2[GPT]; bool pk2[GPT];
#pragma unroll
      for (int i = 0; i < GPT; ++i) {
        const int q = (gt >> 3) + GROWS * i;
        const int atom = q / PXS;
        const uint32_t k = (uint32_t)(tk * 128 + atom * ATOM_E + j * CH);
        if (!SMALLC) {
          uint32_t tap, c; g.dC.divmod(k, tap, c);
          const TapRef t = decode_tap(g, tap);
          pk[i] = t.ok; pdr[i] = t.dr; pds[i] = t.ds; pc[i] = (int)c;
          pk2[i] = false; pdr2[i] = pds2[i] = 0;
        } else {
          const TapRef t0 = decode_tap(g, k >> 2), t1 = decode_tap(g, (k >> 2) + 1);
          pk[i] = t0.ok; pdr[i] = t0.dr; pds[i] = t0.ds; pc[i] = 0;
          pk2[i] = t1.ok; pdr2[i] = t1.dr; pds2[i] = t1.ds;
        }
      }
      const T* src = reinterpret_cast<const T*>(g.src);
      // The thread's GPT pieces touch only NPX distinct pixels (piece i -> pixel slot i % NPX, atom i / NPX).
      // Their (n, p, q) coordinates are decoded once per item and then walked forward by PXS per K block.
      constexpr int NPX = PXS / GROWS;
      static_assert(NPX >= 1, "gather rows per pass must not exceed the pixels per stage");
      int sn[NPX], sp[NPX], sq[NPX];
      long long sm[NPX];
#pragma unroll
      for (int e = 0; e < NPX; ++e) {
        sm[e] = (long long)kb0 * PXS + (gt >> 3) + GROWS * e;
        uint32_t nn, rem, p, qq;
        g.dPQ.divmod((uint32_t)min(sm[e], (long long)0x7fffffff), nn, rem);
        g.dQ.divmod(rem, p, qq);
        sn[e] = (int)nn; sp[e] = (int)p; sq[e] = (int)qq;
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&ctl.empty[pi.stage], pi.phase ^ 1);
        const uint32_t a_addr = smem_u32(smem + (size_t)pi.stage * TL::STAGE_BYTES);
#pragma unroll
        for (int i = 0; i < GPT; ++i) {
          const int e = i % NPX;
          const int q = (gt >> 3) + GROWS * i;
          const int px = q % PXS;
          const uint32_t dst = a_addr + (q / PXS) * ATOM_BYTES + sw128_offset(px, j);
          const bool in_m = sm[e] < g.M;
          const int pix = sn[e] * g.H * g.W;
          const int bh = sp[e] * g.stride - g.pad_h, bw = sq[e] * g.stride_w - g.pad_w;
          if (!SMALLC) {
            const int h = bh + pdr[i], w = bw + pds[i];
            const bool ok = pk[i] && in_m && (unsigned)h < (unsigned)g.H && (unsigned)w < (unsigned)g.W;
            const T* p = src + (long long)(pix + h * g.W + w) * g.C + pc[i];
            cp_async16(dst, ok ? (const void*)p : (const void*)src, ok ? 16u : 0u);
          } else {
            const int h0 = bh + pdr[i], w0 = bw + pds[i], h1 = bh + pdr2[i], w1 = bw + pds2[i];
            const bool ok0 = pk[i] && in_m && (unsigned)h0 < (unsigned)g.H && (unsigned)w0 < (unsigned)g.W;
            const bool ok1 = pk2[i] && in_m && (unsigned)h1 < (unsigned)g.H && (unsigned)w1 < (unsigned)g.W;
            const T* p0 = src + (long long)(pix + h0 * g.W + w0) * 4;
            const T* p1 = src + (long long)(pix + h1 * g.W + w1) * 4;
            cp_async8(dst, ok0 ? (const void*)p0 : (const void*)src, ok0 ? 8u : 0u);
            cp_async8(dst + 8, ok1 ? (const void*)p1 : (const void*)src, ok1 ? 8u : 0u);
          }
        }
#pragma unroll
        for (int e = 0; e < NPX; ++e) {      // advance the pixel walk by PXS
          sm[e] += PXS;
          sq[e] += g.adv_q; sp[e] += g.adv_p;
          if (sq[e] >= g.Q) { sq[e] -= g.Q; ++sp[e]; }
          while (sp[e] >= g.P) { sp[e] -= g.P; ++sn[e]; }
        }
        cp_async_commit();
        advance<STAGES>(pi);
        if (++inflight == D) {
          cp_async_wait<D - 1>();
          fence_proxy_async();
          warp_arrive(&ctl.full[pa.stage]);
          advance<STAGES>(pa);
          --inflight;
        }
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (; inflight > 0; --inflight) { warp_arrive(&ctl.full[pa.stage]); advance<STAGES>(pa); }
  }

  __syncthreads();
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
inline int pick_bn(int64_t n) { return n > 64 ? 128 : 64; }

template <typename K> int set_smem_attr(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e)); return (int)e; }
  return SIMCLR_OK;
}

// CTAs of an igemm launch.  With fused statistics each CTA keeps one column block (tile = blockIdx.x + i*gridDim.x
// keeps tn fixed), so the grid is a multiple of tiles_n.
inline int igemm_grid(const Geom& g, bool stats) {
  int grid = g.tiles_m * g.tiles_n; if (grid > num_sms()) grid = num_sms();
  if (stats) {
    grid = grid / g.tiles_n * g.tiles_n;
    if (grid < g.tiles_n) grid = g.tiles_n;
  }
  return grid;
}

template <typename T, typename To, int BN, bool A_TMA, bool SMALLC, bool TMA_EPI, bool STATS>
int launch_igemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout, const Geom& g, double* bn_sums,
                 cudaStream_t st) {
  auto kern = igemm_kernel<T, To, BN, A_TMA, SMALLC, TMA_EPI, STATS>;
  { int rc = set_smem_attr(kern, Tile<BN>::SMEM_BYTES); if (rc) return rc; }   // a per-DEVICE attribute: set on every launch
  const int grid = igemm_grid(g, STATS);
  kern<<<grid, igemm_threads(A_TMA, STATS), Tile<BN>::SMEM_BYTES, st>>>(ta, tb, tout, g, bn_sums);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

template <typename T, typename To, int BN, bool TMA_EPI, bool STATS>
int dispatch_igemm3(bool a_tma, bool smallc, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                    const Geom& g, double* bn_sums, cudaStream_t st) {
  if (a_tma) return launch_igemm<T, To, BN, true, false, TMA_EPI, STATS>(ta, tb, tout, g, bn_sums, st);
  if (smallc) return launch_igemm<T, To, BN, false, true, TMA_EPI, STATS>(ta, tb, tout, g, bn_sums, st);
  return launch_igemm<T, To, BN, false, false, TMA_EPI, STATS>(ta, tb, tout, g, bn_sums, st);
}
template <typename T, typename To, int BN>
int dispatch_igemm2(bool a_tma, bool smallc, bool tma_epi, const CUtensorMap& ta, const CUtensorMap& tb,
                    const CUtensorMap& tout, const Geom& g, double* bn_sums, cudaStream_t st) {
  if (tma_epi && bn_sums) return dispatch_igemm3<T, To, BN, true, true>(a_tma, smallc, ta, tb, tout, g, bn_sums, st);
  if (tma_epi) return dispatch_igemm3<T, To, BN, true, false>(a_tma, smallc, ta, tb, tout, g, nullptr, st);
  return dispatch_igemm3<T, To, BN, false, false>(a_tma, smallc, ta, tb, tout, g, nullptr, st);
}
template <typename T, typename To>
int dispatch_igemm(int bn, bool a_tma, bool smallc, bool tma_epi, const CUtensorMap& ta, const CUtensorMap& tb,
                   const CUtensorMap& tout, const Geom& g, cudaStream_t st, double* bn_sums = nullptr) {
  if (bn == 128) return dispatch_igemm2<T, To, 128>(a_tma, smallc, tma_epi, ta, tb, tout, g, bn_sums, st);
  return dispatch_igemm2<T, To, 64>(a_tma, smallc, tma_epi, ta, tb, tout, g, bn_sums, st);
}

// TMA im2col applicability and bounding-box corners for a gathered tensor [N][Hs][Ws][Cs] whose
// GEMM rows are the P x Q pixel grid.  mode 0: source pixel = p*stride - pad + r (fprop, wgrad);
// mode 1: p + pad - r (stride-1 dgrad), expressed as base p + pad - (R-1) and offset R-1-r.
// Base pixels run lo .. (W-1)+up with the traversal stride: exactly Q (P) positions per row (image).
// SIMCLR_TC_IM2COL=0 forces the cp.async gather (A/B testing).
struct Im2colPlan { int lo, up; };
inline bool im2col_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("SIMCLR_TC_IM2COL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v == 1;
}
inline bool plan_im2col(int mode, int64_t Hs, int64_t Ws, int64_t Cs, int64_t P, int64_t Q, int64_t R, int64_t S,
                        int64_t stride, int kbe, Im2colPlan* pl) {
  if (!im2col_enabled() || R != S || Cs % kbe != 0 || stride > 8 || get_encode_im2col() == nullptr) return false;
  const int pad = (int)((R - 1) / 2);
  int lo, up_w, up_h;
  if (mode == 0) {
    lo = -pad;
    up_w = (int)(lo + stride * (Q - 1) - (Ws - 1));
    up_h = (int)(lo + stride * (P - 1) - (Hs - 1));
  } else {
    if (stride != 1 || P != Hs || Q != Ws) return false;
    lo = pad - (int)(R - 1);
    up_w = up_h = lo;
  }
  if (up_w != up_h || lo < -128 || lo > 127 || up_w < -128 || up_w > 127) return false;
  if (R - 1 > 255 || Hs >= 32768 || Ws >= 32768) return false;
  pl->lo = lo; pl->up = up_w;
  return true;
}

// Geometry of the stem's K order (see run_igemm).
struct StemGeom { bool pairs; int64_t S, W; int pad_w, stride_w; };
inline StemGeom stem_geom(bool smallc, int mode, int64_t W, int64_t S, int64_t stride) {
  StemGeom sg; sg.pairs = false; sg.S = S; sg.W = W; sg.pad_w = (int)((S - 1) / 2); sg.stride_w = (int)stride;
  if (!smallc) return sg;
  const int pad = (int)((S - 1) / 2);
  static int en = -1;
  if (en < 0) { const char* e = getenv("SIMCLR_TC_STEM_PAIRS"); en = (e && e[0] == '0') ? 0 : 1; }
  if (en && mode == 0 && stride == 2 && (pad & 1) && W % 2 == 0) {
    sg.pairs = true; sg.S = (S + 1) / 2; sg.W = W / 2; sg.pad_w = (pad + 1) / 2; sg.stride_w = 1;
  } else {
    sg.S = S + 1; sg.pad_w = pad + 1;
  }
  return sg;
}

// Shared driver for fprop (mode 0) and dgrad (mode 1).
//   gathered tensor [N][Hs][Ws][Cs]; GEMM rows = N*P*Q; weights wk [n_out][Kp]
int run_igemm(int mode, const void* src, const void* wk, void* out, int dtype, int out_dtype, int64_t N, int64_t Hs,
              int64_t Ws, int64_t Cs, int64_t P, int64_t Q, int64_t n_out, int64_t R, int64_t S, int64_t stride,
              cudaStream_t st, const char* what, double* bn_sums = nullptr, bool accum = false) {
  const int es = dtype == SIMCLR_BF16 ? 2 : 4;
  const int KBE = 128 / es, CH = 16 / es;
  if (accum && (out_dtype != SIMCLR_F32 || bn_sums)) { set_error("%s: accumulation needs fp32 outputs and no fused statistics", what); return SIMCLR_ERR_INVALID_ARG; }
  bool smallc = (dtype == SIMCLR_BF16 && Cs == 4);
  if (!(Cs % CH == 0 || smallc)) { set_error("%s: stored channels (%lld) must be a multiple of %d", what, (long long)Cs, CH); return SIMCLR_ERR_UNSUPPORTED; }
  if (smallc && mode != 0) { set_error("%s: 4-channel tensors are only supported as the conv input", what); return SIMCLR_ERR_UNSUPPORTED; }
  if (!aligned16(src) || !aligned16(wk)) { set_error("%s: operands must be 16-byte aligned", what); return SIMCLR_ERR_INVALID_ARG; }
  const int64_t M = N * P * Q;
  if (M >= (1ll << 31)) { set_error("%s: M too large", what); return SIMCLR_ERR_UNSUPPORTED; }
  // stem: slab of pixel pairs read through overlapping no-swizzle descriptors (tc_stem.cu)
  if (mode == 0 && smallc && !accum && stem7x7_applicable(dtype, out_dtype, N, Hs, Ws, Cs, n_out, R, S, stride, P, Q, src, wk, out))
    return run_stem7x7(src, wk, out, N, Hs, Ws, n_out, st, bn_sums);
  // 64 / 128-channel 3x3 stride-1 layers: halo-reuse kernel (one slab load instead of nine im2col loads)
  if (!accum && P == Hs && Q == Ws && halo3x3_applicable(dtype, out_dtype, N, Hs, Ws, Cs, n_out, R, S, stride, src, wk, out))
    return run_halo3x3(mode, src, wk, out, N, Hs, Ws, Cs, n_out, st, bn_sums);
  // Stem (4 stored channels, bf16): K runs over (r, s' in [0, S], c) with a zero slot s' = 0, i.e. the
  // filter is S+1 wide with one more pixel of left padding.  With stride 2, odd padding and an even
  // width the S+1 slots are whole 16-byte pixel pairs: the tensor is then read as [N][H][W/2][8] with
  // (S+1)/2 taps per row, unit column stride, and goes through the ordinary 16-byte gather.
  StemGeom sg = stem_geom(smallc, mode, Ws, S, stride);
  if (sg.pairs) { smallc = false; Cs = 8; Ws = sg.W; }
  const int64_t Sk = smallc || sg.pairs ? sg.S : S;
  const int64_t K = R * Sk * Cs;
  const int64_t Kp = (K + KBE - 1) / KBE * KBE;
  const int bn = pick_bn(n_out);
  Geom g;
  g.src = src; g.out = out; g.mode = mode;
  g.H = (int)Hs; g.W = (int)Ws; g.C = (int)Cs; g.R = (int)R; g.S = (int)Sk; g.RS = (int)(R * Sk);
  g.stride = (int)stride; g.pad_h = (int)((R - 1) / 2); g.pad_w = (int)((S - 1) / 2);
  g.stride_w = (int)stride; g.s2 = 0;
  if (smallc || sg.pairs) { g.pad_w = sg.pad_w; g.stride_w = sg.stride_w; g.s2 = (int)S + 1; }
  g.dPQ = FastDiv((uint32_t)(P * Q)); g.dQ = FastDiv((uint32_t)Q); g.dC = FastDiv((uint32_t)Cs); g.dS = FastDiv((uint32_t)Sk);
  g.P = (int)P; g.Q = (int)Q; g.adv_p = g.adv_q = 0;
  g.M = M; g.n_out = (int)n_out; g.ldc = (int)n_out; g.num_kb = (int)(Kp / KBE);
  g.tiles_m = (int)((M + 127) / 128); g.tiles_n = (int)((n_out + bn - 1) / bn);
  g.Cin = g.Cout = 0; g.splits = 1; g.kb_per_split = g.num_kb;
  g.use_tab = 0; g.cblocks = 1; g.os = 0; g.oh0 = g.ow0 = 0; g.OH = g.OW = 0;
  g.tap_sign = mode == 0 ? 1 : -1;
  g.im2col = 0; g.im_base = 0; g.im_nimg = (int)N; g.accum = accum ? 1 : 0;
  // plain GEMM (1x1, stride 1, no padding): activations go through TMA as well
  bool a_tma = (R == 1 && S == 1 && stride == 1 && !smallc && (Cs * es) % 16 == 0);
  CUtensorMap ta, tb, tout;
  int rc = make_tmap_2d(&tb, wk, es, (uint64_t)n_out, (uint64_t)Kp, (uint64_t)Kp * es, (uint32_t)bn, (uint32_t)KBE);
  if (rc) return rc;
  if (a_tma) { rc = make_tmap_2d(&ta, src, es, (uint64_t)M, (uint64_t)Cs, (uint64_t)Cs * es, 128, (uint32_t)KBE); if (rc) return rc; }
  else {
    ta = tb;
    // every other shape with whole 128-byte channel blocks: TMA im2col (square filter, symmetric padding)
    Im2colPlan pl;
    if (!smallc && plan_im2col(mode, Hs, Ws, Cs, P, Q, R, S, stride, KBE, &pl)) {
      rc = make_tmap_im2col(&ta, src, es, (uint64_t)N, (uint64_t)Hs, (uint64_t)Ws, (uint64_t)Cs, pl.lo, pl.up, (uint32_t)stride, 128);
      if (rc) return rc;
      g.im2col = 1; g.im_base = pl.lo; g.cblocks = (int)(Cs / KBE);
      a_tma = true;
    }
  }
  // coalesced TMA-store epilogue whenever the output rows are 16-byte aligned
  const int eo = out_dtype == SIMCLR_BF16 ? 2 : 4;
  const bool tma_epi = aligned16(out) && ((n_out * eo) % 16 == 0);
  if (tma_epi) { rc = make_tmap_2d(&tout, out, eo, (uint64_t)M, (uint64_t)n_out, (uint64_t)n_out * eo, 128, (uint32_t)(128 / eo)); if (rc) return rc; }
  else tout = tb;
  double* parts = nullptr;            // fused statistics: [CTAs][4 warps][2][n_out] partials, added in order
  const int nparts = 4 * igemm_grid(g, true);
  if (bn_sums) {
    if (!tma_epi) { set_error("%s: fused BN statistics need 16-byte aligned output rows", what); return SIMCLR_ERR_UNSUPPORTED; }
    if (!accumulate_prezeroed()) {
      cudaError_t e = cudaMemsetAsync(bn_sums, 0, 2 * (size_t)n_out * sizeof(double), st);
      if (e != cudaSuccess) { set_error("%s: memset: %s", what, cudaGetErrorString(e)); return (int)e; }
    }
    rc = scratch_alloc(&parts, (size_t)nparts * 2 * n_out * sizeof(double), st);
    if (rc) return rc;
    cudaError_t e = cudaMemsetAsync(parts, 0, (size_t)nparts * 2 * n_out * sizeof(double), st);
    if (e != cudaSuccess) { set_error("%s: memset: %s", what, cudaGetErrorString(e)); scratch_free(parts, st); return (int)e; }
    if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_BF16)
      rc = dispatch_igemm<__nv_bfloat16, __nv_bfloat16>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, parts);
    else if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_F32)
      rc = dispatch_igemm<__nv_bfloat16, float>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, parts);
    else if (dtype == SIMCLR_F32 && out_dtype == SIMCLR_F32)
      rc = dispatch_igemm<float, float>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, parts);
    else { set_error("%s: unsupported dtype combination %d -> %d", what, dtype, out_dtype); rc = SIMCLR_ERR_UNSUPPORTED; }
    if (!rc) rc = run_sum_partials_f64(parts, 2 * n_out, bn_sums, 2 * n_out, nparts, st);
    const int rf = scratch_free(parts, st);
    return rc ? rc : rf;
  }
  if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_BF16) return dispatch_igemm<__nv_bfloat16, __nv_bfloat16>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, bn_sums);
  if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_F32) return dispatch_igemm<__nv_bfloat16, float>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, bn_sums);
  if (dtype == SIMCLR_F32 && out_dtype == SIMCLR_F32) return dispatch_igemm<float, float>(bn, a_tma, smallc, tma_epi, ta, tb, tout, g, st, bn_sums);
  set_error("%s: unsupported dtype combination %d -> %d", what, dtype, out_dtype);
  return SIMCLR_ERR_UNSUPPORTED;
}

// dgrad of a strided conv, decomposed by output-pixel parity: the pixels of dX with
// (h mod s, w mod s) == (ph, pw) only receive the taps with (ph + pad - r) % s == 0, reading
// dY at h/s + (ph + pad - r)/s.  Each class is a dense stride-1 gather over the dY grid with its
// own tap list -- no multiplications by structural zeros (a stride-2 3x3 does 9/4 of the dense
// work instead of 9x).  Classes without taps (1x1 kernels) stay zero from the memset.
int run_dgrad_strided(const void* dy, const void* wd, void* dx, int dtype, int out_dtype, int64_t N, int64_t H,
                      int64_t W, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride, cudaStream_t st,
                      bool accum = false) {
  const int es = dtype == SIMCLR_BF16 ? 2 : 4;
  const int eo = out_dtype == SIMCLR_BF16 ? 2 : 4;
  if (accum && out_dtype != SIMCLR_F32) { set_error("conv2d_dgrad_tc: accumulation needs fp32 outputs"); return SIMCLR_ERR_INVALID_ARG; }
  const int KBE = 128 / es;
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int pad_h = (int)((R - 1) / 2), pad_w = (int)((S - 1) / 2);
  const int64_t Kdp = (R * S * Cout + KBE - 1) / KBE * KBE;
  const int bn = pick_bn(Cin);
  CUtensorMap tb;
  int rc = make_tmap_2d(&tb, wd, es, (uint64_t)Cin, (uint64_t)Kdp, (uint64_t)Kdp * es, (uint32_t)bn, (uint32_t)KBE);
  if (rc) return rc;
  bool need_zero = false;
  for (int ph = 0; ph < stride; ++ph) {
    int cnt = 0;
    for (int r = 0; r < R; ++r) if ((ph + pad_h - r) % (int)stride == 0) ++cnt;
    if (cnt == 0) need_zero = true;
  }
  for (int pw = 0; pw < stride; ++pw) {
    int cnt = 0;
    for (int s2 = 0; s2 < S; ++s2) if ((pw + pad_w - s2) % (int)stride == 0) ++cnt;
    if (cnt == 0) need_zero = true;
  }
  if (need_zero && !accum) SIMCLR_CHECK_CUDA(cudaMemsetAsync(dx, 0, (size_t)(N * H * W * Cin) * eo, st));
  for (int ph = 0; ph < stride; ++ph) {
    for (int pw = 0; pw < stride; ++pw) {
      Geom g;
      int nt = 0;
      for (int r = 0; r < R; ++r) {
        if ((ph + pad_h - r) % (int)stride != 0) continue;
        for (int s2 = 0; s2 < S; ++s2) {
          if ((pw + pad_w - s2) % (int)stride != 0) continue;
          if (nt >= 9) { set_error("conv2d_dgrad_tc: too many taps per parity class"); return SIMCLR_ERR_UNSUPPORTED; }
          // C division truncates toward zero; the numerator is an exact multiple of the stride
          g.tab_r[nt] = (ph + pad_h - r) / (int)stride;
          g.tab_s[nt] = (pw + pad_w - s2) / (int)stride;
          g.tab_kcol[nt] = (int)((r * S + s2) * Cout);
          ++nt;
        }
      }
      const int64_t P2 = (H - ph + stride - 1) / stride, Q2 = (W - pw + stride - 1) / stride;
      if (nt == 0 || P2 <= 0 || Q2 <= 0) continue;
      for (int t = nt; t < 9; ++t) { g.tab_r[t] = g.tab_s[t] = 0; g.tab_kcol[t] = 0; }
      const int64_t M = N * P2 * Q2;
      g.src = dy; g.out = dx; g.mode = 0;
      g.H = (int)Ho; g.W = (int)Wo; g.C = (int)Cout; g.R = 1; g.S = 1; g.RS = nt;
      g.stride = 1; g.stride_w = 1; g.s2 = 0; g.pad_h = 0; g.pad_w = 0;
      g.dPQ = FastDiv((uint32_t)(P2 * Q2)); g.dQ = FastDiv((uint32_t)Q2); g.dC = FastDiv((uint32_t)Cout); g.dS = FastDiv(1);
      g.P = (int)P2; g.Q = (int)Q2; g.adv_p = g.adv_q = 0;
      g.M = M; g.n_out = (int)Cin; g.ldc = (int)Cin;
      g.cblocks = (int)(Cout / KBE); g.num_kb = nt * g.cblocks;
      g.tiles_m = (int)((M + 127) / 128); g.tiles_n = (int)((Cin + bn - 1) / bn);
      g.Cin = g.Cout = 0; g.splits = 1; g.kb_per_split = g.num_kb;
      g.tap_sign = 1;
      g.use_tab = 1; g.os = (int)stride; g.oh0 = ph; g.ow0 = pw; g.OH = (int)H; g.OW = (int)W;
      // the class is a stride-1 walk over the dY grid: TMA im2col when its pixel grid is the dY grid
      g.im2col = 0; g.im_base = 0; g.im_nimg = (int)N; g.accum = accum ? 1 : 0;
      CUtensorMap ta = tb;
      bool a_tma = false;
      if (im2col_enabled() && get_encode_im2col() != nullptr && P2 == Ho && Q2 == Wo && Ho < 32768 && Wo < 32768) {
        int lo = g.tab_r[0];
        for (int t = 0; t < nt; ++t) { lo = g.tab_r[t] < lo ? g.tab_r[t] : lo; lo = g.tab_s[t] < lo ? g.tab_s[t] : lo; }
        int hi = lo;
        for (int t = 0; t < nt; ++t) { hi = g.tab_r[t] > hi ? g.tab_r[t] : hi; hi = g.tab_s[t] > hi ? g.tab_s[t] : hi; }
        if (lo >= -128 && hi - lo <= 255) {
          rc = make_tmap_im2col(&ta, dy, es, (uint64_t)N, (uint64_t)Ho, (uint64_t)Wo, (uint64_t)Cout, lo, lo, 1, 128);
          if (rc) return rc;
          g.im2col = 1; g.im_base = lo; a_tma = true;
        }
      }
      if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_BF16) rc = dispatch_igemm<__nv_bfloat16, __nv_bfloat16>(bn, a_tma, false, false, ta, tb, tb, g, st);
      else if (dtype == SIMCLR_BF16 && out_dtype == SIMCLR_F32) rc = dispatch_igemm<__nv_bfloat16, float>(bn, a_tma, false, false, ta, tb, tb, g, st);
      else if (dtype == SIMCLR_F32 && out_dtype == SIMCLR_F32) rc = dispatch_igemm<float, float>(bn, a_tma, false, false, ta, tb, tb, g, st);
      else { set_error("conv2d_dgrad_tc: unsupported dtype combination"); return SIMCLR_ERR_UNSUPPORTED; }
      if (rc) return rc;
    }
  }
  return SIMCLR_OK;
}

template <typename T, int BN, bool SMALLC, bool A_TMA, bool TMA_RED>
int launch_wgrad(const CUtensorMap& tx, const CUtensorMap& tdy, const CUtensorMap& tdw, const Geom& g, float* dw,
                 cudaStream_t st) {
  auto kern = wgrad_kernel<T, BN, SMALLC, A_TMA, TMA_RED>;
  int rc = set_smem_attr(kern, WTile<BN>::SMEM_BYTES); if (rc) return rc;      // per device: set every time
  int grid = g.tiles_m * g.tiles_n * g.splits; if (grid > num_sms()) grid = num_sms();
  kern<<<grid, wgrad_threads(A_TMA), WTile<BN>::SMEM_BYTES, st>>>(tx, tdy, tdw, g, dw);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}
template <typename T, int BN>
int dispatch_wgrad2(bool smallc, bool a_tma, bool tma_red, const CUtensorMap& tx, const CUtensorMap& tdy,
                    const CUtensorMap& tdw, const Geom& g, float* dw, cudaStream_t st) {
  if (smallc) return launch_wgrad<T, BN, true, false, false>(tx, tdy, tdw, g, dw, st);
  if (tma_red) {
    if (a_tma) return launch_wgrad<T, BN, false, true, true>(tx, tdy, tdw, g, dw, st);
    return launch_wgrad<T, BN, false, false, true>(tx, tdy, tdw, g, dw, st);
  }
  if (a_tma) return launch_wgrad<T, BN, false, true, false>(tx, tdy, tdw, g, dw, st);
  return launch_wgrad<T, BN, false, false, false>(tx, tdy, tdw, g, dw, st);
}
template <typename T>
int dispatch_wgrad(int bn, bool smallc, bool a_tma, bool tma_red, const CUtensorMap& tx, const CUtensorMap& tdy,
                   const CUtensorMap& tdw, const Geom& g, float* dw, cudaStream_t st) {
  if (bn == 128) return dispatch_wgrad2<T, 128>(smallc, a_tma, tma_red, tx, tdy, tdw, g, dw, st);
  return dispatch_wgrad2<T, 64>(smallc, a_tma, tma_red, tx, tdy, tdw, g, dw, st);
}

}  // namespace

}  // namespace tc

// A block takes 32 consecutive elements; lane ty of 16 adds parts ty, ty + 16, ... in order, then the 16 lane sums are
// added in lane order.  The order depends only on `parts`, so the result is the same on every run.
constexpr int SUM_LANES = 16;
template <typename T>
__global__ void __launch_bounds__(32 * SUM_LANES) sum_partials_kernel(const T* __restrict__ ws, long long stride, T* __restrict__ dst,
                                                                      long long n, int parts) {
  __shared__ T sh[SUM_LANES][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (long long i0 = blockIdx.x * 32ll; i0 < n; i0 += (long long)gridDim.x * 32) {
    const long long i = i0 + tx;
    T a = 0;
    if (i < n)
      for (int p = ty; p < parts; p += SUM_LANES) a += ws[p * stride + i];
    sh[ty][tx] = a;
    __syncthreads();
    if (ty == 0 && i < n) {
      T d = dst[i];
#pragma unroll
      for (int k = 0; k < SUM_LANES; ++k) d += sh[k][tx];
      dst[i] = d;
    }
    __syncthreads();
  }
}

template <typename T>
int sum_partials(const T* ws, int64_t stride, T* dst, int64_t n, int parts, cudaStream_t st) {
  int64_t blocks = (n + 31) / 32;
  if (blocks > 16 * (int64_t)num_sms()) blocks = 16 * (int64_t)num_sms();
  if (blocks < 1) blocks = 1;
  sum_partials_kernel<T><<<(int)blocks, 32 * SUM_LANES, 0, st>>>(ws, stride, dst, n, parts);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int run_sum_partials(const float* ws, int64_t stride, float* dst, int64_t n, int parts, cudaStream_t st) {
  return sum_partials(ws, stride, dst, n, parts, st);
}
int run_sum_partials_f64(const double* ws, int64_t stride, double* dst, int64_t n, int parts, cudaStream_t st) {
  return sum_partials(ws, stride, dst, n, parts, st);
}

}  // namespace simclr

using namespace simclr;

extern "C" {

int simclr_conv2d_fprop_tc(const void* x, const void* wf, void* y, int dtype, int y_dtype, int64_t N, int64_t H,
                           int64_t W, int64_t Cs, int64_t Cout, int64_t R, int64_t S, int64_t stride, double* bn_sums,
                           void* stream) {
  SIMCLR_CHECK_ARG(x && wf && y, "conv2d_fprop_tc: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cs > 0 && Cout > 0 && R > 0 && S > 0 && (R & 1) && (S & 1) && stride > 0,
                   "conv2d_fprop_tc: bad geometry");
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  return tc::run_igemm(0, x, wf, y, dtype, y_dtype, N, H, W, Cs, Ho, Wo, Cout, R, S, stride, (cudaStream_t)stream,
                       "conv2d_fprop_tc", bn_sums);
}

int simclr_conv2d_dgrad_tc(const void* dy, const void* wd, void* dx, int dtype, int dx_dtype, int64_t N, int64_t H,
                           int64_t W, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream) {
  SIMCLR_CHECK_ARG(dy && wd && dx, "conv2d_dgrad_tc: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && R > 0 && S > 0 && (R & 1) && (S & 1) && stride > 0,
                   "conv2d_dgrad_tc: bad geometry");
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  {
    const int es = dtype == SIMCLR_BF16 ? 2 : 4;
    if (stride > 1 && stride <= 3 && Cout % (128 / es) == 0 && simclr::aligned16(dy) && simclr::aligned16(wd) && simclr::aligned16(dx))
      return tc::run_dgrad_strided(dy, wd, dx, dtype, dx_dtype, N, H, W, Cin, Cout, R, S, stride, (cudaStream_t)stream);
    if (stride > 1) {
      simclr::set_error("conv2d_dgrad_tc: stride %lld needs Cout %% %d == 0, stride <= 3 and 16-byte aligned operands",
                        (long long)stride, 128 / es);
      return SIMCLR_ERR_UNSUPPORTED;
    }
  }
  // gathered tensor is dY [N][Ho][Wo][Cout]; GEMM rows are the pixels of dX
  return tc::run_igemm(1, dy, wd, dx, dtype, dx_dtype, N, Ho, Wo, Cout, H, W, Cin, R, S, stride, (cudaStream_t)stream,
                       "conv2d_dgrad_tc");
}

static int wgrad_tc_impl(const void* x, const void* dy, float* dw, int dtype, int64_t N, int64_t H, int64_t W,
                         int64_t Cs, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream,
                         bool zero) {
  using namespace simclr::tc;
  SIMCLR_CHECK_ARG(x && dy && dw, "conv2d_wgrad_tc: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cin > 0 && Cs >= Cin && Cout > 0 && R > 0 && S > 0 && (R & 1) && (S & 1) && stride > 0,
                   "conv2d_wgrad_tc: bad geometry");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SIMCLR_F32) {
    // wgmma takes tf32 operands K-major only, and both wgrad operands are MN-major; fp32 storage is the verification mode and takes its wgrad from the CUDA-core engine.
    set_error("conv2d_wgrad_tc: fp32 operands are not supported (use conv2d_wgrad_simt)");
    return SIMCLR_ERR_UNSUPPORTED;
  }
  if (halo3x3_wgrad_applicable(dtype, N, H, W, Cs, Cin, Cout, R, S, stride, x, dy, dw))
    return run_halo3x3_wgrad(x, dy, dw, N, H, W, st, zero);
  if (stem7x7_wgrad_applicable(dtype, N, H, W, Cs, Cin, Cout, R, S, stride, x, dy, dw))
    return run_stem7x7_wgrad(x, dy, dw, N, H, W, Cin, st, zero);
  const int es = dtype == SIMCLR_BF16 ? 2 : 4;
  const int ATOM_E = 128 / es, CH = 16 / es;
  bool smallc = (dtype == SIMCLR_BF16 && Cs == 4);
  if (!(Cs % CH == 0 || smallc)) { set_error("conv2d_wgrad_tc: stored channels (%lld) must be a multiple of %d", (long long)Cs, CH); return SIMCLR_ERR_UNSUPPORTED; }
  if ((Cout * es) % 16 != 0) { set_error("conv2d_wgrad_tc: Cout*elt must be a multiple of 16 bytes"); return SIMCLR_ERR_UNSUPPORTED; }
  SIMCLR_CHECK_ARG(aligned16(x) && aligned16(dy), "conv2d_wgrad_tc: operands must be 16-byte aligned");
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int64_t M = N * Ho * Wo;
  if (M >= (1ll << 31)) { set_error("conv2d_wgrad_tc: M too large"); return SIMCLR_ERR_UNSUPPORTED; }
  const int pxs = dtype == SIMCLR_BF16 ? 64 : 32;
  const int bn = pick_bn(Cout);
  // the stem's K order and its pixel-pair reading (see run_igemm); dW keeps the [R][S][Cin][Cout] layout
  const StemGeom sg = stem_geom(smallc, 0, W, S, stride);
  const bool stem = smallc;
  int64_t Wg = W;
  if (sg.pairs) { smallc = false; Cs = 8; Wg = sg.W; }
  const int64_t Sk = stem ? sg.S : S;
  Geom g;
  g.src = x; g.out = nullptr; g.mode = 0;
  g.H = (int)H; g.W = (int)Wg; g.C = (int)Cs; g.R = (int)R; g.S = (int)Sk; g.RS = (int)(R * Sk);
  g.stride = (int)stride; g.pad_h = (int)((R - 1) / 2); g.pad_w = (int)((S - 1) / 2);
  g.stride_w = (int)stride; g.s2 = 0;
  if (stem) { g.pad_w = sg.pad_w; g.stride_w = sg.stride_w; g.s2 = (int)S + 1; }
  g.dPQ = FastDiv((uint32_t)(Ho * Wo)); g.dQ = FastDiv((uint32_t)Wo); g.dC = FastDiv((uint32_t)Cs); g.dS = FastDiv((uint32_t)Sk);
  g.P = (int)Ho; g.Q = (int)Wo; g.adv_p = pxs / (int)Wo; g.adv_q = pxs % (int)Wo;
  g.M = M; g.n_out = (int)Cout; g.ldc = (int)Cout;
  g.num_kb = (int)((M + pxs - 1) / pxs);
  g.tiles_m = (int)((R * Sk * Cs + 127) / 128); g.tiles_n = (int)((Cout + bn - 1) / bn);
  g.Cin = (int)Cin; g.Cout = (int)Cout;
  g.use_tab = 0; g.cblocks = 1; g.os = 0; g.oh0 = g.ow0 = 0; g.OH = g.OW = 0; g.tap_sign = 1; g.accum = 0;
  g.ws = nullptr; g.ws_stride = 0;
  const int tiles = g.tiles_m * g.tiles_n;
  int splits = (2 * num_sms() + tiles - 1) / tiles;
  const int max_splits = g.num_kb / 8 > 0 ? g.num_kb / 8 : 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  g.kb_per_split = (g.num_kb + splits - 1) / splits;
  g.splits = (g.num_kb + g.kb_per_split - 1) / g.kb_per_split;
  CUtensorMap tdy, tx;
  int rc = make_tmap_2d(&tdy, dy, es, (uint64_t)M, (uint64_t)Cout, (uint64_t)Cout * es, (uint32_t)pxs, (uint32_t)ATOM_E);
  if (rc) return rc;
  bool a_tma = (R == 1 && S == 1 && stride == 1 && !smallc && (Cs * es) % 16 == 0);
  g.im2col = 0; g.im_base = 0; g.im_nimg = (int)N;
  if (a_tma) { rc = make_tmap_2d(&tx, x, es, (uint64_t)M, (uint64_t)Cs, (uint64_t)Cs * es, (uint32_t)pxs, (uint32_t)ATOM_E); if (rc) return rc; }
  else {
    tx = tdy;
    Im2colPlan pl;
    if (!smallc && plan_im2col(0, H, W, Cs, Ho, Wo, R, S, stride, ATOM_E, &pl)) {
      rc = make_tmap_im2col(&tx, x, es, (uint64_t)N, (uint64_t)H, (uint64_t)W, (uint64_t)Cs, pl.lo, pl.up, (uint32_t)stride, (uint32_t)pxs);
      if (rc) return rc;
      g.im2col = 1; g.im_base = pl.lo; a_tma = true;
    }
  }
  // splits are combined by TMA reduce-add when dW is a plain [R*S*Cin][Cout] fp32 matrix with 16-byte rows
  CUtensorMap tdw;
  const bool tma_red = !stem && Cs == Cin && aligned16(dw) && (Cout * 4) % 16 == 0;
  const int64_t dw_elems = R * S * Cin * Cout;
  if (dtype != SIMCLR_BF16) { set_error("conv2d_wgrad_tc: unknown dtype %d", dtype); return SIMCLR_ERR_INVALID_ARG; }
  if (zero && !accumulate_prezeroed()) SIMCLR_CHECK_CUDA(cudaMemsetAsync(dw, 0, (size_t)dw_elems * sizeof(float), st));
  if (g.splits == 1) {          // every dW element is written once: reduce-add / atomics straight into dW
    if (tma_red) { rc = make_tmap_2d(&tdw, dw, 4, (uint64_t)(R * S * Cin), (uint64_t)Cout, (uint64_t)Cout * 4, 128, 32); if (rc) return rc; }
    else tdw = tdy;
    return dispatch_wgrad<__nv_bfloat16>(bn, smallc, a_tma, tma_red, tx, tdy, tdw, g, dw, st);
  }
  // partials: TMA-stored tiles [splits][tiles_m * 128 rows][Cout] (the rows of a split past R*S*Cin are never read),
  // or the dW layout per split for the scattered (stem / padded-channel) rows
  g.ws_stride = tma_red ? (long long)g.tiles_m * 128 * Cout : (long long)dw_elems;
  rc = scratch_alloc(&g.ws, (size_t)g.splits * g.ws_stride * sizeof(float), st);
  if (rc) return rc;
  if (tma_red) rc = make_tmap_2d(&tdw, g.ws, 4, (uint64_t)g.splits * g.tiles_m * 128, (uint64_t)Cout, (uint64_t)Cout * 4, 128, 32);
  else tdw = tdy;
  if (!rc) rc = dispatch_wgrad<__nv_bfloat16>(bn, smallc, a_tma, tma_red, tx, tdy, tdw, g, dw, st);
  if (!rc) rc = run_sum_partials(g.ws, g.ws_stride, dw, dw_elems, g.splits, st);
  const int rf = scratch_free(g.ws, st);
  return rc ? rc : rf;
}

int simclr_conv2d_wgrad_tc(const void* x, const void* dy, float* dw, int dtype, int64_t N, int64_t H, int64_t W,
                           int64_t Cs, int64_t Cin, int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream) {
  return wgrad_tc_impl(x, dy, dw, dtype, N, H, W, Cs, Cin, Cout, R, S, stride, stream, true);
}

// ---------------------------------------------------------------------------
// Split-bf16 products: fp32-accurate GEMMs on the bf16 tensor pipe.  Every fp32 operand is split three
// ways, v = v0 + v1 + v2 (8 + 8 + 8 mantissa bits, exact to 2^-25 |v|), and a product a*b is taken as
//   a0*b0 + (a0*b1 + a1*b0) + (a1*b1 + a0*b2 + a2*b0)
// -- all terms down to 2^-16 relative; what is dropped is 2^-24 -- each an exact-product / fp32-accumulate
// tensor-core GEMM, summed in fp32 at L2 (TMA reduce-add).  A two-way split (three GEMMs) leaves 2^-17 per
// operand: measured 1e-2 on the step's gradients, not enough for the 1e-3 bar.  This is the tensor-core
// verification mode: fp32 storage, 1e-3 step parity with the fp32 reference.
// ---------------------------------------------------------------------------
static const int kSplitPairs[6][2] = {{0, 0}, {0, 1}, {1, 0}, {1, 1}, {0, 2}, {2, 0}};

int simclr_conv2d_fprop_tc3(const void* x0, const void* x1, const void* x2, const void* w0, const void* w1,
                            const void* w2, float* y, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cout,
                            int64_t R, int64_t S, int64_t stride, void* stream) {
  SIMCLR_CHECK_ARG(x0 && x1 && x2 && w0 && w1 && w2 && y, "conv2d_fprop_tc3: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cs > 0 && Cout > 0 && R > 0 && S > 0 && (R & 1) && (S & 1) && stride > 0,
                   "conv2d_fprop_tc3: bad geometry");
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const void* xs[3] = {x0, x1, x2};
  const void* ws[3] = {w0, w1, w2};
  for (int p = 0; p < 6; ++p) {
    int rc = tc::run_igemm(0, xs[kSplitPairs[p][0]], ws[kSplitPairs[p][1]], y, SIMCLR_BF16, SIMCLR_F32, N, H, W, Cs, Ho, Wo,
                           Cout, R, S, stride, (cudaStream_t)stream, "conv2d_fprop_tc3", nullptr, p > 0);
    if (rc) return rc;
  }
  return SIMCLR_OK;
}

int simclr_conv2d_dgrad_tc3(const void* dy0, const void* dy1, const void* dy2, const void* w0, const void* w1,
                            const void* w2, float* dx, int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                            int64_t R, int64_t S, int64_t stride, void* stream) {
  SIMCLR_CHECK_ARG(dy0 && dy1 && dy2 && w0 && w1 && w2 && dx, "conv2d_dgrad_tc3: null pointer");
  SIMCLR_CHECK_ARG(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && R > 0 && S > 0 && (R & 1) && (S & 1) && stride > 0,
                   "conv2d_dgrad_tc3: bad geometry");
  const int64_t Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const void* ds[3] = {dy0, dy1, dy2};
  const void* ws[3] = {w0, w1, w2};
  for (int p = 0; p < 6; ++p) {
    const void* d = ds[kSplitPairs[p][0]];
    const void* w = ws[kSplitPairs[p][1]];
    int rc;
    if (stride > 1) {
      if (!(stride <= 3 && Cout % 64 == 0 && simclr::aligned16(d) && simclr::aligned16(w) && simclr::aligned16(dx))) {
        simclr::set_error("conv2d_dgrad_tc3: stride %lld needs Cout %% 64 == 0, stride <= 3 and 16-byte aligned operands", (long long)stride);
        return SIMCLR_ERR_UNSUPPORTED;
      }
      rc = tc::run_dgrad_strided(d, w, dx, SIMCLR_BF16, SIMCLR_F32, N, H, W, Cin, Cout, R, S, stride, (cudaStream_t)stream, p > 0);
    } else {
      rc = tc::run_igemm(1, d, w, dx, SIMCLR_BF16, SIMCLR_F32, N, Ho, Wo, Cout, H, W, Cin, R, S, stride,
                         (cudaStream_t)stream, "conv2d_dgrad_tc3", nullptr, p > 0);
    }
    if (rc) return rc;
  }
  return SIMCLR_OK;
}

int simclr_conv2d_wgrad_tc3(const void* x0, const void* x1, const void* x2, const void* dy0, const void* dy1,
                            const void* dy2, float* dw, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin,
                            int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream) {
  SIMCLR_CHECK_ARG(x0 && x1 && x2 && dy0 && dy1 && dy2 && dw, "conv2d_wgrad_tc3: null pointer");
  const void* xs[3] = {x0, x1, x2};
  const void* ds[3] = {dy0, dy1, dy2};
  for (int p = 0; p < 6; ++p) {
    int rc = wgrad_tc_impl(xs[kSplitPairs[p][0]], ds[kSplitPairs[p][1]], dw, SIMCLR_BF16, N, H, W, Cs, Cin, Cout, R, S, stride,
                           stream, p == 0);
    if (rc) return rc;
  }
  return SIMCLR_OK;
}

}  // extern "C"
