// 3x3 stride-1 convolutions (fprop and dgrad) with HALO REUSE on the wgmma engine
// (tf2/resnet.py:446-455: the 3x3 of every bottleneck; 64 channels at 56x56, 128 at 28x28).
//
// The implicit-GEMM kernel of tc_conv.cu fetches every input byte once per filter tap (nine TMA
// im2col loads per K sweep): the 64/128-channel layers are bound by L2->SM traffic, not by the tensor
// pipe.  Here the input pixels of TR output rows (plus one halo row above / below and one halo
// column left / right, produced by the TMA unit's out-of-bounds zero fill) are loaded ONCE as a slab
// [TR+2][W+2][64 ch] of 128-byte, 128B-swizzled pixel rows.  GEMM row v of the tile is the "virtual
// pixel" (v / Wp, v % Wp) of a (W+2)-wide grid, so the A operand of tap (r, s) is the SAME slab seen
// from pixel offset r*Wp + s: a K-major SWIZZLE_128B descriptor whose start address is shifted by
// that many 128-byte rows (the swizzle is applied to absolute shared-memory address bits, so the
// slab stays 1024-byte aligned and only the start moves).  The two virtual columns per row
// that fall outside the image are computed and dropped (zeroed in the staging tile so the fused
// BatchNorm statistics ignore them; clipped by the TMA store).  With 64 input channels the whole
// filter (73 KB) stays resident in shared memory; wider layers stream it through a ring.
//
//   warps 0-3  consumer   9 taps x CB channel blocks x 4 K16 steps x two m64 wgmmas (N=BN) per tile, then
//                         registers -> bf16 -> 128B-swizzled staging tile -> TMA store (+ column sums)
//   warp  4    TMA        slab loads (4-D tiled boxes), filter tiles
#include "tc_common.cuh"

namespace simclr {
namespace tc {
namespace {

constexpr int SLAB_PIX = 256;                    // pixels per slab buffer (>= 127 + 2*Wp + 3)
constexpr int SLAB_BYTES = SLAB_PIX * 128;       // one 64-channel block
constexpr int EPI_TILE = 128 * 128;

struct HaloGeom {
  int H, W, Wp, TR, N;
  int tiles_per_img, num_tiles;
  int box_bytes;               // bytes one slab TMA box delivers ((TR+2) * Wp * 128)
  int n_out;                   // output channels
  int tap_base, tap_sign;      // pixel offset of the A window of tap (r, s) in the slab: tap_base + tap_sign*(r*Wp + s)
  int C;                       // input channels: tap t starts at K column t*C of the packed filter
};

template <int BN, int CB, bool B_RES> struct HaloCfg {
  static constexpr int SLAB_STAGES = (CB == 1) ? 3 : 2;
  static constexpr int SLAB_STAGE_BYTES = CB * SLAB_BYTES;
  static constexpr int B_TILE = BN * 128;                       // one (tap, channel block) filter tile
  static constexpr int B_STAGES = B_RES ? 9 * CB : 4;
  static constexpr size_t SMEM = 1024 + (size_t)SLAB_STAGES * SLAB_STAGE_BYTES + (size_t)B_STAGES * B_TILE + 2 * EPI_TILE + 512;
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"((uint64_t)tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void warp_arrive_h(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

template <int BN, int CB, bool B_RES, bool STATS>
__global__ void __launch_bounds__(160, 1)
halo3x3_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ CUtensorMap tmap_y, const HaloGeom g, double* __restrict__ bn_sums) {
  using CFG = HaloCfg<BN, CB, B_RES>;
  constexpr int SS = CFG::SLAB_STAGES, BS = CFG::B_STAGES;
  constexpr int BOXES = BN / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* slab = smem;
  uint8_t* bt = slab + (size_t)SS * CFG::SLAB_STAGE_BYTES;
  uint8_t* epi = bt + (size_t)BS * CFG::B_TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi + 2 * EPI_TILE);
  uint64_t* slab_full = bars;              // [SS]
  uint64_t* slab_empty = bars + SS;        // [SS]
  uint64_t* b_full = bars + 2 * SS;        // [BS]  (resident filter: b_full[0] only, completes once)
  uint64_t* b_empty = b_full + BS;         // [BS]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SS; ++s) { mbar_init(&slab_full[s], 1); mbar_init(&slab_empty[s], 4); }
    for (int s = 0; s < BS; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 4); }
    fence_barrier_init();
  }
  if (warp == 4 && lane == 0) { tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_w); tma_prefetch_desc(&tmap_y); }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------ consumer: MMA + epilogue ------------------------------
    // descriptor low words are running warp-uniform 32-bit sums; m64 half h is 64 virtual pixels further
    constexpr uint32_t HI = desc_hi_sw128(1024);
    int ss = 0; uint32_t sphase = 0;
    int bs = 0; uint32_t bphase = 0;
    const uint32_t slab0_lo = uniform_u32(desc_lo(smem_u32(slab), 16));
    const uint32_t bt_lo = uniform_u32(desc_lo(smem_u32(bt), 16));
    float acc[2][BN / 2];
    uint32_t box_ctr = 0;
    bool rows_in[2][2];                                 // the thread's accumulator rows: virtual pixel inside the image
    const int sj = threadIdx.x & 7, srg = threadIdx.x >> 3;
    float st_sum[BOXES][8], st_sq[BOXES][8];
#pragma unroll
    for (int b = 0; b < BOXES; ++b)
#pragma unroll
      for (int c = 0; c < 8; ++c) { st_sum[b][c] = 0.f; st_sq[b][c] = 0.f; }
    if (B_RES) { mbar_wait(&b_full[0], 0); }
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      const int n = tile / g.tiles_per_img, p0 = (tile - n * g.tiles_per_img) * g.TR;
      mbar_wait(&slab_full[ss], sphase);
      const uint32_t a_tile_lo = slab0_lo + (uint32_t)ss * (CFG::SLAB_STAGE_BYTES >> 4) + (uint32_t)g.tap_base * 8u;
      int prev_bs = 0;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int r = t / 3, sx = t % 3;
        const uint32_t a_tap_lo = a_tile_lo + (uint32_t)(g.tap_sign * (r * g.Wp + sx)) * 8u;   // 128 B per pixel
#pragma unroll
        for (int cb = 0; cb < CB; ++cb) {
          uint32_t b_lo;
          if (B_RES) {
            b_lo = bt_lo + (uint32_t)(t * CB + cb) * (CFG::B_TILE >> 4);
          } else {
            mbar_wait(&b_full[bs], bphase);
            b_lo = bt_lo + (uint32_t)bs * (CFG::B_TILE >> 4);
          }
          const uint32_t a_lo = a_tap_lo + cb * (SLAB_BYTES >> 4);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              wgmma<BN, false, false, false>(acc[h], desc_pack(a_lo + h * (64 * 128 >> 4) + 2 * k, HI), desc_pack(b_lo + 2 * k, HI),
                                             (t | cb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          if (!B_RES) {
            if (t | cb) { wgmma_wait<1>(); warp_arrive_h(&b_empty[prev_bs]); }
            prev_bs = bs;
            if (++bs == BS) { bs = 0; bphase ^= 1; }
          }
        }
      }
      wgmma_wait<0>(acc);
      if (!B_RES) warp_arrive_h(&b_empty[prev_bs]);
      warp_arrive_h(&slab_empty[ss]);
      if (++ss == SS) { ss = 0; sphase ^= 1; }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int rp = 0; rp < 2; ++rp) {
          const int row = frag_row(h, rp), vi = row / g.Wp, vj = row - vi * g.Wp;
          rows_in[h][rp] = vi < g.TR && vj < g.W && p0 + vi < g.H;      // outside the image: stored as zeros
        }
#pragma unroll
      for (int b = 0; b < BOXES; ++b, ++box_ctr) {
        uint8_t* stage = epi + (box_ctr & 1) * EPI_TILE;
        if (threadIdx.x == 0) tma_store_wait_read<1>();     // the store issued two boxes ago has read its tile
        named_barrier_sync(1, 128);
        stage_frag<__nv_bfloat16>(smem_u32(stage), acc, b * 8, rows_in);
        fence_proxy_async();
        named_barrier_sync(1, 128);
        if (threadIdx.x == 0) { tma_store_4d(&tmap_y, stage, b * 64, 0, p0, n); tma_store_commit(); }
        if (STATS) {
          float a0[8], a1[8];
#pragma unroll
          for (int c = 0; c < 8; ++c) { a0[c] = 0.f; a1[c] = 0.f; }
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint4 raw = *reinterpret_cast<const uint4*>(stage + (srg * 8 + i) * 128 + ((sj ^ i) << 4));
            const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float v0 = __uint_as_float(w[e] << 16), v1 = __uint_as_float(w[e] & 0xffff0000u);
              a0[2 * e] += v0; a1[2 * e] = fmaf(v0, v0, a1[2 * e]);
              a0[2 * e + 1] += v1; a1[2 * e + 1] = fmaf(v1, v1, a1[2 * e + 1]);
            }
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) { st_sum[b][c] += a0[c]; st_sq[b][c] += a1[c]; }
        }
      }
    }
    if (STATS) {
      // Fold the row groups of a warp by shuffles, the four warps through shared memory (the slab ring is
      // idle: the last tile's MMAs have retired), then ONE fp64 atomic per column per CTA -- same-address
      // atomics serialise in L2 (~30 ns each).
      float* red = reinterpret_cast<float*>(slab);        // [4 warps][BN columns][2]
#pragma unroll
      for (int b = 0; b < BOXES; ++b) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          float s0 = st_sum[b][c], s1 = st_sq[b][c];
          s0 += __shfl_xor_sync(0xffffffffu, s0, 8);  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
          s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
          const int lc = b * 64 + sj * 8 + c;
          if (lane < 8) { red[(warp * BN + lc) * 2] = s0; red[(warp * BN + lc) * 2 + 1] = s1; }
        }
      }
      named_barrier_sync(1, 128);
      for (int lc = threadIdx.x; lc < BN; lc += 128) {
        if ((int)blockIdx.x < g.num_tiles) {
          double s0 = 0.0, s1 = 0.0;
#pragma unroll
          for (int w = 0; w < 4; ++w) { s0 += (double)red[(w * BN + lc) * 2]; s1 += (double)red[(w * BN + lc) * 2 + 1]; }
          bn_sums[(size_t)blockIdx.x * 2 * g.n_out + lc] = s0;            // this CTA's partial (added in CTA order)
          bn_sums[(size_t)blockIdx.x * 2 * g.n_out + g.n_out + lc] = s1;
        }
      }
    }
    if (threadIdx.x == 0) tma_store_wait_all<0>();
  } else {
    // ------------------------------ TMA producer --------------------------
    if (lane == 0) {
      if (B_RES) {
        mbar_arrive_expect_tx(&b_full[0], 9 * CB * CFG::B_TILE);
        for (int t = 0; t < 9; ++t)
          for (int cb = 0; cb < CB; ++cb)
            tma_load_2d(bt + (size_t)(t * CB + cb) * CFG::B_TILE, &tmap_w, &b_full[0], t * g.C + cb * 64, 0);
      }
      int ss = 0; uint32_t sphase = 0;
      int bs = 0; uint32_t bphase = 0;
      auto load_slab = [&](int tile) {
        const int n = tile / g.tiles_per_img, p0 = (tile - n * g.tiles_per_img) * g.TR;
        mbar_wait(&slab_empty[ss], sphase ^ 1);
        mbar_arrive_expect_tx(&slab_full[ss], CB * g.box_bytes);
        for (int cb = 0; cb < CB; ++cb)
          tma_load_4d(slab + (size_t)ss * CFG::SLAB_STAGE_BYTES + cb * SLAB_BYTES, &tmap_x, &slab_full[ss], cb * 64, -1, p0 - 1, n);
        if (++ss == SS) { ss = 0; sphase ^= 1; }
      };
      if ((int)blockIdx.x < g.num_tiles) load_slab(blockIdx.x);
      for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
        // the next tile's slab goes out before this tile's filter stream: its latency hides behind the MMAs
        if (tile + (int)gridDim.x < g.num_tiles) load_slab(tile + gridDim.x);
        if (!B_RES) {
          for (int t = 0; t < 9; ++t)
            for (int cb = 0; cb < CB; ++cb) {
              mbar_wait(&b_empty[bs], bphase ^ 1);
              mbar_arrive_expect_tx(&b_full[bs], CFG::B_TILE);
              tma_load_2d(bt + (size_t)bs * CFG::B_TILE, &tmap_w, &b_full[bs], t * g.C + cb * 64, 0);
              if (++bs == BS) { bs = 0; bphase ^= 1; }
            }
        }
      }
    }
    __syncwarp();
  }

  __syncthreads();
}

// ===========================================================================
// wgrad of the 64 -> 64 channel 3x3 layers with halo reuse.
//   dW[(r,s,c)][co] = sum over pixels  X[pixel + (r,s)][c] * dY[pixel][co]
// Both operands are MN-major (the reduction K runs over pixels, rows of 128 bytes): the X slab of a tile is the
// fprop slab, and tap (r, s) is the slab shifted by r*Wp + s rows along K -- an M = 64 operand whose start is any
// 128-byte row of the 1024-byte-aligned slab.  Nine accumulators [64 x 64] (one per tap) live in registers for the
// whole kernel, three per consumer warpgroup: every CTA sweeps its tiles, then TMA-stores its [576 x 64] partial to
// its rows of a scratch buffer, and run_sum_partials adds the CTAs' partials into dW in CTA order.  The generic wgrad kernel re-fetches X once per tap and dY once per 128 filter rows: 120 KB of
// L2 -> SM traffic per 64 pixels against 24 KB here.  dY columns outside the image arrive as zeros (TMA
// out-of-bounds fill), buffer rows the boxes never write are zeroed once, so virtual pixels contribute nothing.
//
//   warps 0-11  consumers  warpgroup w owns taps 3w .. 3w + 2
//   warp  12    TMA        X slab and dY boxes
// ===========================================================================
constexpr int WG_DY_BYTES = 128 * 128;                       // [128 virtual pixels][64 co]
constexpr int WG_STAGE_BYTES = SLAB_BYTES + WG_DY_BYTES;     // 48 KB
constexpr int WG_STAGES = 3;
constexpr int WG_GROUPS = 3;                                 // consumer warpgroups
constexpr int WG_EPI_TILE = 64 * 128;                        // [64 filter rows][32 fp32]
constexpr size_t WG_SMEM = 1024 + (size_t)WG_STAGES * WG_STAGE_BYTES + WG_GROUPS * 2 * WG_EPI_TILE + 256;

__global__ void __launch_bounds__(WG_GROUPS * 128 + 32, 1)
halo3x3_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy,
                     const __grid_constant__ CUtensorMap tmap_dw, const HaloGeom g) {
  constexpr uint32_t HI = desc_hi_sw128(1024);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* epi = smem + (size_t)WG_STAGES * WG_STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi + WG_GROUPS * 2 * WG_EPI_TILE);
  uint64_t* full = bars;                     // [WG_STAGES]
  uint64_t* empty = bars + WG_STAGES;        // [WG_STAGES]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // zero the operand ring once: the TMA boxes never write the tail rows, and 0 * stale NaN would poison the sums
  for (int i = threadIdx.x; i < WG_STAGES * WG_STAGE_BYTES / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], WG_GROUPS * 4); }
    fence_barrier_init();
  }
  fence_proxy_async();
  if (warp == WG_GROUPS * 4 && lane == 0) { tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_dy); tma_prefetch_desc(&tmap_dw); }
  __syncthreads();
  const bool has_work = (int)blockIdx.x < g.num_tiles;

  if (warp < WG_GROUPS * 4) {
    // ------------------------------ consumers ------------------------------
    const int wg = warp >> 2, wt = threadIdx.x & 127;
    int ss = 0; uint32_t sphase = 0;
    const uint32_t smem_lo = uniform_u32(desc_lo(smem_u32(smem), 1024));
    const int Wp = g.Wp;
    uint32_t off[3];                                      // slab row of tap 3*wg + j (128 B per row)
#pragma unroll
    for (int j = 0; j < 3; ++j) { const int t = 3 * wg + j; off[j] = (uint32_t)((t / 3) * Wp + t % 3) * 8u; }
    float acc[3][32];
    bool first = true;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      mbar_wait(&full[ss], sphase);
      const uint32_t x_lo = smem_lo + (uint32_t)ss * (WG_STAGE_BYTES >> 4);
      const uint32_t dy_lo = x_lo + (SLAB_BYTES >> 4);
      wgmma_fence();
      // K step outermost, the three accumulators innermost: consecutive MMAs never accumulate into the same registers
#pragma unroll
      for (int k = 0; k < 8; ++k) {        // 16 pixels (16 rows of 128 B) per MMA
        const uint64_t bd = desc_pack(dy_lo + k * 128, HI);
#pragma unroll
        for (int j = 0; j < 3; ++j)
          wgmma<64, false, true, true>(acc[j], desc_pack(x_lo + off[j] + k * 128, HI), bd, (!first || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>(acc);
      warp_arrive_h(&empty[ss]);
      first = false;
      if (++ss == WG_STAGES) { ss = 0; sphase ^= 1; }
    }
    // ------------------------------ epilogue (once) ------------------------------
    if (has_work) {
      const int q = lane & 3;
      uint32_t box_ctr = 0;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
#pragma unroll
        for (int cc = 0; cc < 2; ++cc, ++box_ctr) {
          uint8_t* stage = epi + (size_t)(wg * 2 + (box_ctr & 1)) * WG_EPI_TILE;
          if (wt == 0) tma_store_wait_read<1>();
          named_barrier_sync(1 + wg, 128);
          const uint32_t srow = smem_u32(stage);
#pragma unroll
          for (int rp = 0; rp < 2; ++rp) {
            const int row = 16 * (warp & 3) + (lane >> 2) + 8 * rp;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(srow + sw128_offset(row, 2 * ii + (q >> 1)) + 8 * (q & 1)),
                           "f"(acc[j][4 * (4 * cc + ii) + 2 * rp]), "f"(acc[j][4 * (4 * cc + ii) + 2 * rp + 1]) : "memory");
          }
          fence_proxy_async();
          named_barrier_sync(1 + wg, 128);
          // rows of tap t are filter rows [t*64, t*64 + 64) of this CTA's [9*64][64] partial
          if (wt == 0) { tma_store_2d(&tmap_dw, stage, cc * 32, (int)blockIdx.x * 576 + (3 * wg + j) * 64); tma_store_commit(); }
        }
      }
      if (wt == 0) tma_store_wait_all<0>();
    }
  } else {
    // ------------------------------ TMA producer --------------------------
    if (lane == 0) {
      int ss = 0; uint32_t sphase = 0;
      for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
        const int n = tile / g.tiles_per_img, p0 = (tile - n * g.tiles_per_img) * g.TR;
        mbar_wait(&empty[ss], sphase ^ 1);
        uint8_t* st = smem + (size_t)ss * WG_STAGE_BYTES;
        mbar_arrive_expect_tx(&full[ss], g.box_bytes + g.TR * g.Wp * 128);
        tma_load_4d(st, &tmap_x, &full[ss], 0, -1, p0 - 1, n);
        tma_load_4d(st + SLAB_BYTES, &tmap_dy, &full[ss], 0, 0, p0, n);
        if (++ss == WG_STAGES) { ss = 0; sphase ^= 1; }
      }
    }
    __syncwarp();
  }

  __syncthreads();
}

// rank-4 tiled map over an NHWC tensor {C, W, H, N}, boxes {64 channels, bw, bh, 1}, 128B swizzle, zero fill
int make_tmap_nhwc_tiled(CUtensorMap* map, const void* base, uint64_t N, uint64_t H, uint64_t W, uint64_t C, uint32_t bw,
                         uint32_t bh) {
  EncodeTiledFn fn = get_encode_tiled();
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return SIMCLR_ERR_DRIVER; }
  const cuuint64_t dims[4] = {C, W, H, N};
  const cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
  const cuuint32_t box[4] = {64, bw, bh, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed (%d): N=%llu H=%llu W=%llu C=%llu box=%ux%u", (int)r, (unsigned long long)N,
              (unsigned long long)H, (unsigned long long)W, (unsigned long long)C, bw, bh);
    return SIMCLR_ERR_DRIVER;
  }
  return SIMCLR_OK;
}

template <int BN, int CB, bool B_RES, bool STATS>
int launch_halo(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& ty, const HaloGeom& g, double* bn_sums,
                cudaStream_t st) {
  auto kern = halo3x3_kernel<BN, CB, B_RES, STATS>;
  using CFG = HaloCfg<BN, CB, B_RES>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CFG::SMEM);
  if (e != cudaSuccess) { set_error("halo3x3: cudaFuncSetAttribute(smem=%zu): %s", CFG::SMEM, cudaGetErrorString(e)); return (int)e; }
  int grid = g.num_tiles < num_sms() ? g.num_tiles : num_sms();
  kern<<<grid, 160, CFG::SMEM, st>>>(tx, tw, ty, g, bn_sums);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

inline bool halo_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("SIMCLR_TC_HALO"); v = (e && e[0] == '0') ? 0 : 1; }
  return v == 1;
}

}  // namespace

bool halo3x3_applicable(int dtype, int out_dtype, int64_t N, int64_t H, int64_t W, int64_t C, int64_t n_out, int64_t R,
                        int64_t S, int64_t stride, const void* src, const void* wk, const void* out) {
  if (!halo_enabled() || dtype != SIMCLR_BF16 || out_dtype != SIMCLR_BF16 || R != 3 || S != 3 || stride != 1) return false;
  if (!((C == 64 && n_out == 64) || (C == 128 && n_out == 128))) return false;
  const int64_t Wp = W + 2;
  if (Wp > 64) return false;                            // 127 + 2*Wp + 3 <= SLAB_PIX
  const int64_t TR = 128 / Wp;
  if (TR < 1 || TR + 2 > 256) return false;
  const int64_t tiles_per_img = (H + TR - 1) / TR;
  if ((double)(H * W) / (double)(tiles_per_img * 128) < 0.80) return false;    // virtual-pixel waste
  if (N * tiles_per_img >= (1ll << 31) || N >= (1ll << 31)) return false;
  if (!aligned16(src) || !aligned16(wk) || !aligned16(out)) return false;
  return get_encode_tiled() != nullptr;
}

// mode 0: fprop, wk = wf [n_out][9*C] (k = (r*3+s)*C + c).  mode 1: stride-1 dgrad, src = dY, C = Cout of the
// conv, n_out = Cin, wk = wd [Cin][9*Cout] (k = (r*3+s)*Cout + co): dX[p,q] = sum dY[p+1-r, q+1-s] W[r,s].
int run_halo3x3(int mode, const void* src, const void* wk, void* out, int64_t N, int64_t H, int64_t W, int64_t C,
                int64_t n_out, cudaStream_t st, double* bn_sums) {
  HaloGeom g;
  g.H = (int)H; g.W = (int)W; g.Wp = (int)W + 2; g.TR = 128 / g.Wp; g.N = (int)N;
  g.tiles_per_img = (int)((H + g.TR - 1) / g.TR); g.num_tiles = (int)(N * g.tiles_per_img);
  g.box_bytes = (g.TR + 2) * g.Wp * 128; g.n_out = (int)n_out;
  g.C = (int)C;
  g.tap_base = mode == 0 ? 0 : 2 * g.Wp + 2;        // dgrad: dX[p,q] = sum dY[p+1-r, q+1-s] W[r,s]: flipped window
  g.tap_sign = mode == 0 ? 1 : -1;
  const int64_t K = 9 * C;
  CUtensorMap tx, tw, ty;
  int rc = make_tmap_nhwc_tiled(&tx, src, (uint64_t)N, (uint64_t)H, (uint64_t)W, (uint64_t)C, (uint32_t)g.Wp, (uint32_t)(g.TR + 2));
  if (rc) return rc;
  rc = make_tmap_2d(&tw, wk, 2, (uint64_t)n_out, (uint64_t)K, (uint64_t)K * 2, (uint32_t)n_out, 64);
  if (rc) return rc;
  rc = make_tmap_nhwc_tiled(&ty, out, (uint64_t)N, (uint64_t)H, (uint64_t)W, (uint64_t)n_out, (uint32_t)g.Wp, (uint32_t)g.TR);
  if (rc) return rc;
  if (bn_sums && !accumulate_prezeroed()) {
    cudaError_t e = cudaMemsetAsync(bn_sums, 0, 2 * (size_t)n_out * sizeof(double), st);
    if (e != cudaSuccess) { set_error("halo3x3: memset: %s", cudaGetErrorString(e)); return (int)e; }
  }
  if (!bn_sums) return C == 64 ? launch_halo<64, 1, true, false>(tx, tw, ty, g, nullptr, st)
                                : launch_halo<128, 2, false, false>(tx, tw, ty, g, nullptr, st);
  // fused statistics: one [2][n_out] partial per CTA, added into bn_sums in CTA order
  const int nparts = num_sms();
  double* parts = nullptr;
  rc = scratch_alloc(&parts, (size_t)nparts * 2 * n_out * sizeof(double), st);
  if (rc) return rc;
  const cudaError_t e = cudaMemsetAsync(parts, 0, (size_t)nparts * 2 * n_out * sizeof(double), st);
  if (e != cudaSuccess) { set_error("halo3x3: memset: %s", cudaGetErrorString(e)); scratch_free(parts, st); return (int)e; }
  rc = C == 64 ? launch_halo<64, 1, true, true>(tx, tw, ty, g, parts, st) : launch_halo<128, 2, false, true>(tx, tw, ty, g, parts, st);
  if (!rc) rc = run_sum_partials_f64(parts, 2 * n_out, bn_sums, 2 * n_out, nparts, st);
  const int rf = scratch_free(parts, st);
  return rc ? rc : rf;
}

bool halo3x3_wgrad_applicable(int dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                              int64_t S, int64_t stride, const void* x, const void* dy, const void* dw) {
  static int en = -1;
  if (en < 0) { const char* e = getenv("SIMCLR_TC_HALO_WGRAD"); en = (e && e[0] == '0') ? 0 : 1; }
  if (!en || !halo_enabled() || dtype != SIMCLR_BF16 || R != 3 || S != 3 || stride != 1) return false;
  if (Cs != 64 || Cin != 64 || Cout != 64) return false;
  const int64_t Wp = W + 2;
  if (Wp > 64) return false;
  const int64_t TR = 128 / Wp;
  if (TR < 1) return false;
  const int64_t tiles_per_img = (H + TR - 1) / TR;
  if ((double)(H * W) / (double)(tiles_per_img * 128) < 0.80) return false;
  if (N * tiles_per_img >= (1ll << 31)) return false;
  if (!aligned16(x) || !aligned16(dy) || !aligned16(dw)) return false;
  return get_encode_tiled() != nullptr;
}

int run_halo3x3_wgrad(const void* x, const void* dy, float* dw, int64_t N, int64_t H, int64_t W, cudaStream_t st, bool zero) {
  HaloGeom g;
  g.H = (int)H; g.W = (int)W; g.Wp = (int)W + 2; g.TR = 128 / g.Wp; g.N = (int)N;
  g.tiles_per_img = (int)((H + g.TR - 1) / g.TR); g.num_tiles = (int)(N * g.tiles_per_img);
  g.box_bytes = (g.TR + 2) * g.Wp * 128; g.n_out = 64; g.C = 64; g.tap_base = 0; g.tap_sign = 1;
  const int grid = g.num_tiles < num_sms() ? g.num_tiles : num_sms();
  CUtensorMap tx, tdy, tdw;
  int rc = make_tmap_nhwc_tiled(&tx, x, (uint64_t)N, (uint64_t)H, (uint64_t)W, 64, (uint32_t)g.Wp, (uint32_t)(g.TR + 2));
  if (rc) return rc;
  rc = make_tmap_nhwc_tiled(&tdy, dy, (uint64_t)N, (uint64_t)H, (uint64_t)W, 64, (uint32_t)g.Wp, (uint32_t)g.TR);
  if (rc) return rc;
  if (zero && !accumulate_prezeroed()) SIMCLR_CHECK_CUDA(cudaMemsetAsync(dw, 0, (size_t)9 * 64 * 64 * sizeof(float), st));
  float* ws = nullptr;                                      // [grid][576][64] per-CTA partials
  rc = scratch_alloc(&ws, (size_t)grid * 576 * 64 * sizeof(float), st);
  if (rc) return rc;
  rc = make_tmap_2d(&tdw, ws, 4, (uint64_t)grid * 576, 64, 64 * 4, 64, 32);
  if (rc) { scratch_free(ws, st); return rc; }
  cudaError_t e = cudaFuncSetAttribute(halo3x3_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM);
  if (e != cudaSuccess) { set_error("halo3x3_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); scratch_free(ws, st); return (int)e; }
  halo3x3_wgrad_kernel<<<grid, WG_GROUPS * 128 + 32, WG_SMEM, st>>>(tx, tdy, tdw, g);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("halo3x3_wgrad: launch: %s", cudaGetErrorString(e)); scratch_free(ws, st); return (int)e; }
  rc = run_sum_partials(ws, 576 * 64, dw, 576 * 64, grid, st);
  const int rf = scratch_free(ws, st);
  return rc ? rc : rf;
}

}  // namespace tc
}  // namespace simclr
