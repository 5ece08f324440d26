// The stem convolution (tf2/resnet.py:593-604: 7x7, stride 2, 3 -> 64*width channels on the 224x224 input) on the
// wgmma engine WITHOUT an im2col copy.
//
// The generic kernel gathers every A row (one output pixel: 7 filter rows x 64 bytes) with cp.async from L2: 57 KB
// per 128-pixel tile against 6 KB of distinct input -- the layer ran at 0.23 of its HBM roofline, bound by L2 -> SM
// traffic.  Here the 7 input rows of ONE output row are loaded once by TMA as a slab [7][Q + 3 pixel pairs][16 B]
// (4 stored channels: a "pair" = 2 pixels = 8 bf16 = 16 bytes; out-of-image pairs arrive as zeros).  For output pixel
// q and filter row r the K run (8 column slots x 4 channels; slot 0 has zero weights, see simclr_pack_conv_weight) is
// the 64 contiguous bytes starting at pair q of slab row r.  Neighbouring output pixels start ONE pair apart, so the
// A operand of filter row r is a K-major, NON-swizzled wgmma operand whose 8-row x 16-byte core matrices overlap:
// row pitch 16 B, leading (K) byte offset 16 B, stride (8-row group) byte offset 128 B, start = slab row r.  A tile
// is one output row: M = 128 GEMM rows of which Q are real (rows >= Q read stale shared memory and are dropped),
// 7 x 2 K16 steps x two m64 wgmmas (N=BN <= 128).  The packed filter [BN][256] stays resident in shared memory;
// BatchNorm statistics are taken in the epilogue.
//
//   warps 0-3  consumer   MMAs, then registers -> bf16 -> 128B-swizzled staging tile -> TMA store (+ column sums)
//   warp  4    TMA        slab loads (4-D tiled boxes), filter
#include "tc_common.cuh"

namespace simclr {
namespace tc {
namespace {

constexpr int ST_EPI_TILE = 128 * 128;
constexpr int ST_SLAB_STAGES = 3;
constexpr int ST_KB = 4;                          // K blocks of 64 (7 filter rows x 32, padded to 256)

struct StemGeom7 {
  int P, Q, N;
  int num_tiles;                 // N * P: one output row per tile
  int box_pairs;                 // Q + 3: pairs (16 B) per slab row = slab row pitch / 16
  int slab_stage_bytes;          // 7 * box_pairs * 16 + overread slack, 128-byte multiple
  int box_bytes;                 // bytes one TMA box delivers
  int n_out;
  FoldArgs fold;                 // FOLD: folded BatchNorm epilogue (fold_epilogue), no residual
};

template <int BN> struct StemCfg {
  static constexpr int B_TILE = BN * 128;                          // one K block of the filter
  static size_t smem(int slab_stage_bytes) {
    return 1024 + (size_t)ST_SLAB_STAGES * slab_stage_bytes + (size_t)ST_KB * B_TILE + 2 * ST_EPI_TILE + 256;
  }
};

__device__ __forceinline__ void st_tma_load_4d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void warp_arrive_st(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

template <int BN, bool STATS, bool FOLD>
__global__ void __launch_bounds__(160, 1)
stem7x7_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
               const __grid_constant__ CUtensorMap tmap_y, const StemGeom7 g, double* __restrict__ bn_sums) {
  using CFG = StemCfg<BN>;
  constexpr int SS = ST_SLAB_STAGES;
  constexpr int BOXES = BN / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bt = smem;                                              // [ST_KB][BN][128 B], 128B-swizzled (1024-aligned tiles)
  uint8_t* epi = bt + (size_t)ST_KB * CFG::B_TILE;                 // 2 staging tiles
  uint8_t* slab = epi + 2 * ST_EPI_TILE;                           // [SS][slab_stage_bytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(slab + (size_t)SS * g.slab_stage_bytes);
  uint64_t* slab_full = bars;              // [SS]
  uint64_t* slab_empty = bars + SS;        // [SS]
  uint64_t* b_full = bars + 2 * SS;        // [1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SS; ++s) { mbar_init(&slab_full[s], 1); mbar_init(&slab_empty[s], 4); }
    mbar_init(b_full, 1);
    fence_barrier_init();
  }
  if (warp == 4 && lane == 0) { tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_w); tma_prefetch_desc(&tmap_y); }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------ consumer: MMA + epilogue ------------------------------
    // descriptor low words are running warp-uniform 32-bit values (see tc_halo.cu); A: no swizzle, LBO 16 B, SBO 128 B,
    // m64 half h starts 64 pixel pairs (1024 B) further
    constexpr uint32_t HI_B = desc_hi_sw128(1024);
    constexpr uint32_t HI_A = desc_hi_none(128);
    int ss = 0; uint32_t sphase = 0;
    const uint32_t slab0_lo = uniform_u32(desc_lo(smem_u32(slab), 16));
    const uint32_t bt_lo = uniform_u32(desc_lo(smem_u32(bt), 16));
    const uint32_t stage16 = (uint32_t)(g.slab_stage_bytes >> 4), pitch16 = (uint32_t)g.box_pairs;
    float acc[2][BN / 2];
    uint32_t box_ctr = 0;
    bool rows_in[2][2];                                 // output pixel q of the accumulator row exists
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int rp = 0; rp < 2; ++rp) rows_in[h][rp] = frag_row(h, rp) < g.Q;
    const int sj = threadIdx.x & 7, srg = threadIdx.x >> 3;
    float st_sum[BOXES][8], st_sq[BOXES][8];
#pragma unroll
    for (int b = 0; b < BOXES; ++b)
#pragma unroll
      for (int c = 0; c < 8; ++c) { st_sum[b][c] = 0.f; st_sq[b][c] = 0.f; }
    mbar_wait(b_full, 0);
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      mbar_wait(&slab_full[ss], sphase);
      const uint32_t a_tile_lo = slab0_lo + (uint32_t)ss * stage16;
      wgmma_fence();
#pragma unroll
      for (int r = 0; r < 7; ++r) {
        const uint32_t a_lo = a_tile_lo + (uint32_t)r * pitch16;
        const uint32_t b_lo = bt_lo + (uint32_t)(r >> 1) * (CFG::B_TILE >> 4) + (uint32_t)(r & 1) * 4u;
#pragma unroll
        for (int k = 0; k < 2; ++k)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            wgmma<BN, false, false, false>(acc[h], desc_pack(a_lo + h * 64 + 2 * k, HI_A), desc_pack(b_lo + 2 * k, HI_B),
                                           (r | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>(acc);
      warp_arrive_st(&slab_empty[ss]);
      if (++ss == SS) { ss = 0; sphase ^= 1; }
      if (FOLD) {
        const long long roff[2][2] = {{-1, -1}, {-1, -1}};     // no residual
        fold_epilogue(acc, g.fold, 0, g.n_out, roff);
      }
#pragma unroll
      for (int b = 0; b < BOXES; ++b, ++box_ctr) {
        uint8_t* stage = epi + (box_ctr & 1) * ST_EPI_TILE;
        if (threadIdx.x == 0) tma_store_wait_read<1>();     // the store issued two boxes ago has read its tile
        named_barrier_sync(1, 128);
        stage_frag<__nv_bfloat16>(smem_u32(stage), acc, b * 8, rows_in);   // GEMM rows beyond the image row: zeros
        fence_proxy_async();
        named_barrier_sync(1, 128);
        // output rows of this tile: pixels tile*Q .. tile*Q + Q - 1 of the [N*P*Q][n_out] view (the box is Q rows high)
        if (threadIdx.x == 0) { tma_store_2d(&tmap_y, stage, b * 64, tile * g.Q); tma_store_commit(); }
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
      // fold the row groups of a warp by shuffles, the four warps through shared memory (staging tile 0 is free once
      // its last store has been read), then ONE fp64 atomic per column per CTA
      if (threadIdx.x == 0) tma_store_wait_read<0>();
      named_barrier_sync(1, 128);
      float* red = reinterpret_cast<float*>(epi);        // [4 warps][BN columns][2]  (<= 4 KB)
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
      mbar_arrive_expect_tx(b_full, ST_KB * CFG::B_TILE);
      for (int kb = 0; kb < ST_KB; ++kb) tma_load_2d(bt + (size_t)kb * CFG::B_TILE, &tmap_w, b_full, kb * 64, 0);
      int ss = 0; uint32_t sphase = 0;
      for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
        const int n = tile / g.P, p = tile - n * g.P;
        mbar_wait(&slab_empty[ss], sphase ^ 1);
        mbar_arrive_expect_tx(&slab_full[ss], g.box_bytes);
        // pairs -2 .. Q (column 2q - 4 + slot), rows 2p - 3 .. 2p + 3; everything outside the image is zero-filled
        st_tma_load_4d(slab + (size_t)ss * g.slab_stage_bytes, &tmap_x, &slab_full[ss], 0, -2, 2 * p - 3, n);
        if (++ss == SS) { ss = 0; sphase ^= 1; }
      }
    }
    __syncwarp();
  }

  __syncthreads();
}

// ===========================================================================
// wgrad of the stem from the same slab:  dW[(r, slot, c)][co] = sum over pixels  X[slab row r, pair q + slot/2][..] * dY[q][co]
// computed transposed, D_r[co][k'] (k' = slot*4 + c, 32 per filter row) = sum_q dY[q][co] * slab_r[q][k']:
//   A = dY tile [pixels][64 co]   MN-major, 128B-swizzled (M = 64 output channels, K = pixels), TMA box of Q rows
//   B = slab row r                MN-major, NOT swizzled: 8 k' (16 B) x 8 pixels (16 B apart) core matrices; the next
//                                 8 k' sit ONE pair further (16 B, overlapping), the next 8 pixels 128 B further
// Seven accumulators [64 x 32] (one per filter row) live in registers for the whole kernel; every CTA sweeps its output
// rows and stores its partial dW [7][7][Cin][64] to its slot of a scratch buffer; run_sum_partials adds the CTAs'
// partials into dW in CTA order.  Operand buffers are zeroed
// once: dY rows beyond Q stay zero (the TMA box never writes them), so padded pixels contribute nothing.
//   warps 0-3  consumer (MMAs, then the partial)      warp 4  TMA
// ===========================================================================
constexpr int SWG_STAGES = 3;
struct StemWGeom {
  int P, Q, N, num_tiles;
  int box_pairs, box_bytes;      // slab box
  int ksteps;                    // ceil(Q / 16) MMAs (K = 16 pixels) per filter row
  int dy_bytes, stage_bytes;     // dY part (ksteps * 2048) and whole stage (1024-byte multiple)
  int Cin;
};

__global__ void __launch_bounds__(160, 1)
stem7x7_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy,
                     const StemWGeom g, float* __restrict__ ws) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)SWG_STAGES * g.stage_bytes);
  uint64_t* full = bars;                      // [SWG_STAGES]
  uint64_t* empty = bars + SWG_STAGES;        // [SWG_STAGES]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < SWG_STAGES * g.stage_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x == 0) {
    for (int s = 0; s < SWG_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    fence_barrier_init();
  }
  fence_proxy_async();
  if (warp == 4 && lane == 0) { tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_dy); }
  __syncthreads();
  const bool has_work = (int)blockIdx.x < g.num_tiles;

  if (warp < 4) {
    // ------------------------------ consumer ------------------------------
    constexpr uint32_t HI_A = desc_hi_sw128(1024);
    // slab operand, MN-major without swizzle: SBO = stride between 8-k' core matrices (16 B, overlapping),
    // LBO = stride between 8-pixel groups (128 B) -- the roles are the reverse of the swizzled MN-major layouts
    constexpr uint32_t HI_B = desc_hi_none(16);
    const uint32_t lbo_b = uniform_u32(8u << 16);                // LBO field
    int ss = 0; uint32_t sphase = 0;
    const uint32_t smem_lo = uniform_u32((smem_u32(smem) & 0x3FFFFu) >> 4);
    const uint32_t stage16 = (uint32_t)(g.stage_bytes >> 4), dy16 = (uint32_t)(g.dy_bytes >> 4), pitch16 = (uint32_t)g.box_pairs;
    float acc[7][16];
    bool first = true;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      mbar_wait(&full[ss], sphase);
      const uint32_t dy_lo = (smem_lo + (uint32_t)ss * stage16) | (1u << 16);
      const uint32_t x_lo = (smem_lo + (uint32_t)ss * stage16 + dy16) | lbo_b;
      wgmma_fence();
      // K step outermost: consecutive MMAs go to seven DIFFERENT accumulators (no back-to-back dependence on one)
#pragma unroll 1
      for (int ks = 0; ks < g.ksteps; ++ks) {       // 16 pixels per MMA: 16 dY rows of 128 B, 16 pairs of the slab row
        const uint64_t ad = desc_pack(dy_lo + ks * 128, HI_A);
#pragma unroll
        for (int r = 0; r < 7; ++r)
          wgmma<32, false, true, true>(acc[r], ad, desc_pack(x_lo + r * pitch16 + ks * 16, HI_B), (!first || ks > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>(acc);
      warp_arrive_st(&empty[ss]);
      first = false;
      if (++ss == SWG_STAGES) { ss = 0; sphase ^= 1; }
    }
    // ------------------------------ epilogue (once) ------------------------------
    if (has_work) {
      float* dw = ws + (size_t)blockIdx.x * 49 * g.Cin * 64;
      // acc[r][4*i + v]: output channel 16*warp + lane/4 + 8*(v >> 1), k' = 8*i + 2*(lane % 4) + (v & 1)
#pragma unroll
      for (int r = 0; r < 7; ++r) {
#pragma unroll
        for (int v = 0; v < 16; ++v) {
          const int co = 16 * warp + (lane >> 2) + 8 * ((v & 3) >> 1);
          const int j = 8 * (v >> 2) + 2 * (lane & 3) + (v & 1);
          const int sp = j >> 2, c = j & 3;                 // column slot (0: the zero slot), stored channel
          if (sp >= 1 && c < g.Cin) dw[((size_t)((r * 7 + sp - 1) * g.Cin + c)) * 64 + co] = acc[r][v];
        }
      }
    }
  } else {
    // ------------------------------ TMA producer --------------------------
    if (lane == 0) {
      int ss = 0; uint32_t sphase = 0;
      for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
        const int n = tile / g.P, p = tile - n * g.P;
        mbar_wait(&empty[ss], sphase ^ 1);
        uint8_t* st = smem + (size_t)ss * g.stage_bytes;
        mbar_arrive_expect_tx(&full[ss], g.box_bytes + g.Q * 128);
        tma_load_2d(st, &tmap_dy, &full[ss], 0, tile * g.Q);
        st_tma_load_4d(st + g.dy_bytes, &tmap_x, &full[ss], 0, -2, 2 * p - 3, n);
        if (++ss == SWG_STAGES) { ss = 0; sphase ^= 1; }
      }
    }
    __syncwarp();
  }

  __syncthreads();
}

// x [N][H][W][4] bf16 seen as [N][H][W/2][8]: 16-byte pixel pairs, no swizzle
int make_tmap_pairs(CUtensorMap* map, const void* base, uint64_t N, uint64_t H, uint64_t W2, uint32_t box_pairs, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_tiled();
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return SIMCLR_ERR_DRIVER; }
  const cuuint64_t dims[4] = {8, W2, H, N};
  const cuuint64_t strides[3] = {16, W2 * 16, H * W2 * 16};
  const cuuint32_t box[4] = {8, box_pairs, box_rows, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(stem pairs) failed (%d): N=%llu H=%llu W/2=%llu box=%ux%u", (int)r, (unsigned long long)N,
              (unsigned long long)H, (unsigned long long)W2, box_pairs, box_rows);
    return SIMCLR_ERR_DRIVER;
  }
  return SIMCLR_OK;
}

template <int BN, bool STATS, bool FOLD = false>
int launch_stem(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& ty, const StemGeom7& g, double* bn_sums,
                cudaStream_t st) {
  auto kern = stem7x7_kernel<BN, STATS, FOLD>;
  const size_t smem = StemCfg<BN>::smem(g.slab_stage_bytes);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { set_error("stem7x7: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e)); return (int)e; }
  const int grid = g.num_tiles < num_sms() ? g.num_tiles : num_sms();
  kern<<<grid, 160, smem, st>>>(tx, tw, ty, g, bn_sums);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

inline int slab_stage_bytes(int64_t Q) {
  // 7 rows of Q + 3 pairs, plus the pairs GEMM rows Q .. 127 (+3) reach beyond the last slab row
  const int64_t b = 7 * (Q + 3) * 16 + (131 - (Q + 3) > 0 ? (131 - (Q + 3)) * 16 : 0) + 16;
  return (int)((b + 127) / 128 * 128);
}

}  // namespace

bool stem7x7_applicable(int dtype, int out_dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t n_out, int64_t R,
                        int64_t S, int64_t stride, int64_t P, int64_t Q, const void* src, const void* wk, const void* out) {
  static int en = -1;
  if (en < 0) { const char* e = getenv("SIMCLR_TC_STEM"); en = (e && e[0] == '0') ? 0 : 1; }
  if (!en || dtype != SIMCLR_BF16 || out_dtype != SIMCLR_BF16 || Cs != 4 || R != 7 || S != 7 || stride != 2) return false;
  if (!(n_out == 64 || n_out == 128) || W % 2 || H % 2 || P != H / 2 || Q != W / 2) return false;
  if (Q < 8 || Q > 128 || Q + 3 > 256) return false;
  if (N * P >= (1ll << 31) / 128) return false;
  if (!aligned16(src) || !aligned16(wk) || !aligned16(out)) return false;
  const size_t smem = n_out == 64 ? StemCfg<64>::smem(slab_stage_bytes(Q)) : StemCfg<128>::smem(slab_stage_bytes(Q));
  if (smem > 227 * 1024) return false;
  return get_encode_tiled() != nullptr;
}

// src [N][H][W][4] bf16, wk [n_out][256] (K = r*32 + slot*4 + c, slot 0 zero), out [N][P][Q][n_out] bf16
int run_stem7x7(const void* src, const void* wk, void* out, int64_t N, int64_t H, int64_t W, int64_t n_out, cudaStream_t st,
                double* bn_sums, const FoldArgs* fold) {
  StemGeom7 g;
  g.P = (int)(H / 2); g.Q = (int)(W / 2); g.N = (int)N; g.num_tiles = (int)(N * g.P);
  g.box_pairs = g.Q + 3; g.slab_stage_bytes = slab_stage_bytes(g.Q); g.box_bytes = 7 * g.box_pairs * 16; g.n_out = (int)n_out;
  CUtensorMap tx, tw, ty;
  int rc = make_tmap_pairs(&tx, src, (uint64_t)N, (uint64_t)H, (uint64_t)(W / 2), (uint32_t)g.box_pairs, 7);
  if (rc) return rc;
  rc = make_tmap_2d(&tw, wk, 2, (uint64_t)n_out, 256, 512, (uint32_t)n_out, 64);
  if (rc) return rc;
  rc = make_tmap_2d(&ty, out, 2, (uint64_t)(N * g.P * g.Q), (uint64_t)n_out, (uint64_t)n_out * 2, (uint32_t)g.Q, 64);
  if (rc) return rc;
  if (bn_sums && !accumulate_prezeroed()) {
    cudaError_t e = cudaMemsetAsync(bn_sums, 0, 2 * (size_t)n_out * sizeof(double), st);
    if (e != cudaSuccess) { set_error("stem7x7: memset: %s", cudaGetErrorString(e)); return (int)e; }
  }
  if (fold) {
    g.fold = *fold;
    return n_out == 64 ? launch_stem<64, false, true>(tx, tw, ty, g, nullptr, st) : launch_stem<128, false, true>(tx, tw, ty, g, nullptr, st);
  }
  if (!bn_sums) return n_out == 64 ? launch_stem<64, false>(tx, tw, ty, g, nullptr, st) : launch_stem<128, false>(tx, tw, ty, g, nullptr, st);
  // fused statistics: one [2][n_out] partial per CTA, added into bn_sums in CTA order
  const int nparts = num_sms();
  double* parts = nullptr;
  rc = scratch_alloc(&parts, (size_t)nparts * 2 * n_out * sizeof(double), st);
  if (rc) return rc;
  const cudaError_t e = cudaMemsetAsync(parts, 0, (size_t)nparts * 2 * n_out * sizeof(double), st);
  if (e != cudaSuccess) { set_error("stem7x7: memset: %s", cudaGetErrorString(e)); scratch_free(parts, st); return (int)e; }
  rc = n_out == 64 ? launch_stem<64, true>(tx, tw, ty, g, parts, st) : launch_stem<128, true>(tx, tw, ty, g, parts, st);
  if (!rc) rc = run_sum_partials_f64(parts, 2 * n_out, bn_sums, 2 * n_out, nparts, st);
  const int rf = scratch_free(parts, st);
  return rc ? rc : rf;
}

bool stem7x7_wgrad_applicable(int dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                              int64_t S, int64_t stride, const void* x, const void* dy, const void* dw) {
  const char* e = getenv("SIMCLR_TC_STEM_WGRAD");
  if (e && e[0] == '0') return false;
  if (dtype != SIMCLR_BF16 || Cs != 4 || Cin > 4 || Cout != 64 || R != 7 || S != 7 || stride != 2) return false;
  if (W % 2 || H % 2) return false;
  const int64_t Q = W / 2;
  if (Q < 8 || Q > 128) return false;
  if (N * (H / 2) >= (1ll << 31) / 128) return false;
  if (!aligned16(x) || !aligned16(dy) || !aligned16(dw)) return false;
  return get_encode_tiled() != nullptr;
}

// x [N][H][W][4] bf16, dy [N][H/2][W/2][64] bf16, dw [7][7][Cin][64] fp32 (+=)
int run_stem7x7_wgrad(const void* x, const void* dy, float* dw, int64_t N, int64_t H, int64_t W, int64_t Cin, cudaStream_t st,
                      bool zero) {
  StemWGeom g;
  g.P = (int)(H / 2); g.Q = (int)(W / 2); g.N = (int)N; g.num_tiles = (int)(N * g.P);
  g.box_pairs = g.Q + 3; g.box_bytes = 7 * g.box_pairs * 16;
  g.ksteps = (g.Q + 15) / 16;
  g.dy_bytes = g.ksteps * 2048;
  // slab part: 7 rows + the pairs the last K step of the last filter row reaches beyond them
  const int slab = 6 * g.box_pairs * 16 + (g.ksteps * 16 + 3) * 16 + 16;
  const int slab_b = slab > 7 * g.box_pairs * 16 ? slab : 7 * g.box_pairs * 16;
  g.stage_bytes = (g.dy_bytes + slab_b + 1023) / 1024 * 1024;
  g.Cin = (int)Cin;
  CUtensorMap tx, tdy;
  int rc = make_tmap_pairs(&tx, x, (uint64_t)N, (uint64_t)H, (uint64_t)(W / 2), (uint32_t)g.box_pairs, 7);
  if (rc) return rc;
  rc = make_tmap_2d(&tdy, dy, 2, (uint64_t)(N * g.P * g.Q), 64, 128, (uint32_t)g.Q, 64);
  if (rc) return rc;
  if (zero && !accumulate_prezeroed()) {
    cudaError_t e = cudaMemsetAsync(dw, 0, (size_t)(49 * Cin * 64) * sizeof(float), st);
    if (e != cudaSuccess) { set_error("stem7x7_wgrad: memset: %s", cudaGetErrorString(e)); return (int)e; }
  }
  const size_t smem = 1024 + (size_t)SWG_STAGES * g.stage_bytes + 256;
  cudaError_t e = cudaFuncSetAttribute(stem7x7_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { set_error("stem7x7_wgrad: cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e)); return (int)e; }
  const int grid = g.num_tiles < num_sms() ? g.num_tiles : num_sms();
  const int64_t dw_elems = 49 * Cin * 64;
  float* ws = nullptr;                                      // [grid][49 * Cin * 64] per-CTA partials
  rc = scratch_alloc(&ws, (size_t)grid * dw_elems * sizeof(float), st);
  if (rc) return rc;
  stem7x7_wgrad_kernel<<<grid, 160, smem, st>>>(tx, tdy, g, ws);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("stem7x7_wgrad: launch: %s", cudaGetErrorString(e)); scratch_free(ws, st); return (int)e; }
  rc = run_sum_partials(ws, dw_elems, dw, dw_elems, grid, st);
  const int rf = scratch_free(ws, st);
  return rc ? rc : rf;
}

}  // namespace tc
}  // namespace simclr
