// sm_90a building blocks for the tensor-core engine: mbarrier, TMA and wgmma
// wrappers (inline PTX), shared-memory descriptors, host-side tensor maps.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace simclr {
namespace tc {

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Spin on a phase parity.  A bounded spin turns a protocol bug into a trap (the launch fails with an
// error) instead of a hung GPU.  No function call (printf) may sit here: the consumers wait inside their
// wgmma pipelines, and a call there makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    if (ok) break;
    if ((++spins & 0xFF) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();     // 4 s: a protocol bug, not a long kernel
    }
  }
}
// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// fp32 pairs kept in one 64-bit register (the statistics loops' running sums)
__device__ __forceinline__ uint64_t f2_pack(float lo, float hi) {
  uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r;
}
__device__ __forceinline__ void f2_unpack(uint64_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1; f2_unpack(a, a0, a1); f2_unpack(b, b0, b1); return f2_pack(a0 + b0, a1 + b1);
}
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1; f2_unpack(a, a0, a1); f2_unpack(b, b0, b1); f2_unpack(c, c0, c1);
  return f2_pack(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

// im2col-mode load from an NHWC tensor (rank 4: {C, W, H, N}): `pixels-per-column` consecutive base
// pixels starting at (w, h, n) -- walking W, then H, then N inside the map's bounding box with its
// traversal stride -- each displaced by the filter offset (off_w, off_h); `channels-per-pixel`
// channels from c.  Pixels outside the image (padding, n >= N) read as zero.  The smem image is the
// same [pixel][128 B] 128B-swizzled tile a tiled 2-D box produces.
__device__ __forceinline__ void tma_load_im2col(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c, int w,
                                                int h, int n, int off_w, int off_h) {
  const uint16_t ow = (uint16_t)off_w, oh = (uint16_t)off_h;
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tmap), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(ow), "h"(oh)
      : "memory");
}

// smem tile -> global through the tensor map (rows/cols outside the tensor are clipped)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"((uint64_t)tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// smem tile added into global (fp32 add performed by the TMA unit at L2)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"((uint64_t)tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N> __device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------
// cp.async (LDGSTS): global -> shared without registers; src_bytes == 0 zero-fills
// ---------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------------------
// wgmma (sm_90a): D[registers of the issuing warpgroup] (+)= A[smem] * B[smem]
// ---------------------------------------------------------------------------
// A 128-row tile is two m64 halves; D of one half, m64nNk16 with fp32 accumulators, is N/2 registers per thread:
// d[4*i + v] holds row 16*(warp % 4) + lane/4 + 8*(v >> 1), column 8*i + 2*(lane % 4) + (v & 1).
template <int N, bool TF32, bool A_MN, bool B_MN> struct Wgmma;
template <> struct Wgmma<32, false, false, false> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<32, false, true, true> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<64, false, false, false> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<64, false, true, true> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<128, false, false, false> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<128, false, true, true> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<64, true, false, false> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

template <> struct Wgmma<128, true, false, false> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(acc));
  }
};

// D (+)= A * B for one m64 half; `acc` == 0 overwrites D (first K step of a tile)
template <int N, bool TF32, bool A_MN, bool B_MN>
__device__ __forceinline__ void wgmma(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  Wgmma<N, TF32, A_MN, B_MN>::mma(d, da, db, acc);
}
// orders register / shared-memory accesses of the warpgroup before the wgmmas that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups still in flight; the accumulators are named so that they are not read early
template <int N, int H, int R>
__device__ __forceinline__ void wgmma_wait(float (&d)[H][R]) {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
#pragma unroll
  for (int h = 0; h < H; ++h)
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[h][i])::"memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Row of the 128-row tile that accumulator registers 4*i + 2*rp (+1) of half h hold (rp: first or second row of
// the thread within its 16-row slice), for a warpgroup made of warps 0-3 of its own 128 threads.
__device__ __forceinline__ int frag_row(int h, int rp) {
  return 64 * h + 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * rp;
}

// ---------------------------------------------------------------------------
// Descriptors (sm_90 wgmma layout)
// ---------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128B swizzle.  K-major tiles: rows of 128 B,
// 8-row groups SBO bytes apart (LBO unused, encoded as 1).  MN-major tiles:
// 128-B rows along MN, 8-row (K) groups SBO apart, MN atoms LBO apart.
// Only the 14-bit start-address field (bytes >> 4) changes between the MMAs of a tile, so the issuing warpgroup
// keeps the low word as a running 32-bit value instead of rebuilding 64 bits from an address.
__host__ __device__ constexpr uint32_t desc_hi_sw128(uint32_t sbo_bytes) {
  return ((sbo_bytes >> 4) & 0x3FFFu) | (1u << 30);                 // layout type 1 (SWIZZLE_128B), bits 62-63
}
// no swizzle ("interleaved" 8-row x 16-byte core matrices)
__host__ __device__ constexpr uint32_t desc_hi_none(uint32_t sbo_bytes) { return (sbo_bytes >> 4) & 0x3FFFu; }
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo_bytes) {
  return ((saddr & 0x3FFFFu) >> 4) | (((lbo_bytes >> 4) & 0x3FFFu) << 16);
}
__device__ __forceinline__ uint64_t desc_pack(uint32_t lo, uint32_t hi) {
  uint64_t d; asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi)); return d;
}
// value of lane 0, provably warp-uniform for the compiler
__device__ __forceinline__ uint32_t uniform_u32(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }

// byte offset of 16-byte chunk j of row r inside a [rows][128 B] SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) {
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// Accumulator columns [8*i0, 8*i0 + 128 / sizeof(To)) of a 128-row tile (both halves) -> [128 rows][128 B]
// 128B-swizzled staging tile at shared address `tile`, converted to To; rows with ok[h][rp] false are stored as zeros.
template <typename To, int NF>
__device__ __forceinline__ void stage_frag(uint32_t tile, const float (&acc)[2][NF], int i0, const bool (&ok)[2][2]) {
  constexpr int NI = 128 / (int)sizeof(To) / 8;      // 8-column groups per 128-byte row
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int rp = 0; rp < 2; ++rp) {
      const int row = frag_row(h, rp);
#pragma unroll
      for (int ii = 0; ii < NI; ++ii) {
        float a = acc[h][4 * (i0 + ii) + 2 * rp], b = acc[h][4 * (i0 + ii) + 2 * rp + 1];
        if (!ok[h][rp]) { a = 0.f; b = 0.f; }
        if (sizeof(To) == 2) {
          __nv_bfloat162 hh = __floats2bfloat162_rn(a, b);
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(tile + sw128_offset(row, ii) + 4 * q), "r"(*reinterpret_cast<uint32_t*>(&hh)) : "memory");
        } else {
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(tile + sw128_offset(row, 2 * ii + (q >> 1)) + 8 * (q & 1)), "f"(a), "f"(b) : "memory");
        }
      }
    }
}
// the 32 fp32 values of `row` from a [128 rows][128 B] 128B-swizzled staging tile
__device__ __forceinline__ void load_row32(const uint8_t* tile, int row, uint32_t* r) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint4 v = *reinterpret_cast<const uint4*>(tile + sw128_offset(row, j));
    r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
  }
}

// Division by a runtime constant (CUTLASS FastDivmod scheme; n < 2^31).
struct FastDiv {
  uint32_t d, m, s;
  __host__ FastDiv() : d(1), m(0), s(0) {}
  __host__ explicit FastDiv(uint32_t div) : d(div), m(0), s(0) {
    if (div != 1) {
      uint32_t lg = 31 - __builtin_clz(div);
      if (div & (div - 1)) lg += 1;
      const uint32_t p = 31 + lg;
      m = (uint32_t)(((1ull << p) + div - 1) / div);
      s = p - 32;
    }
  }
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return d == 1 ? n : (__umulhi(n, m) >> s); }
  __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const { q = div(n); r = n - q * d; }
};

// ---------------------------------------------------------------------------
// Host: tensor maps through the driver entry point (no libcuda link dependency)
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D row-major matrix [rows][cols] of `elt_bytes` elements, box [box_rows][box_cols], 128B swizzle,
// out-of-bounds elements read as zero.
inline int make_tmap_2d(CUtensorMap* map, const void* base, int elt_bytes, uint64_t rows, uint64_t cols,
                        uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_tiled();
  if (!fn) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return SIMCLR_ERR_DRIVER; }
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {row_stride_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = elt_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUresult r = fn(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): base=%p rows=%llu cols=%llu stride=%llu box=%ux%u", (int)r, base,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)row_stride_bytes, box_rows, box_cols);
    return SIMCLR_ERR_DRIVER;
  }
  return SIMCLR_OK;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

inline EncodeIm2colFn get_encode_im2col() {
  static EncodeIm2colFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeIm2colFn)p;
  }
  return fn;
}

// im2col map over an NHWC tensor: base pixels lo .. (W-1)+up (same corners for H and W: square
// filters with symmetric padding only), visited with `trav` (the conv stride); boxes of `pixels`
// pixels x 128 bytes of channels, 128B swizzle.
inline int make_tmap_im2col(CUtensorMap* map, const void* base, int elt_bytes, uint64_t N, uint64_t H, uint64_t W,
                            uint64_t C, int lo, int up, uint32_t trav, uint32_t pixels) {
  EncodeIm2colFn fn = get_encode_im2col();
  if (!fn) { set_error("cuTensorMapEncodeIm2col unavailable (no CUDA driver?)"); return SIMCLR_ERR_DRIVER; }
  const cuuint64_t dims[4] = {C, W, H, N};
  const cuuint64_t strides[3] = {C * elt_bytes, W * C * elt_bytes, H * W * C * elt_bytes};
  const int lower[2] = {lo, lo}, upper[2] = {up, up};
  const cuuint32_t estr[4] = {1, trav, trav, 1};
  const CUtensorMapDataType dt = elt_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUresult r = fn(map, dt, 4, const_cast<void*>(base), dims, strides, lower, upper, (cuuint32_t)(128 / elt_bytes),
                        pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (%d): base=%p N=%llu H=%llu W=%llu C=%llu corners=%d/%d stride=%u pixels=%u",
              (int)r, base, (unsigned long long)N, (unsigned long long)H, (unsigned long long)W, (unsigned long long)C,
              lo, up, trav, pixels);
    return SIMCLR_ERR_DRIVER;
  }
  return SIMCLR_OK;
}

// 7x7 stride-2 stem fprop from a slab of 16-byte pixel pairs, no im2col copy (tc_stem.cu)
bool stem7x7_applicable(int dtype, int out_dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t n_out, int64_t R,
                        int64_t S, int64_t stride, int64_t P, int64_t Q, const void* src, const void* wk, const void* out);
int run_stem7x7(const void* src, const void* wk, void* out, int64_t N, int64_t H, int64_t W, int64_t n_out, cudaStream_t st,
                double* bn_sums);
bool stem7x7_wgrad_applicable(int dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                              int64_t S, int64_t stride, const void* x, const void* dy, const void* dw);
int run_stem7x7_wgrad(const void* x, const void* dy, float* dw, int64_t N, int64_t H, int64_t W, int64_t Cin, cudaStream_t st,
                      bool zero);
// 3x3 stride-1 fprop / dgrad with halo reuse (tc_halo.cu); see run_halo3x3 for the argument meaning
bool halo3x3_applicable(int dtype, int out_dtype, int64_t N, int64_t H, int64_t W, int64_t C, int64_t n_out, int64_t R,
                        int64_t S, int64_t stride, const void* src, const void* wk, const void* out);
int run_halo3x3(int mode, const void* src, const void* wk, void* out, int64_t N, int64_t H, int64_t W, int64_t C,
                int64_t n_out, cudaStream_t st, double* bn_sums);
// wgrad of the 64 -> 64 channel 3x3 stride-1 layers with halo reuse (tc_halo.cu)
bool halo3x3_wgrad_applicable(int dtype, int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                              int64_t S, int64_t stride, const void* x, const void* dy, const void* dw);
int run_halo3x3_wgrad(const void* x, const void* dy, float* dw, int64_t N, int64_t H, int64_t W, cudaStream_t st, bool zero);

}  // namespace tc
}  // namespace simclr
