// PTX wrappers for the Hopper (sm_90a) tensor-core kernels: mbarrier, cp.async / cp.async.bulk / TMA, wgmma and its shared-memory
// matrix descriptor (bit layout: PTX ISA, "Matrix Descriptor Format" of the asynchronous warpgroup-level MMA).
#pragma once
#include "common.cuh"

namespace cmgan_tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 28)) __trap();        // protocol bug: fail loudly instead of hanging the device
    }
}
// one non-blocking probe: true when the phase with this parity has completed
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// TMA tiled load of a 2-D box (coordinates: c0 = innermost) into shared memory; completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const void* tmap, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const void* tmap, int c0, int c1, int c2, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst_smem, const void* tmap, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst_smem, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// wgmma (sm_90a warpgroup MMA).  Shared-memory matrix descriptor for a K-major SWIZZLE_128B operand (rows = M/N index, 128 B = 32 tf32
// along K, 8-row groups 1024 B apart; the tile must start on a 1024-byte boundary): leading byte offset unused (1), stride byte offset 1024.
// Advancing K by 8 tf32 (one instruction) = +32 bytes = +2 in the address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);            // start address >> 4         bits [0,14)
    d |= (uint64_t)1 << 16;                             // leading byte offset >> 4   bits [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;                   // stride byte offset >> 4    bits [32,46)
    d |= (uint64_t)1 << 62;                             // layout type 1 = SWIZZLE_128B
    return d;
}
// warpgroup register re-allocation (sm_90a): every warp of the warpgroup executes it.  dec hands registers back to the CTA's pool, inc
// waits until the pool has them.  The kernel's entry count (launch bounds) and every split must keep the CTA within the 64 K registers.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 16] (+)= A[64 x 8] B[16 x 8]^T, tf32 operands from shared memory, fp32 accumulators in registers.  Fragment of warp w of the
// warpgroup, lane l: d[4 i + 0 / 1] = row 16 w + l / 4, columns 8 i + 2 (l % 4) + 0 / 1;  d[4 i + 2 / 3] = the same columns 8 rows further.
__device__ __forceinline__ void wgmma_m64n16k8_tf32(float d[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 8] B[64 x 8]^T: the fragment of d[b] (b = 0..3) is that of the m64n16k8 instruction on columns 16 b .. 16 b + 15
#define CMGAN_D8(b) "+f"(d[b][0]), "+f"(d[b][1]), "+f"(d[b][2]), "+f"(d[b][3]), "+f"(d[b][4]), "+f"(d[b][5]), "+f"(d[b][6]), "+f"(d[b][7])
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[4][8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                 : CMGAN_D8(0), CMGAN_D8(1), CMGAN_D8(2), CMGAN_D8(3)
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// the same with A from registers: a[0..3] = tf32 elements (row 16 w + l / 4, column l % 4), (row + 8, column), (row, column + 4),
// (row + 8, column + 4) of warp w's 16 x 8 slice of A.  They must not be overwritten until a wgmma_wait covers this instruction.
__device__ __forceinline__ void wgmma_m64n64k8_tf32_rs(float (&d)[4][8], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
                 : CMGAN_D8(0), CMGAN_D8(1), CMGAN_D8(2), CMGAN_D8(3)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
#undef CMGAN_D8

// D[64 x 16 W] (+)= A[64 x 8] B[16 W x 8]^T on the accumulator blocks d[0] .. d[W - 1] (W = 4, 8, 12, 16): one wgmma m64n(16 W)k8,
// whose fragment is the W m64n16k8 fragments side by side.  The A slice is read once for the whole width instead of once per 16 columns.
#define CMGAN_DJ(b) "+f"(d[b][0]), "+f"(d[b][1]), "+f"(d[b][2]), "+f"(d[b][3]), "+f"(d[b][4]), "+f"(d[b][5]), "+f"(d[b][6]), "+f"(d[b][7])
template <int W, int NBMAX>
__device__ __forceinline__ void wgmma_tf32_blocks(float (&d)[NBMAX][8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    static_assert(W <= NBMAX, "accumulator blocks out of range");
    if constexpr (W == 4) {
        wgmma_m64n64k8_tf32(*reinterpret_cast<float(*)[4][8]>(&d[0]), adesc, bdesc, accumulate);
    } else if constexpr (W == 8) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
                     "}, %64, %65, p, 1, 1;\n\t}"
                     : CMGAN_DJ(0), CMGAN_DJ(1), CMGAN_DJ(2), CMGAN_DJ(3),
                       CMGAN_DJ(4), CMGAN_DJ(5), CMGAN_DJ(6), CMGAN_DJ(7)
                     : "l"(adesc), "l"(bdesc), "r"(accumulate));
    } else if constexpr (W == 12) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {"
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                     "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
                     "}, %96, %97, p, 1, 1;\n\t}"
                     : CMGAN_DJ(0), CMGAN_DJ(1), CMGAN_DJ(2), CMGAN_DJ(3),
                       CMGAN_DJ(4), CMGAN_DJ(5), CMGAN_DJ(6), CMGAN_DJ(7),
                       CMGAN_DJ(8), CMGAN_DJ(9), CMGAN_DJ(10), CMGAN_DJ(11)
                     : "l"(adesc), "l"(bdesc), "r"(accumulate));
    } else if constexpr (W == 16) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                     "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
                     "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
                     "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
                     "}, %128, %129, p, 1, 1;\n\t}"
                     : CMGAN_DJ(0), CMGAN_DJ(1), CMGAN_DJ(2), CMGAN_DJ(3),
                       CMGAN_DJ(4), CMGAN_DJ(5), CMGAN_DJ(6), CMGAN_DJ(7),
                       CMGAN_DJ(8), CMGAN_DJ(9), CMGAN_DJ(10), CMGAN_DJ(11),
                       CMGAN_DJ(12), CMGAN_DJ(13), CMGAN_DJ(14), CMGAN_DJ(15)
                     : "l"(adesc), "l"(bdesc), "r"(accumulate));
    } else {
        static_assert(W == 4, "no wgmma wrapper for this width");
    }
}
#undef CMGAN_DJ

// one 32-float K chunk (4 K steps of 8) of a 64 x (16 NB) accumulator, both operands K-major SWIZZLE_128B (16 B rows = 2048 bytes =
// 128 descriptor units): one wgmma m64n(16 NB)k8 per K step, NB = 4, 8, 12 or 16.
template <int NB, int NBMAX>
__device__ __forceinline__ void mma_chunk(float (&acc)[NBMAX][8], uint64_t adesc, uint64_t bdesc, bool first) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
        wgmma_tf32_blocks<NB, NBMAX>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (first && k == 0) ? 0u : 1u);
}

}  // namespace cmgan_tc
