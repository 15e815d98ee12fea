// Hopper wgmma / mbarrier PTX wrappers shared by the tensor-core kernels (gemm.cu, det_head.cu); sm_90a only.
#pragma once

#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace bevf {

// ---- PTX wrappers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the accumulator reads of the epilogue after wgmma.wait_group
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (wgmma), SWIZZLE_128B.
//   K-major operand: rows of 128 B (64 bf16 along K), 8-row groups 1024 B apart (SBO); LBO unused.
//   MN-major operand: 64 MN-contiguous elements (128 B) per K row, 8-K-row groups 1024 B apart (SBO), the next
//   64-element MN chunk `chunk_bytes` further (LBO).
// Bits: start address >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), layout type [62,64) = 1 (128 B swizzle).
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// D[64 x N] (+)= A[64 x 16] . B[16 x N], TE (bf16 | fp16) in, fp32 accumulate in registers; kTA / kTB: operand MN-major.
// Accumulator layout (per warp w of the warpgroup, lane l): d[4j + 2h + e] = D[16 w + 8 h + l / 4][8 j + 2 (l % 4) + e].
template <int N, int kTA, int kTB, typename TE> struct Wgmma;
#define BEVF_WGMMA_N16(TY) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {" \
                     "%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n" \
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]) \
                     : "l"(da), "l"(db), "r"((int)accumulate), "n"(kTA), "n"(kTB))
template <int kTA, int kTB, typename TE> struct Wgmma<16, kTA, kTB, TE> {
    __device__ static __forceinline__ void run(float (&d)[8], uint64_t da, uint64_t db, bool accumulate) {
        if constexpr (std::is_same<TE, __half>::value) BEVF_WGMMA_N16("f16");
        else BEVF_WGMMA_N16("bf16");
    }
};
#undef BEVF_WGMMA_N16
#define BEVF_WGMMA_N64(TY) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {" \
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31" \
                     "}, %32, %33, p, 1, 1, %35, %36;\n}\n" \
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                     "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                     "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                     "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
                     : "l"(da), "l"(db), "r"((int)accumulate), "n"(kTA), "n"(kTB))
template <int kTA, int kTB, typename TE> struct Wgmma<64, kTA, kTB, TE> {
    __device__ static __forceinline__ void run(float (&d)[32], uint64_t da, uint64_t db, bool accumulate) {
        if constexpr (std::is_same<TE, __half>::value) BEVF_WGMMA_N64("f16");
        else BEVF_WGMMA_N64("bf16");
    }
};
#undef BEVF_WGMMA_N64
#define BEVF_WGMMA_N128(TY) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {" \
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63" \
                     "}, %64, %65, p, 1, 1, %67, %68;\n}\n" \
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                     "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                     "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                     "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                     "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                     "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                     "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                     "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
                     : "l"(da), "l"(db), "r"((int)accumulate), "n"(kTA), "n"(kTB))
template <int kTA, int kTB, typename TE> struct Wgmma<128, kTA, kTB, TE> {
    __device__ static __forceinline__ void run(float (&d)[64], uint64_t da, uint64_t db, bool accumulate) {
        if constexpr (std::is_same<TE, __half>::value) BEVF_WGMMA_N128("f16");
        else BEVF_WGMMA_N128("bf16");
    }
};
#undef BEVF_WGMMA_N128
#define BEVF_WGMMA_N256(TY) asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {" \
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
                     "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
                     "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
                     "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127" \
                     "}, %128, %129, p, 1, 1, %131, %132;\n}\n" \
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
                     "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
                     "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
                     "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
                     "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
                     "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
                     "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
                     "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
                     "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
                     "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
                     "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
                     "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
                     "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
                     "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
                     "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
                     "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
                     : "l"(da), "l"(db), "r"((int)accumulate), "n"(kTA), "n"(kTB))
template <int kTA, int kTB, typename TE> struct Wgmma<256, kTA, kTB, TE> {
    __device__ static __forceinline__ void run(float (&d)[128], uint64_t da, uint64_t db, bool accumulate) {
        if constexpr (std::is_same<TE, __half>::value) BEVF_WGMMA_N256("f16");
        else BEVF_WGMMA_N256("bf16");
    }
};
#undef BEVF_WGMMA_N256

}  // namespace bevf
