// Dense projections of the encoder layer on the Hopper tensor cores (sm_90a: TMA + mbarrier + wgmma).
//
//   forward  Y[M, N]  = act( X[M, K] . W[N, K]^T + bias[N] ) (+ addend[M, N])      bf16 in, fp32 accumulate
//   dgrad    dX[M, K] = dY[M, N] . W[N, K] (+ addend[M, K])                          (W read in place)
//   wgrad    dW[N, K] = dY[M, N]^T . X[M, K],  db[N] = column sums of dY             (split over the M rows)
//
// replaces the cuBLAS GEMM + separate bias/ReLU/residual kernels behind every nn.Linear of
// TemporalSelfAttention / MSDeformableAttention3D / SpatialCrossAttention / mmcv FFN
// (temporal_self_attention.py:198,206-209,267; spatial_cross_attention.py:173,334,338-341;
// custom_base_transformer_layer.py:157-158).
//
// Operands differ only in which is MN-major in shared memory (the non-reduced index contiguous, i.e. the tensor
// read in its natural row-major layout without a transpose).  Forward and dgrad run on the weight-stationary
// kernel gemm_ws_wgmma further down (the weight tile of a column block stays in shared memory; ping-pong consumer
// warpgroups; TMA-store epilogue).  The weight gradient, and forward / dgrad with a reduction too long for the
// weight tile to fit (> 1024), run on gemm_bf16_wgmma: persistent CTAs of three warpgroups walking a flat list
// of (128 x BN output tile, reduction split) units:
//   warpgroup 0, warp 0   TMA producer: cp.async.bulk.tensor loads of the A (128 x 64) and B (BN x 64) k-blocks
//                          into a ring of SWIZZLE_128B shared-memory stages, completion on mbarriers
//   warpgroup 0, warp 1   weight gradient only: column sums of the dY tiles straight from the same stages (db)
//   warpgroups 1 and 2    rows 0-63 / 64-127 of the tile: wgmma.mma_async m64nBNk16 from the two shared-memory
//                          descriptors into fp32 registers; a stage is released (mbarrier) once its wgmma group
//                          has retired, so the producer runs up to `stages` k-blocks ahead -- across tiles too,
//                          i.e. the loads of tile i+1 overlap the epilogue of tile i.
//   epilogue               straight from the accumulator registers: bias, ReLU, addend, convert, store (or fp32
//                          reduction / per-split slab for the weight gradient).
// These GEMMs have K = 256 or 512 only: they are bound by streaming X / Y through HBM.
#include <cuda.h>

#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "common.cuh"

namespace bevf {

constexpr int kBM = 128;                 // rows per tile: two consumer warpgroups x m64
constexpr int kBK = 64;                  // bf16 elements per k-block row == 128 B == one swizzle atom
constexpr int kGemmThreads = 384;        // producer warpgroup + two consumer warpgroups
constexpr int kChunk = 64 * 128;         // one 64 x 64 bf16 box (MN-major operands come in these)
constexpr int kMaxStages = 6;

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

// bias[col] as fp32 from an f32 / bf16 / fp16 vector (dt: BEVF_DTYPE_*)
__device__ __forceinline__ float load_bias(const void *bias, int dt, int col) {
    if (dt == BEVF_DTYPE_BF16) return __bfloat162float(reinterpret_cast<const bf16 *>(bias)[col]);
    if (dt == BEVF_DTYPE_F16) return __half2float(reinterpret_cast<const __half *>(bias)[col]);
    return reinterpret_cast<const float *>(bias)[col];
}

struct GemmParams {
    int M, N;              // product rows / columns
    int R;                 // reduction length
    int rows_per_split;    // reduction rows per unit (multiple of 64)
    int splits;
    int stages;            // shared-memory ring depth
    int relu;
    const void *bias;      // (N) f32 or the operand type, or null
    int bias_dt;           // BEVF_DTYPE_* of bias
    const void *addend;    // (M, N) in the operand type, added after the activation, or null
    void *y;               // output, row stride ldy
    int64_t ldy;
    int64_t split_stride;  // elements between the output slabs of successive splits (two-pass weight gradient)
    int out_f32;
    int red;               // 1: fp32 reduction into y instead of a store
    float *db;             // weight gradient: column sums of dY reduced into db (N_dY = M floats), or null
    float *db_ws;          // two-pass weight gradient: (splits, n_pad) slabs of column sums, or null
    int n_pad;
};

template <int BN, bool kAmn, bool kBmn, typename TE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                const GemmParams p) {
    static_assert(BN == 64 || BN == 128, "tile width");
    constexpr int kABytes = kBM * 128, kStageBytes = kABytes + BN * 128;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)p.stages * kStageBytes);
    uint64_t *empty = full + p.stages;

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_m = (p.M + kBM - 1) / kBM, tiles_n = (p.N + BN - 1) / BN;
    const int units = tiles_m * tiles_n * p.splits;
    const bool colsum = p.db != nullptr || p.db_ws != nullptr;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        // a stage is released by the 8 consumer warps and, when the bias gradient is wanted, by warp 1
        for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], colsum ? 9 : 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // unit -> (row tile, column tile, split of the reduction rows); splits fastest, then columns
    auto decode = [&](int u, int &tm, int &tn, int &split, int &r0, int &kblocks) {
        split = u % p.splits;
        const int tile = u / p.splits;
        tm = tile / tiles_n; tn = tile - tm * tiles_n;
        r0 = split * p.rows_per_split;
        const int r1 = min(p.R, r0 + p.rows_per_split);
        kblocks = r1 > r0 ? (r1 - r0 + kBK - 1) / kBK : 0;
    };

    if (wg == 0) {
        if (warp == 0) {
            // ===================== TMA producer =====================
            if (lane == 0) {
                int s = 0; uint32_t ph = 0;
                for (int u = blockIdx.x; u < units; u += gridDim.x) {
                    int tm, tn, split, r0, kblocks;
                    decode(u, tm, tn, split, r0, kblocks);
                    for (int kb = 0; kb < kblocks; ++kb) {
                        mbar_wait(&empty[s], ph ^ 1);
                        uint8_t *sa = smem + (size_t)s * kStageBytes, *sb = sa + kABytes;
                        mbar_expect_tx(&full[s], (uint32_t)kStageBytes);
                        const int rr = r0 + kb * kBK;
                        if (!kAmn) {
                            tma_load_2d(sa, &map_a, &full[s], rr, tm * kBM);
                        } else {                     // 64 reduction rows x 128 MN columns as two 8 KB chunks
                            tma_load_2d(sa, &map_a, &full[s], tm * kBM, rr);
                            tma_load_2d(sa + kChunk, &map_a, &full[s], tm * kBM + 64, rr);
                        }
                        if (!kBmn) {
                            tma_load_2d(sb, &map_b, &full[s], rr, tn * BN);
                        } else {
#pragma unroll
                            for (int c = 0; c < BN / 64; ++c)
                                tma_load_2d(sb + c * kChunk, &map_b, &full[s], tn * BN + c * 64, rr);
                        }
                        if (++s == p.stages) { s = 0; ph ^= 1; }
                    }
                }
            }
        } else if (warp == 1 && colsum) {
            // ===================== bias gradient: column sums of the dY tiles (MN-major A) ==============
            // lane = (16 B unit j = lane % 8 of a 64-column chunk, row group lane / 8); the tile is stored
            // with the 128 B swizzle: unit j of reduction row r sits at position j ^ (r & 7).
            int s = 0; uint32_t ph = 0;
            const int j = lane & 7, rg = lane >> 3;
            for (int u = blockIdx.x; u < units; u += gridDim.x) {
                int tm, tn, split, r0, kblocks;
                decode(u, tm, tn, split, r0, kblocks);
                float acc[2][8];
#pragma unroll
                for (int c = 0; c < 2; ++c)
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[c][e] = 0.f;
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(&full[s], ph);
                    if (tn == 0) {                                // count every dY element once
                        const uint8_t *sa = smem + (size_t)s * kStageBytes;
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
#pragma unroll 4
                            for (int r = rg; r < 64; r += 4) {
                                const uint4 v = *reinterpret_cast<const uint4 *>(sa + c * kChunk + r * 128 + ((j ^ (r & 7)) << 4));
                                const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                                for (int e = 0; e < 4; ++e) { acc[c][2 * e] += St16<TE>::lo(w4[e]); acc[c][2 * e + 1] += St16<TE>::hi(w4[e]); }
                            }
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[s]);
                    if (++s == p.stages) { s = 0; ph ^= 1; }
                }
                if (tn == 0 && kblocks > 0) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            float t = acc[c][e];
                            t += __shfl_xor_sync(0xffffffffu, t, 8);
                            t += __shfl_xor_sync(0xffffffffu, t, 16);
                            acc[c][e] = t;
                        }
                        const int col = tm * kBM + c * 64 + j * 8;
                        if (rg == 0) {
                            if (p.db_ws) {
                                float *dst = p.db_ws + (size_t)split * p.n_pad + col;
                                *reinterpret_cast<float4 *>(dst) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
                                *reinterpret_cast<float4 *>(dst + 4) = make_float4(acc[c][4], acc[c][5], acc[c][6], acc[c][7]);
                            } else if (col < p.M) {
                                red_add_v4(p.db + col, acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
                                red_add_v4(p.db + col + 4, acc[c][4], acc[c][5], acc[c][6], acc[c][7]);
                            }
                        }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cw owns rows 64 cw .. 64 cw + 63 of the tile ==============
    const int cw = wg - 1, w4 = warp & 3;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int tm, tn, split, r0, kblocks;
        decode(u, tm, tn, split, r0, kblocks);
        if (kblocks == 0) continue;
        for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&full[s], ph);
            __syncwarp();
            const uint32_t sa = smem_u32(smem + (size_t)s * kStageBytes), sb = sa + kABytes;
            // K-major A: this warpgroup's 64 rows start 64 x 128 B in; MN-major A: its 64 columns are chunk cw.
            // One k16 step: K-major +32 B (inside the swizzle atom), MN-major +16 rows = 2048 B.
            const uint64_t da = smem_desc_sw128(sa + (uint32_t)(cw * 8192), kChunk);
            const uint64_t db = smem_desc_sw128(sb, kChunk);
            constexpr uint64_t da_step = kAmn ? 128 : 2, db_step = kBmn ? 128 : 2;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k)
                Wgmma<BN, kAmn, kBmn, TE>::run(acc, da + da_step * k, db + db_step * k, (kb | k) != 0);
            wgmma_commit();
            wgmma_wait0();
            fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
            if (++s == p.stages) { s = 0; ph ^= 1; }
        }
        // ---- epilogue from the registers: rows row_a (h = 0) and row_a + 8 (h = 1), columns col .. col + 1
        const int row_a = tm * kBM + cw * 64 + w4 * 16 + (lane >> 2);
        const int col0 = tn * BN + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = col0 + 8 * j;
            if (col >= p.N) continue;
            float b0 = 0.f, b1 = 0.f;
            if (p.bias) { b0 = load_bias(p.bias, p.bias_dt, col); b1 = load_bias(p.bias, p.bias_dt, col + 1); }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row_a + 8 * h;
                if (row >= p.M) continue;
                float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
                if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (p.addend) {
                    const uint32_t a2 = __ldg(reinterpret_cast<const unsigned int *>(
                        reinterpret_cast<const TE *>(p.addend) + (size_t)row * p.N + col));
                    v0 += St16<TE>::lo(a2); v1 += St16<TE>::hi(a2);
                }
                const size_t off = (size_t)split * p.split_stride + (size_t)row * p.ldy + col;
                if (p.red) {
                    float *dst = reinterpret_cast<float *>(p.y) + off;
                    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
                } else if (p.out_f32) {
                    *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.y) + off) = make_float2(v0, v1);
                } else {
                    *reinterpret_cast<uint32_t *>(reinterpret_cast<TE *>(p.y) + off) = St16<TE>::pack(v0, v1);
                }
            }
        }
    }
}

// ================================================================================================
// Weight-stationary forward / dgrad:  Y[M, N] = act( A[M, R] . B + bias ) (+ addend),  A K-major,
// B = the weight, K-major (forward, W[N, R]) or MN-major (dgrad, W[R, N] read in place).
//
// CTA b owns column block b % tiles_n for its whole life and a contiguous range of 64-row tiles; the CTAs
// of one column block split the rows evenly, and CTA g * tiles_n + j (j = 0 .. tiles_n - 1) walk the same
// rows in step, so an activation row read from HBM by one column block is an L2 hit for the others.
//   warp 0 / warp 1 (lane 0)  TMA producers of consumer warpgroup 1 / 2: the BN x R weight tile once (warp 0),
//                             then the 64 x 64 A k-blocks of that warpgroup's tiles through its own ring, and
//                             the tile's addend (bf16, 64 x BN) into its staging buffer
//   warpgroups 1 and 2        ping-pong: each owns every other row tile of the range whole (m64nBNk16 wgmmas
//                             against the resident weight, one group in flight behind the one being issued),
//                             so one warpgroup's epilogue runs while the other issues its wgmmas
//   epilogue                  bias, ReLU, addend (from the staging buffer) in registers, convert, write into
//                             the SWIZZLE_128B staging buffer, cp.async.bulk.tensor store; rows past M and
//                             columns past N are clipped by the tensor map
// Shared memory (227 KB): weight BN x R x 2 (<= 128 KB) + 2 x staging (64 rows x min(BN x out bytes, 512 B))
// + 2 x ring (stages x 8 KB), the ring taking what is left (at most kMaxStages):
//   BN 256, R 256: 128 + 2 x 32 + 2 x 2 x 8 KB     BN 128, R 512: 128 + 2 x 16 (bf16) / 32 (fp32) + 2 x 4 / 2 x 8 KB
//   BN 256, R 192:  96 + 2 x 32 + 2 x 4 x 8 KB     BN  64, R 768:  96 + 2 x 8 + 2 x 6 x 8 KB
// ================================================================================================
constexpr int kWsRows = 64;               // rows per tile: one consumer warpgroup, m64
constexpr int kWsBoxBytes = 64 * 128;     // one 64-row x 128 B TMA box (A k-block, addend/output box)
constexpr int kWsStageMax = 4 * kWsBoxBytes;
constexpr int kWsWeightMax = 128 * 1024;

struct WsParams {
    int M, N, R;           // output rows / columns, reduction length (multiple of 64)
    int tiles_m, tiles_n, groups;
    int stages;            // A ring depth per consumer warpgroup
    int stg_bytes;         // staging buffer per consumer warpgroup
    int relu;
    const void *bias;      // (N) f32 or the operand type, or null
    int bias_dt;           // BEVF_DTYPE_* of bias
    int addend;            // 1: (M, N) addend in the operand type (map_add) added after the activation
    int out_f32;
};

__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}

template <int BN, bool kBmn, typename TE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_ws_wgmma(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
              const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_add,
              const WsParams p) {
    static_assert(BN == 64 || BN == 128 || BN == 256, "tile width");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int kblocks = p.R / kBK;
    const int w_bytes = kblocks * BN * 128;
    uint8_t *sw = smem;
    uint8_t *stg0 = sw + w_bytes;
    uint8_t *ring0 = stg0 + 2 * p.stg_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(ring0 + 2 * p.stages * kWsBoxBytes);
    uint64_t *w_full = bars;
    uint64_t *full = bars + 1, *empty = full + 2 * kMaxStages;          // [warpgroup][stage]
    uint64_t *add_full = empty + 2 * kMaxStages, *stg_empty = add_full + 2;
    float *sbias = reinterpret_cast<float *>(stg_empty + 2);

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tn = blockIdx.x % p.tiles_n, g = blockIdx.x / p.tiles_n;
    const int t_begin = (int)((int64_t)g * p.tiles_m / p.groups);
    const int t_end = (int)((int64_t)(g + 1) * p.tiles_m / p.groups);
    const int col0 = tn * BN;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_y) : "memory");
        mbar_init(w_full, 1);
        for (int i = 0; i < 2 * kMaxStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
        for (int i = 0; i < 2; ++i) { mbar_init(&add_full[i], 1); mbar_init(&stg_empty[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        // ===================== TMA producers: warp c feeds consumer warpgroup c ==================
        if (warp < 2 && lane == 0) {
            const int c = warp;
            if (c == 0) {
                // columns of the block past N are not loaded (MN-major) or read as zeros (K-major); either way
                // they only reach output columns the store clips
                const int chunks = kBmn ? min(BN / 64, (p.N - col0 + 63) / 64) : 1;
                mbar_expect_tx(w_full, (uint32_t)(kblocks * (kBmn ? chunks * kChunk : BN * 128)));
                for (int kb = 0; kb < kblocks; ++kb) {
                    uint8_t *dst = sw + (size_t)kb * BN * 128;
                    if (!kBmn) {
                        tma_load_2d(dst, &map_w, w_full, kb * kBK, col0);
                    } else {
                        for (int ch = 0; ch < chunks; ++ch)
                            tma_load_2d(dst + ch * kChunk, &map_w, w_full, col0 + ch * 64, kb * kBK);
                    }
                }
            }
            uint8_t *ring = ring0 + (size_t)c * p.stages * kWsBoxBytes, *stg = stg0 + (size_t)c * p.stg_bytes;
            uint64_t *f = full + c * kMaxStages, *e = empty + c * kMaxStages;
            const int add_boxes = min(BN / 64, (p.N - col0 + 63) / 64);
            int s = 0; uint32_t ph = 0, t = 0;
            for (int tm = t_begin + c; tm < t_end; tm += 2, ++t) {
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(&e[s], ph ^ 1);
                    mbar_expect_tx(&f[s], (uint32_t)kWsBoxBytes);
                    tma_load_2d(ring + (size_t)s * kWsBoxBytes, &map_a, &f[s], kb * kBK, tm * kWsRows);
                    if (++s == p.stages) { s = 0; ph ^= 1; }
                }
                if (p.addend) {
                    if (t > 0) mbar_wait(&stg_empty[c], (t - 1) & 1);
                    mbar_expect_tx(&add_full[c], (uint32_t)(add_boxes * kWsBoxBytes));
                    for (int b = 0; b < add_boxes; ++b)
                        tma_load_2d(stg + b * kWsBoxBytes, &map_add, &add_full[c], col0 + b * 64, tm * kWsRows);
                }
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");

    // ===================== consumers: warpgroup cw owns row tiles t_begin + cw, t_begin + cw + 2, ... =========
    const int cw = wg - 1, w4 = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    uint8_t *ring = ring0 + (size_t)cw * p.stages * kWsBoxBytes, *stg = stg0 + (size_t)cw * p.stg_bytes;
    uint64_t *f = full + cw * kMaxStages, *e = empty + cw * kMaxStages;
    // fp32 output of a 256-wide block goes out in two staging fills of 128 columns
    constexpr int kF32PassCols = BN > 128 ? 128 : BN;
    const int passes = p.out_f32 ? BN / kF32PassCols : 1;
    const uint32_t sw_base = smem_u32(sw);
    constexpr uint64_t db_step = kBmn ? 128 : 2;
    float acc[BN / 2];
    // the block's bias as fp32 (zeros past N or without a bias), read from shared memory by the epilogue
    for (int i = threadIdx.x - 128; i < BN; i += 256) {
        const int col = col0 + i;
        float b = 0.f;
        if (p.bias && col < p.N) b = load_bias(p.bias, p.bias_dt, col);
        sbias[i] = b;
    }
    asm volatile("bar.sync 3, 256;" ::: "memory");
    mbar_wait(w_full, 0);
    int s = 0; uint32_t ph = 0, t = 0;
    for (int tm = t_begin + cw; tm < t_end; tm += 2, ++t) {
        int prev = -1;
        for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&f[s], ph);
            const uint64_t da = smem_desc_sw128(smem_u32(ring + (size_t)s * kWsBoxBytes), 0);
            const uint64_t db = smem_desc_sw128(sw_base + (uint32_t)(kb * BN * 128), kChunk);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k)
                Wgmma<BN, 0, kBmn, TE>::run(acc, da + 2 * k, db + db_step * k, (kb | k) != 0);
            wgmma_commit();
            if (prev >= 0) {
                // the group of k-block kb - 1 has retired: its A stage can be refilled
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(&e[prev]);
            }
            prev = s;
            if (++s == p.stages) { s = 0; ph ^= 1; }
        }
        wgmma_wait0();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&e[prev]);

        // ---- epilogue: thread holds rows r0 (h = 0) and r0 + 8 (h = 1), columns 8 j + cq, 8 j + cq + 1
        const int r0 = w4 * 16 + (lane >> 2), cq = 2 * (lane & 3);
        if (p.addend) mbar_wait(&add_full[cw], t & 1);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const float2 bv = *reinterpret_cast<const float2 *>(sbias + 8 * j + cq);
            const float b0 = bv.x, b1 = bv.y;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
                if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (p.addend) {
                    // 16-bit box j / 8, 16 B unit j % 8 of row r, stored at unit (j % 8) ^ (r % 8)
                    const int r = r0 + 8 * h;
                    const uint32_t a2 = *reinterpret_cast<const uint32_t *>(
                        stg + (j >> 3) * kWsBoxBytes + r * 128 + (((j & 7) ^ (r & 7)) << 4) + 2 * cq);
                    v0 += St16<TE>::lo(a2); v1 += St16<TE>::hi(a2);
                }
                acc[4 * j + 2 * h] = v0; acc[4 * j + 2 * h + 1] = v1;
            }
        }
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == passes) break;
            // the previous store has finished reading the staging buffer (leader waited) and the addend is read
            asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                    if (p.out_f32) {
                        // fp32 box jj / 4 of this pass, 16 B unit 2 (jj % 4) + cq / 4
                        if (j * 8 / kF32PassCols != pass) continue;
                        const int jj = j - pass * (kF32PassCols / 8);
                        const int unit = 2 * (jj & 3) + (cq >> 2);
                        *reinterpret_cast<float2 *>(stg + (jj >> 2) * kWsBoxBytes + r * 128 + ((unit ^ (r & 7)) << 4) +
                                                    4 * (cq & 3)) = make_float2(v0, v1);
                    } else {
                        *reinterpret_cast<uint32_t *>(stg + (j >> 3) * kWsBoxBytes + r * 128 +
                                                      (((j & 7) ^ (r & 7)) << 4) + 2 * cq) = St16<TE>::pack(v0, v1);
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
            if (leader) {
                const int cols_per_box = p.out_f32 ? 32 : 64, pc0 = col0 + pass * (BN / passes);
                for (int b = 0; b < BN / passes / cols_per_box && pc0 + b * cols_per_box < p.N; ++b)
                    tma_store_2d(&map_y, stg + b * kWsBoxBytes, pc0 + b * cols_per_box, tm * kWsRows);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            }
        }
        if (leader && p.addend) mbar_arrive(&stg_empty[cw]);
    }
    if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// second pass of the two-pass weight gradient: dW[n, k] = sum over splits of the partial slabs, written
// in the parameter's own dtype (no zero-fill, no cast kernel); db likewise.  kAcc: dw / db (fp32) are added into.
// The slabs are summed in split order, so the result does not depend on how the splits were scheduled.
template <typename TO, bool kAcc = false>
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float *__restrict__ ws, const float *__restrict__ ws_b, TO *__restrict__ dw,
                    TO *__restrict__ db, int N, int K, int n_pad, int splits) {
    static_assert(!kAcc || sizeof(TO) == 4, "accumulation into fp32 only");
    const int kv = K / 4;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)N * kv;
    if (t < total) {
        const int n = (int)(t / kv), c = (int)(t % kv) * 4;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        const float *src = ws + (size_t)n * K + c;
        const size_t slab = (size_t)n_pad * K;
#pragma unroll 4
        for (int s2 = 0; s2 < splits; ++s2) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(src + s2 * slab));
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        if constexpr (sizeof(TO) == 2) {
            *reinterpret_cast<uint2 *>(dw + (size_t)n * K + c) = make_uint2(St16<TO>::pack(a.x, a.y), St16<TO>::pack(a.z, a.w));
        } else if constexpr (kAcc) {
            float4 *d = reinterpret_cast<float4 *>(dw + (size_t)n * K + c);
            const float4 o = *d;
            *d = make_float4(o.x + a.x, o.y + a.y, o.z + a.z, o.w + a.w);
        } else {
            *reinterpret_cast<float4 *>(dw + (size_t)n * K + c) = a;
        }
    } else if (db && t < total + N) {
        const int n = (int)(t - total);
        float a = 0.f;
        for (int s2 = 0; s2 < splits; ++s2) a += ws_b[(size_t)s2 * n_pad + n];
        if constexpr (sizeof(TO) == 2) db[n] = St16<TO>::from_f(a);
        else if constexpr (kAcc) db[n] += a;
        else db[n] = a;
    }
}

// ---- host side ----------------------------------------------------------------------------------
// cuTensorMapEncodeTiled is a driver-API symbol; resolve it through the runtime at first use so that
// the library carries no link-time dependency on libcuda.so (it must load on GPU-less build hosts).
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// row-major (rows, cols) of BEVF_DTYPE_* dt; box = box_rows x 128 B, SWIZZLE_128B; out-of-range rows and columns of
// a box read as zeros (and still count towards the transaction bytes), and are not written by a store
static int make_map_2d(CUtensorMap *map, const void *ptr, uint64_t rows, uint64_t cols, uint32_t box_rows, int dt) {
    EncodeTiledFn encode = encode_tiled_fn();
    if (!encode) return -1;
    const bool f32 = dt == BEVF_DTYPE_F32;
    const uint32_t esz = f32 ? 4 : 2;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * esz};
    cuuint32_t box[2] = {128 / esz, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType ty = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : dt == BEVF_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult r = encode(map, ty, 2,
                        const_cast<void *>(ptr), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

// Launch of one instantiation; the operand maps are built by the caller.  A is 128 x 64 per k-block (K-major:
// one 128-row box; MN-major: two 64 x 64 boxes), B is BN x 64 (K-major: one BN-row box; MN-major: BN / 64 boxes).
template <int BN, bool kAmn, bool kBmn, typename TE>
static int launch_gemm(const char *who, const CUtensorMap &map_a, const CUtensorMap &map_b, GemmParams p,
                       cudaStream_t st) {
    constexpr int kStageBytes = kBM * 128 + BN * 128;
    int stages = (227 * 1024 - 1024 - 256) / kStageBytes;
    if (stages > kMaxStages) stages = kMaxStages;
    p.stages = stages;
    const size_t smem = 1024 + (size_t)stages * kStageBytes + 2 * kMaxStages * 8;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(gemm_bf16_wgmma<BN, kAmn, kBmn, TE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory for the GEMM", who);
        }
        configured = true;
    }
    const int units = ((p.M + kBM - 1) / kBM) * ((p.N + BN - 1) / BN) * p.splits;
    const int grid = units < device_sms() ? units : device_sms();
    gemm_bf16_wgmma<BN, kAmn, kBmn, TE><<<grid, kGemmThreads, smem, st>>>(map_a, map_b, p);
    return check_launch(who);
}

// Column block of the weight-stationary kernel: the widest of 256 / 128 / 64 whose BN x R weight tile fits in
// kWsWeightMax and that the N output columns do not leave more than half empty; 0 if not even 64 fits
// (reductions longer than 1024, which the encoder never runs, go to the streamed kernel above).
static int ws_block(int N, int R) {
    int bn = 256;
    while (bn > 64 && (bn * R * 2 > kWsWeightMax || bn / 2 >= N)) bn /= 2;
    return bn * R * 2 <= kWsWeightMax ? bn : 0;
}

template <int BN, bool kBmn, typename TE>
static int launch_ws(const char *who, const CUtensorMap &map_a, const CUtensorMap &map_w, const CUtensorMap &map_y,
                     const CUtensorMap &map_add, WsParams p, cudaStream_t st) {
    constexpr int kSmemMax = 227 * 1024;
    constexpr int kBarBytes = (1 + 4 * kMaxStages + 4) * 8 + BN * 4;   // + the bias block
    p.stg_bytes = kWsRows * BN * (p.out_f32 ? 4 : 2);
    if (p.stg_bytes > kWsStageMax) p.stg_bytes = kWsStageMax;
    const int w_bytes = p.R * BN * 2;
    int stages = (kSmemMax - 1024 - kBarBytes - w_bytes - 2 * p.stg_bytes) / (2 * kWsBoxBytes);
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 2) return fail("%s: no room for a two-stage A ring next to the weight tile", who);
    p.stages = stages;
    const size_t smem = 1024 + (size_t)w_bytes + 2 * p.stg_bytes + 2 * (size_t)stages * kWsBoxBytes + kBarBytes;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(gemm_ws_wgmma<BN, kBmn, TE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax) !=
            cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory for the GEMM", who);
        }
        configured = true;
    }
    p.tiles_m = (p.M + kWsRows - 1) / kWsRows;
    p.tiles_n = (p.N + BN - 1) / BN;
    p.groups = device_sms() / p.tiles_n;
    if (p.groups > p.tiles_m) p.groups = p.tiles_m;
    if (p.groups < 1) p.groups = 1;
    gemm_ws_wgmma<BN, kBmn, TE><<<p.groups * p.tiles_n, kGemmThreads, smem, st>>>(map_a, map_w, map_y, map_add, p);
    return check_launch(who);
}

// Y (M, N) = act(A (M, R) . B + bias) (+ addend) on the weight-stationary kernel; B is W (N, R) for the forward
// product, or W (R, N) read in place (MN-major) for the input gradient.
template <typename TE> constexpr int dtype_of() { return std::is_same<TE, __half>::value ? BEVF_DTYPE_F16 : BEVF_DTYPE_BF16; }

template <typename TE>
static int linear_ws(const char *who, int bn, bool b_mn, const void *a, const void *w, const void *bias, int bias_dt,
                     const void *addend, void *y, bool out_f32, int M, int N, int R, int relu, cudaStream_t st) {
    constexpr int dt = dtype_of<TE>();
    CUtensorMap map_a, map_w, map_y, map_add;
    if (int e = make_map_2d(&map_a, a, (uint64_t)M, (uint64_t)R, kWsRows, dt))
        return fail("%s: cuTensorMapEncodeTiled(A) failed (%lld)", who, e);
    if (int e = b_mn ? make_map_2d(&map_w, w, (uint64_t)R, (uint64_t)N, 64, dt)
                     : make_map_2d(&map_w, w, (uint64_t)N, (uint64_t)R, (uint32_t)bn, dt))
        return fail("%s: cuTensorMapEncodeTiled(B) failed (%lld)", who, e);
    if (int e = make_map_2d(&map_y, y, (uint64_t)M, (uint64_t)N, kWsRows, out_f32 ? BEVF_DTYPE_F32 : dt))
        return fail("%s: cuTensorMapEncodeTiled(Y) failed (%lld)", who, e);
    map_add = map_y;
    if (addend)
        if (int e = make_map_2d(&map_add, addend, (uint64_t)M, (uint64_t)N, kWsRows, dt))
            return fail("%s: cuTensorMapEncodeTiled(addend) failed (%lld)", who, e);
    WsParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.R = R;
    p.relu = relu; p.bias = bias; p.bias_dt = bias_dt;
    p.addend = addend != nullptr; p.out_f32 = out_f32;
    switch (bn * 2 + (int)b_mn) {
        case 512: return launch_ws<256, false, TE>(who, map_a, map_w, map_y, map_add, p, st);
        case 513: return launch_ws<256, true, TE>(who, map_a, map_w, map_y, map_add, p, st);
        case 256: return launch_ws<128, false, TE>(who, map_a, map_w, map_y, map_add, p, st);
        case 257: return launch_ws<128, true, TE>(who, map_a, map_w, map_y, map_add, p, st);
        case 128: return launch_ws<64, false, TE>(who, map_a, map_w, map_y, map_add, p, st);
        case 129: return launch_ws<64, true, TE>(who, map_a, map_w, map_y, map_add, p, st);
    }
    return fail("%s: no weight-stationary tile for this shape", who);
}

static GemmParams base_params(int M, int N, int R) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.R = R; p.rows_per_split = ((R + kBK - 1) / kBK) * kBK; p.splits = 1;
    p.ldy = N;
    return p;
}

}  // namespace bevf

using namespace bevf;

// operand type of the *_dt entry points: bf16 or fp16
static bool operand_dtype_ok(int dtype) { return dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F16; }

template <typename TE>
static int linear_dgrad_impl(const char *who, const void *dy, const void *w, const void *addend, void *dx, int64_t M,
                             int N, int K, void *stream) {
    constexpr int dt = dtype_of<TE>();
    if (M < 0 || N <= 0 || K <= 0) return fail("%s: bad dimension", who);
    if (M == 0) return 0;
    if (!dy || !w || !dx) return fail("%s: null pointer argument", who);
    if (N % kBK != 0 || K % 64 != 0) return fail("%s: N and K must be multiples of 64 (got %lld, %lld)", who, N, K);
    if (M >= (1ll << 31)) return fail("%s: M too large", who);
    if (!aligned16(dy) || !aligned16(w) || !aligned16(dx)) return fail("%s: pointers must be 16-byte aligned", who);
    // dX (M, K) = dY (M, N) . W (N, K): A = dY K-major, B = W with its output columns contiguous (MN-major)
    cudaStream_t st = (cudaStream_t)stream;
    if (int bn = ws_block(K, N))
        return linear_ws<TE>(who, bn, true, dy, w, nullptr, BEVF_DTYPE_F32, addend, dx, false, (int)M, K, N, 0, st);
    CUtensorMap map_a, map_b;
    if (int e = make_map_2d(&map_a, dy, (uint64_t)M, (uint64_t)N, kBM, dt))
        return fail("%s: cuTensorMapEncodeTiled(A) failed (%lld)", who, e);
    if (int e = make_map_2d(&map_b, w, (uint64_t)N, (uint64_t)K, 64, dt))
        return fail("%s: cuTensorMapEncodeTiled(B) failed (%lld)", who, e);
    GemmParams p = base_params((int)M, K, N);
    p.addend = addend;
    p.y = dx;
    return K % 128 == 0 ? launch_gemm<128, false, true, TE>(who, map_a, map_b, p, st)
                        : launch_gemm<64, false, true, TE>(who, map_a, map_b, p, st);
}

static int linear_dgrad_dispatch(const char *who, const void *dy, const void *w, const void *addend, void *dx,
                                 int64_t M, int N, int K, int dtype, void *stream) {
    if (addend && !aligned16(addend)) return fail("%s: addend must be 16-byte aligned", who);
    if (dtype == BEVF_DTYPE_F16) return linear_dgrad_impl<__half>(who, dy, w, addend, dx, M, N, K, stream);
    if (dtype == BEVF_DTYPE_BF16) return linear_dgrad_impl<bf16>(who, dy, w, addend, dx, M, N, K, stream);
    return fail("%s: unsupported operand dtype code (bf16 or fp16)", who);
}

extern "C" int bevf_linear_dgrad(const void *dy, const void *w, void *dx, int64_t M, int N, int K, void *stream) {
    return linear_dgrad_dispatch("bevf_linear_dgrad", dy, w, nullptr, dx, M, N, K, BEVF_DTYPE_BF16, stream);
}

extern "C" int bevf_linear_dgrad_dt(const void *dy, const void *w, void *dx, int64_t M, int N, int K, int dtype,
                                    void *stream) {
    return linear_dgrad_dispatch("bevf_linear_dgrad_dt", dy, w, nullptr, dx, M, N, K, dtype, stream);
}

extern "C" int bevf_linear_dgrad_acc(const void *dy, const void *w, const void *addend, void *dx, int64_t M, int N,
                                     int K, void *stream) {
    return linear_dgrad_dispatch("bevf_linear_dgrad_acc", dy, w, addend, dx, M, N, K, BEVF_DTYPE_BF16, stream);
}

extern "C" int bevf_linear_dgrad_acc_dt(const void *dy, const void *w, const void *addend, void *dx, int64_t M, int N,
                                        int K, int dtype, void *stream) {
    return linear_dgrad_dispatch("bevf_linear_dgrad_acc_dt", dy, w, addend, dx, M, N, K, dtype, stream);
}

template <typename TE>
static int linear_forward_impl(const char *who, const void *x, const void *w, const void *bias, int bias_dtype,
                               const void *residual, void *y, int y_dtype, int64_t M, int N, int K, int relu,
                               void *stream) {
    constexpr int dt = dtype_of<TE>();
    if (M < 0 || N <= 0 || K <= 0) return fail("%s: bad dimension", who);
    if (M == 0) return 0;
    if (!x || !w || !y) return fail("%s: null pointer argument", who);
    if (K % kBK != 0) return fail("%s: K must be a multiple of 64 (got %lld)", who, K);
    if (N % 16 != 0) return fail("%s: N must be a multiple of 16 (got %lld)", who, N);
    if (M >= (1ll << 31)) return fail("%s: M too large", who);
    if (!aligned16(x) || !aligned16(w) || !aligned16(y) || (bias && !aligned16(bias)) ||
        (residual && !aligned16(residual)))
        return fail("%s: pointers must be 16-byte aligned", who);
    if (y_dtype != dt && y_dtype != BEVF_DTYPE_F32) return fail("%s: unsupported dtype code", who);
    if (bias && bias_dtype != dt && bias_dtype != BEVF_DTYPE_F32)
        return fail("%s: unsupported bias dtype code", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (int bn = ws_block(N, K))
        return linear_ws<TE>(who, bn, false, x, w, bias, bias_dtype, residual, y, y_dtype == BEVF_DTYPE_F32, (int)M, N,
                             K, relu, st);
    // a column tile of 128 unless N is small (a partial last tile is clipped in the epilogue)
    const bool wide = N > 64;
    CUtensorMap map_a, map_b;
    if (int e = make_map_2d(&map_a, x, (uint64_t)M, (uint64_t)K, kBM, dt))
        return fail("%s: cuTensorMapEncodeTiled(A) failed (%lld)", who, e);
    if (int e = make_map_2d(&map_b, w, (uint64_t)N, (uint64_t)K, wide ? 128 : 64, dt))
        return fail("%s: cuTensorMapEncodeTiled(B) failed (%lld)", who, e);
    GemmParams p = base_params((int)M, N, K);
    p.relu = relu; p.bias = bias; p.bias_dt = bias_dtype;
    p.addend = residual;
    p.y = y; p.out_f32 = y_dtype == BEVF_DTYPE_F32;
    return wide ? launch_gemm<128, false, false, TE>(who, map_a, map_b, p, st)
                : launch_gemm<64, false, false, TE>(who, map_a, map_b, p, st);
}

extern "C" int bevf_linear_forward_dt(const void *x, const void *w, const void *bias, int bias_dtype,
                                      const void *residual, void *y, int y_dtype, int64_t M, int N, int K, int relu,
                                      int dtype, void *stream) {
    const char *who = "bevf_linear_forward_dt";
    if (dtype == BEVF_DTYPE_F16)
        return linear_forward_impl<__half>(who, x, w, bias, bias_dtype, residual, y, y_dtype, M, N, K, relu, stream);
    if (dtype == BEVF_DTYPE_BF16)
        return linear_forward_impl<bf16>(who, x, w, bias, bias_dtype, residual, y, y_dtype, M, N, K, relu, stream);
    return fail("%s: unsupported operand dtype code (bf16 or fp16)", who);
}

extern "C" int bevf_linear_forward(const void *x, const void *w, const void *bias, int bias_dtype,
                                   const void *residual, void *y, int y_dtype, int64_t M, int N, int K,
                                   int relu, void *stream) {
    return linear_forward_impl<bf16>("bevf_linear_forward", x, w, bias, bias_dtype, residual, y, y_dtype, M, N, K,
                                     relu, stream);
}

// Plan of the weight gradient, shared by the workspace query and the launches: tile width along K, number of
// splits of the M rows (about one unit per SM) and rows per split, padded row count of dW.
static void wgrad_plan(int64_t M, int N, int K, int &bn, int &splits, int &rows, int &n_pad) {
    bn = K % 128 == 0 ? 128 : 64;
    const int tiles_m = (N + kBM - 1) / kBM;
    const int tiles = tiles_m * (K / bn);
    splits = (device_sms() + tiles - 1) / tiles;
    rows = (int)((M + splits - 1) / splits);
    rows = ((rows + 63) / 64) * 64;
    splits = (int)((M + rows - 1) / rows);
    n_pad = tiles_m * kBM;
}

// dW (N, K) = dY^T . X: both operands MN-major (dY (M, N) and X (M, K) read row-major, reduction over M)
template <typename TE>
static int launch_wgrad(const char *who, const void *dy, const void *x, GemmParams p, int bn, cudaStream_t st) {
    constexpr int dt = dtype_of<TE>();
    CUtensorMap map_a, map_b;
    if (int e = make_map_2d(&map_a, dy, (uint64_t)p.R, (uint64_t)p.M, 64, dt))
        return fail("%s: cuTensorMapEncodeTiled(dY) failed (%lld)", who, e);
    if (int e = make_map_2d(&map_b, x, (uint64_t)p.R, (uint64_t)p.N, 64, dt))
        return fail("%s: cuTensorMapEncodeTiled(X) failed (%lld)", who, e);
    return bn == 128 ? launch_gemm<128, true, true, TE>(who, map_a, map_b, p, st)
                     : launch_gemm<64, true, true, TE>(who, map_a, map_b, p, st);
}

static int linear_wgrad_impl(const char *who, const void *dy, const void *x, float *dw, float *db, int64_t M, int N,
                             int K, int dtype, void *stream) {
    if (M < 0 || N <= 0 || K <= 0) return fail("%s: bad dimension", who);
    if (M == 0) return 0;
    if (!dy || !x || !dw) return fail("%s: null pointer argument", who);
    if (K % 64 != 0 || N % 8 != 0) return fail("%s: K must be a multiple of 64 and N of 8", who);
    if (db && !aligned16(db)) return fail("%s: pointers must be 16-byte aligned", who);
    if (M >= (1ll << 31)) return fail("%s: M too large", who);
    if (!aligned16(dy) || !aligned16(x) || !aligned16(dw)) return fail("%s: pointers must be 16-byte aligned", who);
    if (!operand_dtype_ok(dtype)) return fail("%s: unsupported operand dtype code (bf16 or fp16)", who);
    int bn, splits, rows, n_pad;
    wgrad_plan(M, N, K, bn, splits, rows, n_pad);
    GemmParams p = base_params(N, K, (int)M);
    p.rows_per_split = rows; p.splits = splits;
    p.y = dw; p.ldy = K; p.out_f32 = 1; p.red = 1;      // every split reduces its partial tile into dW
    p.db = db;
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == BEVF_DTYPE_F16 ? launch_wgrad<__half>(who, dy, x, p, bn, st)
                                   : launch_wgrad<bf16>(who, dy, x, p, bn, st);
}

extern "C" int bevf_linear_wgrad(const void *dy, const void *x, float *dw, float *db, int64_t M, int N,
                                 int K, void *stream) {
    return linear_wgrad_impl("bevf_linear_wgrad", dy, x, dw, db, M, N, K, BEVF_DTYPE_BF16, stream);
}

extern "C" int bevf_linear_wgrad_dt(const void *dy, const void *x, float *dw, float *db, int64_t M, int N, int K,
                                    int dtype, void *stream) {
    return linear_wgrad_impl("bevf_linear_wgrad_dt", dy, x, dw, db, M, N, K, dtype, stream);
}

extern "C" int64_t bevf_linear_wgrad_workspace_bytes(int64_t M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0 || K % 64 != 0) return 0;
    int bn, splits, rows, n_pad;
    wgrad_plan(M, N, K, bn, splits, rows, n_pad);
    return (int64_t)splits * n_pad * ((int64_t)K + 1) * 4 + 256;
}

// grad_dtype, or accumulate != 0: dw / db fp32 and added into
static int wgrad_two_pass(const char *who, const void *dy, const void *x, void *dw, void *db, int grad_dtype,
                          int accumulate, void *workspace, int64_t workspace_bytes, int64_t M, int N, int K,
                          int dtype, void *stream) {
    if (M <= 0 || N <= 0 || K <= 0) return fail("%s: bad dimension", who);
    if (!dy || !x || !dw || !workspace) return fail("%s: null pointer argument", who);
    if (K % 64 != 0 || N % 8 != 0) return fail("%s: K must be a multiple of 64 and N of 8", who);
    if (M >= (1ll << 31)) return fail("%s: M too large", who);
    if (!aligned16(dy) || !aligned16(x) || !aligned16(dw) || !aligned16(workspace))
        return fail("%s: pointers must be 16-byte aligned", who);
    if (!operand_dtype_ok(dtype)) return fail("%s: unsupported operand dtype code (bf16 or fp16)", who);
    if (grad_dtype != BEVF_DTYPE_BF16 && grad_dtype != BEVF_DTYPE_F16 && grad_dtype != BEVF_DTYPE_F32)
        return fail("%s: unsupported dtype code", who);
    if (workspace_bytes < bevf_linear_wgrad_workspace_bytes(M, N, K))
        return fail("%s: workspace too small (need %lld bytes)", who, bevf_linear_wgrad_workspace_bytes(M, N, K));
    int bn, splits, rows, n_pad;
    wgrad_plan(M, N, K, bn, splits, rows, n_pad);
    // pass 1: every split stores its partial tile into its own slab (plain stores, no contended reductions)
    float *ws = reinterpret_cast<float *>(workspace);
    float *ws_b = ws + (size_t)splits * n_pad * K;
    GemmParams p = base_params(N, K, (int)M);
    p.rows_per_split = rows; p.splits = splits;
    p.y = ws; p.ldy = K; p.split_stride = (int64_t)n_pad * K; p.out_f32 = 1;
    p.db_ws = db ? ws_b : nullptr; p.n_pad = n_pad;
    cudaStream_t cs = (cudaStream_t)stream;
    if (int e = dtype == BEVF_DTYPE_F16 ? launch_wgrad<__half>(who, dy, x, p, bn, cs)
                                       : launch_wgrad<bf16>(who, dy, x, p, bn, cs))
        return e;
    // pass 2: sum the slabs in the parameter's dtype
    const long long total = (long long)N * (K / 4) + (db ? N : 0);
    const unsigned rgrid = (unsigned)((total + 255) / 256);
    if (accumulate)
        wgrad_reduce_kernel<float, true><<<rgrid, 256, 0, cs>>>(ws, ws_b, (float *)dw, (float *)db, N, K, n_pad, splits);
    else if (grad_dtype == BEVF_DTYPE_BF16)
        wgrad_reduce_kernel<bf16><<<rgrid, 256, 0, cs>>>(ws, ws_b, (bf16 *)dw, (bf16 *)db, N, K, n_pad, splits);
    else if (grad_dtype == BEVF_DTYPE_F16)
        wgrad_reduce_kernel<__half><<<rgrid, 256, 0, cs>>>(ws, ws_b, (__half *)dw, (__half *)db, N, K, n_pad, splits);
    else
        wgrad_reduce_kernel<float><<<rgrid, 256, 0, cs>>>(ws, ws_b, (float *)dw, (float *)db, N, K, n_pad, splits);
    return check_launch(who);
}

extern "C" int bevf_linear_wgrad_out(const void *dy, const void *x, void *dw, void *db, int grad_dtype,
                                     void *workspace, int64_t workspace_bytes, int64_t M, int N, int K,
                                     void *stream) {
    return wgrad_two_pass("bevf_linear_wgrad_out", dy, x, dw, db, grad_dtype, 0, workspace, workspace_bytes, M, N, K,
                          BEVF_DTYPE_BF16, stream);
}

extern "C" int bevf_linear_wgrad_out_dt(const void *dy, const void *x, void *dw, void *db, int grad_dtype,
                                        void *workspace, int64_t workspace_bytes, int64_t M, int N, int K, int dtype,
                                        void *stream) {
    return wgrad_two_pass("bevf_linear_wgrad_out_dt", dy, x, dw, db, grad_dtype, 0, workspace, workspace_bytes, M, N,
                          K, dtype, stream);
}

extern "C" int bevf_linear_wgrad_into(const void *dy, const void *x, float *dw, float *db, void *workspace,
                                      int64_t workspace_bytes, int64_t M, int N, int K, void *stream) {
    return wgrad_two_pass("bevf_linear_wgrad_into", dy, x, dw, db, BEVF_DTYPE_F32, 1, workspace, workspace_bytes, M, N,
                          K, BEVF_DTYPE_BF16, stream);
}

extern "C" int bevf_linear_wgrad_into_dt(const void *dy, const void *x, float *dw, float *db, void *workspace,
                                         int64_t workspace_bytes, int64_t M, int N, int K, int dtype, void *stream) {
    return wgrad_two_pass("bevf_linear_wgrad_into_dt", dy, x, dw, db, BEVF_DTYPE_F32, 1, workspace, workspace_bytes,
                          M, N, K, dtype, stream);
}
