// Sampler forward with TMA-staged pyramid levels (sm_90a).
//
// Same arithmetic as msda_fwd_d32 (msda.cu; reference: mmcv ms_deform_attn_forward as called at
// projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:118-124), different
// data path for the coarse levels.  In SpatialCrossAttention every camera's 7-9 k in-view queries sample
// 8 points on each pyramid level; on the two coarsest levels (29x50 and 15x25 at base) that is ~600 /
// ~150 fetches per pixel, all of which the plain kernel sends through L1 as 64 B gathers (1.75 GB of L1
// traffic for 0.25 GB of compulsory bytes, l1tex 84 % busy).  Here a CTA owns one (value map, head) pair
// and a contiguous share of that map's rows:
//   * thread 0 issues ONE cp.async.bulk.tensor (TMA, 5-D box {32 channels, 1 head, W_l, H_l, 1 map}) per
//     staged level -- the whole level of this head, H_l*W_l rows of 64 B (bf16) -- completing on an
//     mbarrier; the level then sits densely in shared memory (117 KB for levels 2+3 at base);
//   * samples on staged levels gather with ld.shared.v4 (no tags, no L2 round trips); samples on the
//     fine levels keep the read-only global path;
//   * everything else is msda_fwd_d32's scheme: a lane group of 32/VEC lanes per (row, head), scalar
//     work done once per sample and handed round with shuffles, fp32 FMA accumulation of the widened bf16 operands.
// Levels are staged from the coarsest down while they fit (box sides <= 256, <= 200 KB in total).
// The level shapes must be known on the host to build the tensor maps; the kernel compares them with
// the device-side spatial_shapes and falls back to the global path for a level that disagrees.
#include <cuda.h>

#include "msda_common.cuh"

namespace bevf {

constexpr int kStagedThreads = 1024;
constexpr int kMaxStaged = 4;

struct StagedMaps { CUtensorMap m[kMaxStaged]; };
struct StagedInfo {
    int nstaged;
    int level[kMaxStaged];        // pyramid level of staged slot i
    int h[kMaxStaged], w[kMaxStaged];
    int smem_off[kMaxStaged];     // byte offset of the slot in the staging buffer (128 B aligned)
    int bytes[kMaxStaged];
};

__device__ __forceinline__ uint32_t s_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1,
                                            int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

struct StagedTab {
    int h[kMaxLevels], w[kMaxLevels], rs[kMaxLevels];   // rs: element stride between image rows (global path)
    long long lofs[kMaxLevels];
    int sbase[kMaxLevels];        // shared-memory byte address of the staged level, 0 = not staged
    int srow[kMaxLevels];         // bytes between image rows in the staged copy
};

// Lane mapping (bf16): 8 lanes per (row, head) -- lanes 0-3 own the LEFT corner column (x0), lanes 4-7 the
// RIGHT one (x0 + 1), 16 B (8 channels) each; a warp covers 4 rows.  In the staged copy of a level the
// pixels of one head are dense, so the left and right corner of a sample are ADJACENT 64 B rows: the 8
// lanes of a group read one contiguous 128 B span per image row -- a conflict-free shared-memory phase,
// two ld.shared.v4 per sample instead of four 64 B gathers.  The two column sums meet in one shuffle per
// accumulator at the end of the row.  Unstaged (fine) levels use the same mapping on the global path.
// Work distribution: persistent CTAs (one per SM); the rows of every value map are cut into units of
// kUnitRows rows x one head, listed (map, head, chunk)-major, and every CTA takes an equal contiguous
// share of the list, re-staging whenever the (map, head) changes (117 KB from L2: ~1 us per 40 us unit).
constexpr int kUnitRows = 512;

template <typename T, typename TO>
__global__ void __launch_bounds__(kStagedThreads, 1)
msda_fwd_staged_d32(const __grid_constant__ StagedMaps maps, const StagedInfo info,
                    const T *__restrict__ value, const int64_t *__restrict__ level_hw,
                    const int64_t *__restrict__ level_start, const float *__restrict__ loc,
                    const float *__restrict__ attn, TO *__restrict__ out,
                    const int *__restrict__ map_range, int NB, int S, int M, int L, int P, int magic) {
    constexpr int VEC = Vec<T>::N;                 // channels per lane (16 B)
    constexpr int QL = 32 / VEC;                   // lanes per 32-channel row: 4 (bf16) / 8 (fp32)
    constexpr int LANES = 2 * QL;                  // lanes per (row, head): left + right column
    constexpr int G = 32 / LANES;                  // rows per warp: 4 (bf16) / 2 (fp32)
    constexpr bool kHalf = (VEC == 8);
    constexpr int kRowBytes = 32 * (int)sizeof(T);
    extern __shared__ __align__(128) unsigned char stage[];
    __shared__ StagedTab tab;
    __shared__ __align__(8) unsigned long long bar;
    __shared__ int s_ok[kMaxStaged];

    const int pix = M * 32;
    if ((int)threadIdx.x < L) {
        const int l = threadIdx.x;
        tab.h[l] = (int)level_hw[2 * l];
        tab.w[l] = (int)level_hw[2 * l + 1];
        tab.rs[l] = tab.w[l] * pix;
        tab.lofs[l] = (long long)level_start[l] * pix;
        tab.sbase[l] = 0;
        tab.srow[l] = 0;
    }
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(&bar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // the host's idea of the staged levels must match the device's spatial_shapes / level_start
        long long start = 0;
        for (int i = 0; i < kMaxStaged; ++i) s_ok[i] = 0;
        for (int l = 0; l < L; ++l) {
            for (int i = 0; i < info.nstaged; ++i)
                if (info.level[i] == l && info.h[i] == tab.h[l] && info.w[i] == tab.w[l] &&
                    tab.lofs[l] == start * pix) {
                    s_ok[i] = 1;
                    tab.sbase[l] = (int)s_u32(stage + info.smem_off[i]);
                    tab.srow[l] = info.w[i] * kRowBytes;
                }
            start += (long long)tab.h[l] * tab.w[l];
        }
    }
    __syncthreads();

    // ---- this CTA's share of the unit list
    int total = 0;
    for (int bb = 0; bb < NB; ++bb) {
        const int n = __ldg(map_range + 2 * bb + 1) - __ldg(map_range + 2 * bb);
        total += ((n + kUnitRows - 1) / kUnitRows) * M;
    }
    const int per_cta = (total + (int)gridDim.x - 1) / (int)gridDim.x;
    const int u0 = (int)blockIdx.x * per_cta, u1 = min(total, u0 + per_cta);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane / LANES, gl = lane % LANES;     // row group, lane inside it
    const int half = gl / QL, sub = gl % QL;             // corner column (0 left / 1 right), 16 B slice
    const int LP = L * P;
    int cur_b = -1, cur_m = -1;
    uint32_t phase = 0;

    for (int u = u0; u < u1; ++u) {
        // decode unit -> (map b, head m, chunk)
        int b = 0, rem = u, cnt = 0, ps = 0, pe = 0;
        for (; b < NB; ++b) {
            ps = __ldg(map_range + 2 * b); pe = __ldg(map_range + 2 * b + 1);
            cnt = (pe - ps + kUnitRows - 1) / kUnitRows;
            if (rem < cnt * M) break;
            rem -= cnt * M;
        }
        const int m = rem / cnt, chunk = rem - m * cnt;
        const int r0 = ps + chunk * kUnitRows, r1 = min(pe, r0 + kUnitRows);
        if (b != cur_b || m != cur_m) {                   // (re-)stage the coarse levels of (b, m)
            __syncthreads();                              // every warp is done with the previous copy
            if (threadIdx.x == 0) {
                unsigned bytes = 0;
                for (int i = 0; i < info.nstaged; ++i) if (s_ok[i]) bytes += (unsigned)info.bytes[i];
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(&bar)), "r"(bytes) : "memory");
                for (int i = 0; i < info.nstaged; ++i)
                    if (s_ok[i]) tma_load_5d(s_u32(stage + info.smem_off[i]), &maps.m[i], s_u32(&bar), 0, m, 0, 0, b);
            }
            asm volatile(
                "{\n.reg .pred p;\nWAITL:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONEL;\nbra WAITL;\nDONEL:\n}\n"
                ::"r"(s_u32(&bar)), "r"(phase) : "memory");
            phase ^= 1u;
            cur_b = b; cur_m = m;
        }
        const T *vmap = value + ((long long)b * S * M + m) * 32 + sub * VEC;

        for (int base = r0 + warp * G; base < r1; base += (kStagedThreads / 32) * G) {
            int pair = base + grp;
            const bool live = pair < r1;
            if (!live) pair = r1 - 1;
            const long long row = (long long)pair * M + m;
            const float2 *locp = reinterpret_cast<const float2 *>(loc) + row * LP;
            const float *attp = attn + row * LP;
            float acc[VEC];
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
            for (int s0 = 0; s0 < LP; s0 += LANES) {
                // ---- produce: lane gl of the group prepares sample s0 + gl
                const int sm = s0 + gl;
                int enc = 0;                      // (clamped top-left pixel index << 2) | dx | dy << 1
                float w00 = 0.f, w01 = 0.f, w10 = 0.f, w11 = 0.f;
                bool valid = false;
                if (sm < LP && live) {
                    const int l = level_of(sm, magic);
                    const float2 xy = __ldg(locp + sm);
                    const float a = __ldg(attp + sm);
                    const Corner c = make_corner(xy.x, xy.y, tab.h[l], tab.w[l]);
                    enc = (c.pidx << 2) | c.dx | (c.dy << 1);
                    valid = c.valid;
                    w00 = c.w00 * a; w01 = c.w01 * a; w10 = c.w10 * a; w11 = c.w11 * a;
                }
                uint32_t wa = 0, wb = 0;
                if constexpr (kHalf) { wa = pack_bf16x2(w00, w01); wb = pack_bf16x2(w10, w11); }
                const unsigned vm = __ballot_sync(0xffffffffu, valid);
                // ---- consume: the LANES samples of this round, one after the other
#pragma unroll
                for (int j = 0; j < LANES; ++j) {
                    if (s0 + j >= LP) break;
                    if (!(vm & (GroupMask<LANES>::kBits << j))) continue;
                    const int src = grp * LANES + j;
                    const unsigned e = (unsigned)__shfl_sync(0xffffffffu, enc, src);
                    const int l = level_of(s0 + j, magic);
                    const unsigned pcol = (e >> 2) + ((half && (e & 1u)) ? 1u : 0u);   // pixel of MY corner column, top row
                    Vec<T> vt, vb;                                                   // top / bottom corner of my column
                    const int sb = tab.sbase[l];                                     // warp-uniform
                    if (sb != 0) {
                        const uint32_t at = (uint32_t)sb + pcol * kRowBytes + sub * 16;
                        vt.v = vec_bits<T>(lds128(at));
                        vb.v = vec_bits<T>(lds128(at + ((e & 2u) ? (uint32_t)tab.srow[l] : 0u)));
                    } else {
                        const T *vl = vmap + tab.lofs[l];
                        const unsigned ot = pcol * (unsigned)pix;
                        vt.load(vl + ot);
                        vb.load(vl + (ot + ((e & 2u) ? (unsigned)tab.rs[l] : 0u)));
                    }
                    if constexpr (kHalf) {
                        const uint32_t qa = __shfl_sync(0xffffffffu, wa, src);       // {w00 | w01 << 16}
                        const uint32_t qb = __shfl_sync(0xffffffffu, wb, src);       // {w10 | w11 << 16}
                        const unsigned short ht = (unsigned short)(half ? (qa >> 16) : (qa & 0xffffu));
                        const unsigned short hb = (unsigned short)(half ? (qb >> 16) : (qb & 0xffffu));
                        vt.axpy_h(ht, acc); vb.axpy_h(hb, acc);
                    } else {
                        // the column is the READER's: fetch both and pick here (the source lane's own
                        // `half` says nothing about which column this lane accumulates)
                        const float q00 = __shfl_sync(0xffffffffu, w00, src), q01 = __shfl_sync(0xffffffffu, w01, src);
                        const float q10 = __shfl_sync(0xffffffffu, w10, src), q11 = __shfl_sync(0xffffffffu, w11, src);
                        vt.axpy(half ? q01 : q00, acc); vb.axpy(half ? q11 : q10, acc);
                    }
                }
            }
            // left + right corner columns
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], QL);
            if (live && half == 0) store_vec<TO, VEC>(out + row * 32 + sub * VEC, acc);
        }
    }
}

// ---- host --------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn5)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                   const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
static EncodeTiledFn5 encode_fn5() {
    static EncodeTiledFn5 fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn5>(p);
    }
    return fn;
}

template <typename T, typename TO>
static int launch_staged(const char *who, const void *value, const int64_t *hw_dev, const int64_t *ls_dev,
                         const int32_t *hw_host, const float *loc, const float *attn, void *out,
                         const int32_t *map_range, int NB, int S, int M, int L, int P, int chunks,
                         cudaStream_t st) {
    EncodeTiledFn5 encode = encode_fn5();
    if (!encode) return fail("%s: cuTensorMapEncodeTiled is not available", who);
    const int es = (int)sizeof(T);
    StagedMaps maps;
    StagedInfo info;
    info.nstaged = 0;
    long long starts[kMaxLevels];
    long long s = 0;
    for (int l = 0; l < L; ++l) { starts[l] = s; s += (long long)hw_host[2 * l] * hw_host[2 * l + 1]; }
    if (s != S) return fail("%s: host level shapes do not add up to S (%lld vs %lld)", who, s, S);
    int used = 0;
    const int budget = 200 * 1024;
    for (int l = L - 1; l >= 0 && info.nstaged < kMaxStaged; --l) {          // coarsest first
        const int h = hw_host[2 * l], w = hw_host[2 * l + 1];
        const long long bytes = (long long)h * w * 32 * es;
        if (h > 256 || w > 256 || used + bytes > budget) break;
        const int i = info.nstaged++;
        info.level[i] = l; info.h[i] = h; info.w[i] = w;
        info.smem_off[i] = used; info.bytes[i] = (int)bytes;
        used += (int)((bytes + 127) / 128 * 128);
        cuuint64_t dims[5] = {32, (cuuint64_t)M, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)NB};
        cuuint64_t strides[4] = {(cuuint64_t)32 * es, (cuuint64_t)M * 32 * es, (cuuint64_t)w * M * 32 * es,
                                 (cuuint64_t)S * M * 32 * es};
        cuuint32_t box[5] = {32, 1, (cuuint32_t)w, (cuuint32_t)h, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        void *base = const_cast<char *>(reinterpret_cast<const char *>(value)) + starts[l] * M * 32 * es;
        CUresult r = encode(&maps.m[i], es == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                            5, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail("%s: cuTensorMapEncodeTiled failed (%lld)", who, (long long)r);
    }
    for (int i = info.nstaged; i < kMaxStaged; ++i) {
        maps.m[i] = maps.m[0];
        info.level[i] = -1; info.h[i] = info.w[i] = info.smem_off[i] = info.bytes[i] = 0;
    }
    if (info.nstaged == 0) return -1;                                         // nothing fits: caller uses the plain kernel
    static bool attr_done = false;
    if (!attr_done) {
        if (cudaFuncSetAttribute(msda_fwd_staged_d32<T, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 budget + 1024) != cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory for the staged sampler", who);
        }
        attr_done = true;
    }
    msda_fwd_staged_d32<T, TO><<<(unsigned)chunks, kStagedThreads, (size_t)used, st>>>(
        maps, info, (const T *)value, hw_dev, ls_dev, loc, attn, (TO *)out, map_range, NB, S, M, L, P,
        (65536 + P - 1) / P);
    return check_launch(who);
}

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_msda_rows_forward_staged(const void *value, int value_dtype, const int64_t *level_hw,
                                             const int64_t *level_start, const int32_t *level_hw_host,
                                             const float *loc, const float *attn, void *out, int out_dtype,
                                             const int32_t *map_range, int B, int S, int M, int D, int R,
                                             int L, int P, void *stream) {
    const char *who = "bevf_msda_rows_forward_staged";
    if (B <= 0 || S <= 0 || M <= 0 || L <= 0 || P <= 0 || R < 0) return fail("%s: bad dimension", who);
    if (D != 32 || L > kMaxLevels) return fail("%s: head_dim must be 32 and num_levels <= 16", who);
    if ((long long)L * P * P >= 65536) return fail("%s: num_levels * num_points^2 must be < 65536", who);
    if (R == 0) return 0;
    if (!value || !level_hw || !level_start || !level_hw_host || !loc || !attn || !out || !map_range)
        return fail("%s: null pointer argument", who);
    if (!aligned16(value) || !aligned16(loc) || !aligned16(attn) || !aligned16(out))
        return fail("%s: device pointers must be 16-byte aligned", who);
    if ((long long)S * M * 32 >= (1ll << 31)) return fail("%s: one value map exceeds 2^31 elements", who);
    cudaStream_t st = (cudaStream_t)stream;
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const int chunks = sms;                        // persistent: one CTA per SM
    if ((value_dtype != BEVF_DTYPE_F32 && value_dtype != BEVF_DTYPE_BF16) ||
        (out_dtype != BEVF_DTYPE_F32 && out_dtype != BEVF_DTYPE_BF16))
        return fail("%s: fp32 or bf16 only (fp16 runs on bevf_msda_rows_forward)", who);
    const bool vb = value_dtype == BEVF_DTYPE_BF16, ob = out_dtype == BEVF_DTYPE_BF16;
    int e;
    if (vb && ob) e = launch_staged<bf16, bf16>(who, value, level_hw, level_start, level_hw_host, loc, attn, out, map_range, B, S, M, L, P, chunks, st);
    else if (vb && !ob) e = launch_staged<bf16, float>(who, value, level_hw, level_start, level_hw_host, loc, attn, out, map_range, B, S, M, L, P, chunks, st);
    else if (!vb && !ob) e = launch_staged<float, float>(who, value, level_hw, level_start, level_hw_host, loc, attn, out, map_range, B, S, M, L, P, chunks, st);
    else return fail("%s: fp32 value with bf16 output is not supported", who);
    if (e == -1) return fail("%s: no pyramid level fits the staging buffer (use bevf_msda_rows_forward)", who);
    return e;
}
