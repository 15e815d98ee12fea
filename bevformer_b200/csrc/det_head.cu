// Detection head of BEVFormer on the device: the classification / regression branch MLPs of every decoder level in
// one launch, and the NMS-free top-k decode of the last level in one launch.
//
//   bevf_det_branches_forward   BEVFormerHead.forward after the transformer (dense_heads/bevformer_head.py:171-203):
//                               per level l, cls_branches[l](hs[l]) and reg_branches[l](hs[l]) followed by the
//                               inverse-sigmoid / sigmoid / pc_range arithmetic on the box centres
//   bevf_nms_free_decode        NMSFreeCoder.decode (core/bbox/coders/nms_free_coder.py:40-121) with util.py's
//                               denormalize_bbox, and optionally get_bboxes' z -= h / 2 (bevformer_head.py:500)
//
// Branch kernel: one CTA (one warpgroup) per (level, branch, 64-row tile).  The 64 x 256 activation tile stays in
// shared memory across the branch's three GEMMs; each GEMM stages its (N x 256) weight from L2 into a SWIZZLE_128B
// K-major tile (fp32 weights are rounded to the activation type here) and runs m64nNk16 wgmmas, N = 256 for the
// hidden layers and 16 for the last one.  Epilogue in registers: bias, LayerNorm over the 256 columns (cls branch:
// fp32 statistics from a quad shuffle, the 4 lanes of a row hold its 256 columns), ReLU, rounded to the storage type
// and written back as the next GEMM's A operand.
#include "wgmma.cuh"

namespace bevf {

constexpr int kDhThreads = 128;                // one warpgroup
constexpr int kDhRows = 64;
constexpr int kDhC = 256;
constexpr int kDhMaxLevels = 8;
constexpr int kDhOut = 16;                     // padded width of the last GEMM
constexpr int kDhAChunk = kDhRows * 128;       // 64 rows x 64 K-elements (128 B) of the activation tile
constexpr int kDhSmem = 1024 + kDhRows * kDhC * 2 + kDhC * kDhC * 2;
// per level: cls W0 b0 g0 be0 W1 b1 g1 be1 W2 b2, reg W0 b0 W1 b1 W2 b2
constexpr int kDhPtrsPerLevel = 16;

struct DetBranchParams {
    const void *p[kDhMaxLevels][kDhPtrsPerLevel];
    const void *x;                 // decoder states (L, nq, bs, C), strides sL / sQ / sB elements, channels contiguous
    long long sL, sQ, sB;
    const void *ref0;              // (bs, nq, 3)
    const void *refs;              // (L, bs, nq, 3): level l > 0 reads refs[l - 1]
    int ref_dt;
    void *cls_out;                 // (L, bs, nq, ncls)
    void *box_out;                 // (L, bs, nq, 10)
    int L, bs, nq, ncls, tiles;
    float eps;
    float scale[3], offset[3];     // pc_range: x, y, z -> value * scale + offset
};

template <typename TP> __device__ __forceinline__ float ldp(const void *p, int i) {
    if constexpr (std::is_same<TP, float>::value) return reinterpret_cast<const float *>(p)[i];
    else return St16<TP>::to_f(reinterpret_cast<const TP *>(p)[i]);
}

__device__ __forceinline__ float ld_dt(const void *p, int dt, long long i) {
    if (dt == BEVF_DTYPE_BF16) return __bfloat162float(reinterpret_cast<const bf16 *>(p)[i]);
    if (dt == BEVF_DTYPE_F16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
    return reinterpret_cast<const float *>(p)[i];
}

template <typename T> __device__ __forceinline__ float rnd(float v) { return St16<T>::to_f(St16<T>::from_f(v)); }

// a Linear bias: fp32 parameters reach the kernel under autocast, whose Linear rounds the bias to the storage type
// as it does the weight (LayerNorm's gamma / beta stay fp32 there: autocast runs layer_norm in fp32)
template <typename T, typename TP> __device__ __forceinline__ float ld_bias(const void *p, int i) {
    const float v = ldp<TP>(p, i);
    return std::is_same<TP, float>::value ? rnd<T>(v) : v;
}

// byte offset of the 16-byte unit (row, k / 8) of a K-major SWIZZLE_128B operand with `rows` rows per 64-wide K chunk
__device__ __forceinline__ uint32_t sw_off(int row, int k, int rows) {
    return (uint32_t)((k >> 6) * rows * 128 + row * 128 + ((((k >> 3) & 7) ^ (row & 7)) << 4));
}

// W (n_rows x 256, row-major in TP) -> K-major swizzled tile of `rows` rows in T; rows past n_rows are zeros
template <typename T, typename TP>
__device__ __forceinline__ void stage_weight(uint8_t *sw, const void *w, int n_rows, int rows) {
    const int units = rows * (kDhC / 8);
    for (int u = threadIdx.x; u < units; u += kDhThreads) {
        const int r = u >> 5, k = (u & 31) * 8;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (r < n_rows) {
            if constexpr (std::is_same<TP, float>::value) {
                const float4 a = __ldg(reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(w) + (long long)r * kDhC + k));
                const float4 b = __ldg(reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(w) + (long long)r * kDhC + k) + 1);
                v = make_uint4(St16<T>::pack(a.x, a.y), St16<T>::pack(a.z, a.w), St16<T>::pack(b.x, b.y),
                               St16<T>::pack(b.z, b.w));
            } else {
                v = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const TP *>(w) + (long long)r * kDhC + k));
            }
        }
        *reinterpret_cast<uint4 *>(sw + sw_off(r, k, rows)) = v;
    }
}

// make the generic-proxy shared-memory stores above visible to the wgmma (async proxy) of every warp
__device__ __forceinline__ void smem_to_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}

template <int N, typename T>
__device__ __forceinline__ void tile_gemm(float (&d)[N / 2], uint32_t sa, uint32_t sw) {
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint64_t da = smem_desc_sw128(sa + (uint32_t)(kc * kDhAChunk + kk * 32), 0);
            const uint64_t db = smem_desc_sw128(sw + (uint32_t)(kc * N * 128 + kk * 32), 0);
            Wgmma<N, 0, 0, T>::run(d, da, db, (kc | kk) != 0);
        }
    wgmma_commit();
    wgmma_wait0();
    fence_regs(d);
}

// mmdet's inverse_sigmoid (models/utils/transformer.py, eps 1e-5) in fp32; log evaluated in double
__device__ __forceinline__ float inverse_sigmoid_f(float x) {
    x = fminf(fmaxf(x, 0.f), 1.f);
    const float x1 = fmaxf(x, 1e-5f), x2 = fmaxf(__fsub_rn(1.f, x), 1e-5f);
    return (float)log((double)__fdiv_rn(x1, x2));
}
__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, exp_rn(-x))); }

template <typename T, typename TP>
__global__ void __launch_bounds__(kDhThreads, 1) det_branches_kernel(const __grid_constant__ DetBranchParams p) {
    extern __shared__ uint8_t dh_smem_raw[];
    uint8_t *sa = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(dh_smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sw = sa + kDhRows * kDhC * 2;
    const int tile = blockIdx.x % p.tiles;
    const int branch = (blockIdx.x / p.tiles) & 1;          // 0: cls, 1: reg
    const int lvl = blockIdx.x / (2 * p.tiles);
    const int rows = p.bs * p.nq;
    const int row0 = tile * kDhRows;
    const void *const *pp = p.p[lvl] + (branch ? 10 : 0);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // the activation tile: states row (b, q) of level lvl, zero rows past the end
    for (int u = tid; u < kDhRows * (kDhC / 8); u += kDhThreads) {
        const int r = u >> 5, k = (u & 31) * 8, gr = row0 + r;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (gr < rows) {
            const int b = gr / p.nq, q = gr - b * p.nq;
            v = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const T *>(p.x) + lvl * p.sL + q * p.sQ +
                                                      b * p.sB + k));
        }
        *reinterpret_cast<uint4 *>(sa + sw_off(r, k, kDhRows)) = v;
    }
    const uint32_t sa_u = smem_u32(sa), sw_u = smem_u32(sw);
    const int rloc[2] = {16 * warp + (lane >> 2), 16 * warp + (lane >> 2) + 8};

    // two hidden layers: Linear (+ LayerNorm in the cls branch) + ReLU
#pragma unroll 1
    for (int layer = 0; layer < 2; ++layer) {
        const void *w = pp[branch ? 2 * layer : 4 * layer];
        const void *bias = pp[branch ? 2 * layer + 1 : 4 * layer + 1];
        stage_weight<T, TP>(sw, w, kDhC, kDhC);
        smem_to_async();
        float d[128];
        tile_gemm<256, T>(d, sa_u, sw_u);
        __syncthreads();                                     // every warp's wgmmas have read sa / sw
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + 2 * (lane & 3) + e;
                    float v = rnd<T>(__fadd_rn(d[4 * j + 2 * h + e], ld_bias<T, TP>(bias, col)));   // Linear output
                    d[4 * j + 2 * h + e] = v;
                    s += v;
                }
            if (!branch) {                                   // LayerNorm, fp32 statistics
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                const float mean = s * (1.f / kDhC);
                float var = 0.f;
#pragma unroll
                for (int j = 0; j < 32; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float c = d[4 * j + 2 * h + e] - mean;
                        var = fmaf(c, c, var);
                    }
                var += __shfl_xor_sync(0xffffffffu, var, 1);
                var += __shfl_xor_sync(0xffffffffu, var, 2);
                const float rstd = __frsqrt_rn(__fadd_rn(var * (1.f / kDhC), p.eps));
                const void *g = pp[4 * layer + 2], *be = pp[4 * layer + 3];
#pragma unroll
                for (int j = 0; j < 32; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * j + 2 * (lane & 3) + e;
                        const float c = __fsub_rn(d[4 * j + 2 * h + e], mean) * rstd;
                        d[4 * j + 2 * h + e] = rnd<T>(fmaf(c, ldp<TP>(g, col), ldp<TP>(be, col)));
                    }
            }
            const int r = rloc[h];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int col = 8 * j + 2 * (lane & 3);
                const uint32_t v = St16<T>::pack(fmaxf(d[4 * j + 2 * h], 0.f), fmaxf(d[4 * j + 2 * h + 1], 0.f));
                *reinterpret_cast<uint32_t *>(sa + sw_off(r, col, kDhRows) + (col & 7) * 2) = v;
            }
        }
    }

    // last Linear (N padded to 16), then the logits / the box tail
    const int nout = branch ? 10 : p.ncls;
    stage_weight<T, TP>(sw, pp[branch ? 4 : 8], nout, kDhOut);
    smem_to_async();
    float d[8];
    tile_gemm<kDhOut, T>(d, sa_u, sw_u);
    const void *bias = pp[branch ? 5 : 9];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gr = row0 + rloc[h];
        if (gr >= rows) continue;
        const int b = gr / p.nq, q = gr - b * p.nq;
        const long long orow = ((long long)lvl * p.bs + b) * p.nq + q;
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = 8 * j + 2 * (lane & 3) + e;
                if (col >= nout) continue;
                float v = __fadd_rn(d[4 * j + 2 * h + e], ld_bias<T, TP>(bias, col));
                if (!branch) {
                    reinterpret_cast<T *>(p.cls_out)[orow * p.ncls + col] = St16<T>::from_f(v);
                    continue;
                }
                if (col == 0 || col == 1 || col == 4) {
                    const int c = col == 4 ? 2 : col;
                    const float ref = lvl == 0 ? ld_dt(p.ref0, p.ref_dt, ((long long)b * p.nq + q) * 3 + c)
                                               : ld_dt(p.refs, p.ref_dt,
                                                       ((((long long)lvl - 1) * p.bs + b) * p.nq + q) * 3 + c);
                    v = sigmoid_f(__fadd_rn(v, inverse_sigmoid_f(ref)));
                    v = __fadd_rn(__fmul_rn(v, p.scale[c]), p.offset[c]);
                }
                reinterpret_cast<T *>(p.box_out)[orow * 10 + col] = St16<T>::from_f(v);
            }
    }
}

template <typename T, typename TP> static int launch_branches(const DetBranchParams &p, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(det_branches_kernel<T, TP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDhSmem) !=
            cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory", "bevf_det_branches_forward");
        }
        attr = true;
    }
    det_branches_kernel<T, TP><<<p.L * 2 * p.tiles, kDhThreads, kDhSmem, st>>>(p);
    return check_launch("bevf_det_branches_forward");
}

// ================================================================================================================
// NMS-free decode: one CTA per sample.
//   scores   sigmoid of the widened logits, 1 / (1 + expf(-x)) with libdevice's expf and an IEEE division
//            (torch.sigmoid's formula; --use_fast_math would otherwise approximate both), subnormal results kept
//            (sigmoid_bits)
//   top-k    radix select (8 passes of 8 bits) on the unique 64-bit key (score bits << 32 | ~flat index), so the
//            k selected are the k largest scores with ties taken by ascending flat index, then a bitonic sort of
//            the k keys: output order is (score descending, flat index ascending)
//   decode   label = idx % ncls, query = idx / ncls, denormalize_bbox; score threshold as the reference's loop;
//            post-centre-range mask; stable compaction into (max_num) slots, the rest zero
// ================================================================================================================
constexpr int kNdThreads = 1024;

// libdevice's expf, the one torch.sigmoid's fp32 kernel calls (the library's --use_fast_math would turn a plain expf
// into the approximate __expf); same algorithm, so the scores -- and the ranking -- equal torch.sigmoid's
extern "C" __device__ float __nv_expf(float);

// The fp32 bits of torch.sigmoid(x) = 1 / (1 + expf(-x)).  For x below about -87.3 the IEEE quotient is subnormal,
// which the library's -ftz=true would flush to zero: those are rounded onto the subnormal grid (2^-149 steps) from
// the double quotient and returned as bits, so they still rank by score.  expf(-x) = inf gives 0, as in torch.
__device__ __forceinline__ uint32_t sigmoid_bits(float x) {
    const float den = __fadd_rn(1.f, __nv_expf(-x));
    if (den < 0x1p126f) return __float_as_uint(__fdiv_rn(1.f, den));
    return (uint32_t)rint(__ddiv_rn(1.0, (double)den) * 0x1p149);
}

struct DecodeParams {
    const void *cls;
    const void *box;
    int cls_dt, box_dt;
    int nq, ncls, k, k_pow2;
    float pcr[6];
    int has_thr;                   // threshold given and non-zero (the reference's `if self.score_threshold:`)
    double thr;
    int z_shift;
    float *bboxes;                 // (bs, k, 9)
    float *scores;                 // (bs, k)
    long long *labels;             // (bs, k)
    int *num;                      // (bs)
};

__device__ __forceinline__ unsigned long long dec_key(const uint32_t *keys, int i) {
    return ((unsigned long long)keys[i] << 32) | (0xffffffffu - (uint32_t)i);
}

__global__ void __launch_bounds__(kNdThreads) nms_free_decode_kernel(const __grid_constant__ DecodeParams p) {
    extern __shared__ uint8_t nd_smem_raw[];
    unsigned long long *sel = reinterpret_cast<unsigned long long *>(nd_smem_raw);
    uint32_t *keys = reinterpret_cast<uint32_t *>(sel + p.k_pow2);
    __shared__ int hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_krem, s_cnt, s_base, s_mode;
    __shared__ float s_thr;
    __shared__ int warp_tot[kNdThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = p.nq * p.ncls;
    const long long cls0 = (long long)b * n;
    for (int i = tid; i < n; i += kNdThreads) {
        keys[i] = sigmoid_bits(ld_dt(p.cls, p.cls_dt, cls0 + i));
    }
    if (tid == 0) { s_prefix = 0ull; s_krem = p.k; s_cnt = 0; }
    unsigned long long mask = 0ull;
#pragma unroll 1
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += kNdThreads) hist[i] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        for (int i = tid; i < n; i += kNdThreads) {
            const unsigned long long key = dec_key(keys, i);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xff], 1);
        }
        __syncthreads();
        if (warp == 0) {                                    // lane l owns digits 255 - 8 l .. 248 - 8 l
            int c[8], tot = 0;
#pragma unroll
            for (int t = 0; t < 8; ++t) { c[t] = hist[255 - 8 * lane - t]; tot += c[t]; }
            int incl = tot;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const int krem = s_krem;
            const unsigned hit = __ballot_sync(0xffffffffu, incl >= krem);
            if (lane == __ffs(hit) - 1) {
                int above = incl - tot;
                int t = 0;
                while (above + c[t] < krem) above += c[t++];
                s_krem = krem - above;
                s_prefix = prefix | ((unsigned long long)(255 - 8 * lane - t) << shift);
            }
        }
        mask |= 0xffull << shift;
        __syncthreads();
    }
    const unsigned long long kth = s_prefix;                // the k-th largest key: exactly k keys are >= kth
    for (int i = tid; i < n; i += kNdThreads) {
        const unsigned long long key = dec_key(keys, i);
        if (key >= kth) sel[atomicAdd(&s_cnt, 1)] = key;
    }
    for (int i = p.k + tid; i < p.k_pow2; i += kNdThreads) sel[i] = 0ull;
    __syncthreads();
    for (int size = 2; size <= p.k_pow2; size <<= 1)        // bitonic sort, descending
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < p.k_pow2; i += kNdThreads) {
                const int j = i ^ stride;
                if (j > i) {
                    const unsigned long long a = sel[i], c = sel[j];
                    const bool desc = (i & size) == 0;
                    if (desc ? a < c : a > c) { sel[i] = c; sel[j] = a; }
                }
            }
            __syncthreads();
        }
    if (tid == 0) {
        // score threshold (nms_free_coder.py:65-73): the first test is strict, the decayed ones are >= against the
        // threshold multiplied by 0.9 in double and compared in fp32; below 0.01 everything passes (> -1).  The
        // loop stops at the first threshold some candidate passes, i.e. at the first one the top score passes.
        int mode = 0;                                       // 0: no mask, 1: score > t, 2: score >= t, 3: score > -1
        float t = 0.f;
        if (p.has_thr) {
            const float top = __uint_as_float((uint32_t)(sel[0] >> 32));
            double tmp = p.thr;
            mode = 1; t = (float)tmp;
            if (!(top > t)) {
                for (;;) {
                    tmp *= 0.9;
                    if (tmp < 0.01) { mode = 3; t = -1.f; break; }
                    if (top >= (float)tmp) { mode = 2; t = (float)tmp; break; }
                }
            }
        }
        s_mode = mode; s_thr = t; s_base = 0;
    }
    __syncthreads();
    const int mode = s_mode;
    const float thr = s_thr;
    const long long out0 = (long long)b * p.k;
#pragma unroll 1
    for (int c0 = 0; c0 < p.k; c0 += kNdThreads) {
        const int t = c0 + tid;
        bool keep = false;
        float bx[9];
        float score = 0.f;
        int label = 0;
        if (t < p.k) {
            const unsigned long long key = sel[t];
            score = __uint_as_float((uint32_t)(key >> 32));
            const int idx = (int)(0xffffffffu - (uint32_t)key);
            label = idx % p.ncls;
            const long long row = ((long long)b * p.nq + idx / p.ncls) * 10;
            float v[10];
#pragma unroll
            for (int c = 0; c < 10; ++c) v[c] = ld_dt(p.box, p.box_dt, row + c);
            bx[0] = v[0]; bx[1] = v[1]; bx[2] = v[4];
            bx[3] = exp_rn(v[2]); bx[4] = exp_rn(v[3]); bx[5] = exp_rn(v[5]);
            bx[6] = (float)atan2((double)v[6], (double)v[7]);
            bx[7] = v[8]; bx[8] = v[9];
            keep = true;
#pragma unroll
            for (int c = 0; c < 3; ++c) keep = keep && bx[c] >= p.pcr[c] && bx[c] <= p.pcr[3 + c];
            if (mode == 1 || mode == 3) keep = keep && score > thr;
            else if (mode == 2) keep = keep && score >= thr;
            if (p.z_shift) bx[2] = __fsub_rn(bx[2], bx[5] * 0.5f);
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[warp] = __popc(ballot);
        __syncthreads();
        if (warp == 0) {
            const int v = warp_tot[lane];
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += u;
            }
            warp_tot[lane] = incl - v;
        }
        __syncthreads();
        const int base = s_base;
        if (keep) {
            const long long o = out0 + base + warp_tot[warp] + __popc(ballot & ((1u << lane) - 1u));
#pragma unroll
            for (int c = 0; c < 9; ++c) p.bboxes[o * 9 + c] = bx[c];
            p.scores[o] = score;
            p.labels[o] = label;
        }
        __syncthreads();
        if (tid == kNdThreads - 1) s_base = base + warp_tot[warp] + __popc(ballot);
        __syncthreads();
    }
    const int num = s_base;
    for (int i = num + tid; i < p.k; i += kNdThreads) {
#pragma unroll
        for (int c = 0; c < 9; ++c) p.bboxes[(out0 + i) * 9 + c] = 0.f;
        p.scores[out0 + i] = 0.f;
        p.labels[out0 + i] = 0;
    }
    if (tid == 0) p.num[b] = num;
}

static bool dt_ok(int dt) { return dt == BEVF_DTYPE_F32 || dt == BEVF_DTYPE_BF16 || dt == BEVF_DTYPE_F16; }

}  // namespace bevf

using namespace bevf;

#define BEVF_REQUIRE(cond, who, msg) do { if (!(cond)) return fail("%s: " msg, who); } while (0)

extern "C" int64_t bevf_nms_free_decode_smem_bytes(int nq, int ncls, int max_num) {
    int p2 = 1;
    while (p2 < max_num) p2 <<= 1;
    return (int64_t)p2 * 8 + (int64_t)nq * ncls * 4;
}

extern "C" int bevf_det_branches_forward(const void *x, int64_t stride_l, int64_t stride_q, int64_t stride_b,
                                         int dtype, const void *ref0, const void *refs, int ref_dtype,
                                         const void *const *params, int param_dtype, void *cls_out, void *box_out,
                                         int L, int bs, int nq, int C, int ncls, int code_size, float ln_eps,
                                         const double *pc_range, void *stream) {
    const char *who = "bevf_det_branches_forward";
    BEVF_REQUIRE(L > 0 && L <= kDhMaxLevels && bs > 0 && nq > 0, who, "bad dimension (1 <= L <= 8)");
    BEVF_REQUIRE(C == kDhC, who, "embed_dims must be 256");
    BEVF_REQUIRE(ncls > 0 && ncls <= kDhOut && code_size == 10, who, "need 1 <= num_classes <= 16 and code_size == 10");
    BEVF_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F16, who, "activations must be bf16 or fp16");
    BEVF_REQUIRE(param_dtype == dtype || param_dtype == BEVF_DTYPE_F32, who,
                 "parameters must be in the activation dtype or fp32");
    BEVF_REQUIRE(dt_ok(ref_dtype), who, "unsupported reference-point dtype");
    BEVF_REQUIRE(x && ref0 && (L == 1 || refs) && params && cls_out && box_out && pc_range, who, "null pointer argument");
    BEVF_REQUIRE(aligned16(x) && stride_l % 8 == 0 && stride_q % 8 == 0 && stride_b % 8 == 0, who,
                 "decoder states must be 16-byte aligned with strides that are multiples of 8 elements");
    BEVF_REQUIRE((long long)bs * nq <= (1LL << 30), who, "too many rows");
    DetBranchParams p{};
    for (int l = 0; l < L; ++l)
        for (int i = 0; i < kDhPtrsPerLevel; ++i) {
            p.p[l][i] = params[l * kDhPtrsPerLevel + i];
            BEVF_REQUIRE(p.p[l][i] != nullptr, who, "null parameter pointer");
            const bool weight = i == 0 || i == 4 || i == 8 || i == 10 || i == 12 || i == 14;
            BEVF_REQUIRE(!weight || aligned16(p.p[l][i]), who, "weights must be 16-byte aligned");
        }
    p.x = x; p.sL = stride_l; p.sQ = stride_q; p.sB = stride_b;
    p.ref0 = ref0; p.refs = refs; p.ref_dt = ref_dtype;
    p.cls_out = cls_out; p.box_out = box_out;
    p.L = L; p.bs = bs; p.nq = nq; p.ncls = ncls; p.tiles = (bs * nq + kDhRows - 1) / kDhRows;
    p.eps = ln_eps;
    for (int c = 0; c < 3; ++c) {
        const int lo = c, hi = c + 3;
        p.scale[c] = (float)(pc_range[hi] - pc_range[lo]);
        p.offset[c] = (float)pc_range[lo];
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_BF16)
        return param_dtype == dtype ? launch_branches<bf16, bf16>(p, st) : launch_branches<bf16, float>(p, st);
    return param_dtype == dtype ? launch_branches<__half, __half>(p, st) : launch_branches<__half, float>(p, st);
}

extern "C" int bevf_nms_free_decode(const void *cls, int cls_dtype, const void *box, int box_dtype, int bs, int nq,
                                    int ncls, int code_size, int max_num, const float *post_center_range,
                                    int has_threshold, double score_threshold, int z_shift, float *bboxes,
                                    float *scores, int64_t *labels, int *num, void *stream) {
    const char *who = "bevf_nms_free_decode";
    BEVF_REQUIRE(bs > 0 && nq > 0 && ncls > 0 && code_size == 10, who, "bad dimension (code_size must be 10)");
    BEVF_REQUIRE(max_num > 0 && (long long)max_num <= (long long)nq * ncls, who, "need 1 <= max_num <= nq * ncls");
    BEVF_REQUIRE(dt_ok(cls_dtype) && dt_ok(box_dtype), who, "unsupported dtype code");
    BEVF_REQUIRE(cls && box && post_center_range && bboxes && scores && labels && num, who, "null pointer argument");
    const int64_t smem = bevf_nms_free_decode_smem_bytes(nq, ncls, max_num);
    BEVF_REQUIRE(smem <= 200 * 1024, who, "nq * num_classes too large for the shared-memory top-k");
    DecodeParams p{};
    p.cls = cls; p.box = box; p.cls_dt = cls_dtype; p.box_dt = box_dtype;
    p.nq = nq; p.ncls = ncls; p.k = max_num;
    p.k_pow2 = 1;
    while (p.k_pow2 < max_num) p.k_pow2 <<= 1;
    for (int c = 0; c < 6; ++c) p.pcr[c] = post_center_range[c];
    p.has_thr = has_threshold; p.thr = score_threshold; p.z_shift = z_shift;
    p.bboxes = bboxes; p.scores = scores; p.labels = reinterpret_cast<long long *>(labels); p.num = num;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(nms_free_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) !=
            cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory", who);
        }
        attr = true;
    }
    nms_free_decode_kernel<<<bs, kNdThreads, (size_t)smem, (cudaStream_t)stream>>>(p);
    return check_launch(who);
}
