// Block-diagonal ("grouped") softmax attention for head_dim 32: the self-attention of Group DETR's decoder
// (GroupMultiheadAttention, projects/mmdet3d_plugin/bevformer/modules/group_attention.py:117-162), where each of
// `groups` equal slices of the queries attends only to the same slice of the keys.
//
// Layout: Q, K, V are read in place from the in-projection output; element (token t, batch b, head h, channel c)
// of X lives at X + (t * bs + b) * ldx + h * 32 + c (sequence-first, any row stride that is a multiple of 8).
// Group g covers query tokens [g * Lq, (g + 1) * Lq) and key tokens [g * Lk, (g + 1) * Lk).
//
// Kernels (FlashAttention-2 structure, warp-level mma.sync m16n8k16 with fp32 accumulation; 4 warps x 16 rows):
//   attn_fwd      one CTA per (64 queries, head, batch * group); K/V tiles of 64 keys double-buffered through
//                 cp.async; online softmax in registers with exp2 and the scale folded in; P is rounded to the
//                 storage type as the A operand of P.V.  Writes O and the fp32 log-sum-exp per (b, g, h, query).
//   attn_bwd_dq   queries outer: D = rowsum(dO * O) for its rows (written for attn_bwd_dkv), then dQ = dS.K.
//   attn_bwd_dkv  keys outer: dV = Z^T.dO, dK = dS^T.Q with P recomputed from the log-sum-exp.
// Every output element is produced by exactly one thread in a fixed order: no atomics, so the gradients repeat bit
// for bit.  Measured alone at the V2 training shape (11 groups of 900, 8 x 32; H100 80GB HBM3, 700 W;
// tools/bench_group_attention.py) the three kernels take 65 / 93 / 98 us without dropout and 142 / 169 / 205 us with
// it: 17-26 % of their exp floor and 14-19 % of the dense bf16 tensor-core rate, so neither bounds them -- the
// tile loop (ldmatrix, barriers, mma.sync issue) does, and with dropout the Philox rounds.  They are about a quarter
// of the module's forward + backward there; the rest is the projections and host-side work.  A Hopper
// wgmma / TMA version is the way to take the kernels closer to the exp floor.
//
// Attention-probability dropout (nn.MultiheadAttention's `dropout`): keep(b, g, h, i, j) comes from Philox4x32-10
// keyed by seed + *seed_base with counter (j / 2, i / 2, (b * G + g) * H + h, 0), word 2 * (i & 1) + (j & 1) compared
// against p * 2^32.  Forward and both backward passes regenerate the same bits; nothing is stored.  The softmax
// normaliser is the sum of the undropped probabilities, as in torch.
#include "common.cuh"

namespace bevf {
namespace {

constexpr int kD = 32;         // head_dim
constexpr int kTile = 64;      // queries per CTA (fwd / dq) or keys per CTA (dkv), and the inner tile length
constexpr int kPad = 40;       // smem row pitch in elements: 80 bytes, so ldmatrix rows hit distinct banks
constexpr int kThreads = 128;  // 4 warps x 16 rows
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct AttnParams {
    const void *q, *k, *v, *o, *dout;
    void *out, *dq, *dk, *dv;
    float *lse, *delta;
    long long ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;
    int bs, heads, groups, lq, lk;
    float scale, scale_log2, drop_p, inv_keep;
    uint32_t drop_thr;
    unsigned long long seed;
    const unsigned long long *seed_base;
};

template <typename T> struct Mma;
template <> struct Mma<bf16> {
    static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
        __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t *>(&v);
    }
};
template <> struct Mma<__half> {
    static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
        __half2 v = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t *>(&v);
    }
};

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void *p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void *p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr(smem)), "l"(gmem),
                 "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// rows [r0, r0 + 64) of one (b, h) slice of a group starting at token tok0, zero past the group's length L
template <typename T>
__device__ __forceinline__ void load_tile(T (*s)[kPad], const T *x, long long ld, int bs, int b, int h, int tok0,
                                          int r0, int L) {
#pragma unroll
    for (int c = threadIdx.x; c < kTile * 4; c += kThreads) {
        const int r = c >> 2, part = c & 3;
        const bool ok = r0 + r < L;
        const T *src = ok ? x + ((long long)(tok0 + r0 + r) * bs + b) * ld + h * kD + part * 8 : x;
        cp_async16(&s[r][part * 8], src, ok);
    }
}

// A fragments (16 rows x 32 channels, two k-steps) of rows [row0, row0 + 16) of a tile
template <typename T>
__device__ __forceinline__ void load_a(uint32_t (&f)[2][4], const T (*s)[kPad], int row0, int lane) {
#pragma unroll
    for (int kc = 0; kc < 2; ++kc) ldsm_x4(f[kc], &s[row0 + (lane & 15)][kc * 16 + (lane >> 4) * 8]);
}

// acc[n] (16 x 8, n = 0..7) += A (16 x 32) . X[rows 8n..8n+7]^T  with X a 64 x 32 tile (X read row-major = B col-major)
template <typename T>
__device__ __forceinline__ void mma_abt(float (&acc)[8][4], const uint32_t (&a)[2][4], const T (*x)[kPad], int lane) {
#pragma unroll
    for (int n = 0; n < 8; ++n) {
        uint32_t b[4];
        ldsm_x4(b, &x[n * 8 + (lane & 7)][(lane >> 3) * 8]);
        Mma<T>::run(acc[n], a[0], b[0], b[1]);
        Mma<T>::run(acc[n], a[1], b[2], b[3]);
    }
}

// acc[c] (16 x 8, c = 0..3 channel tiles) += P (16 x 64, A fragments per 16-column step) . X (64 x 32 tile)
template <typename T>
__device__ __forceinline__ void mma_ab(float (&acc)[4][4], const uint32_t (&p)[4][4], const T (*x)[kPad], int lane) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int nc = 0; nc < 2; ++nc) {
            uint32_t b[4];
            ldsm_x4_t(b, &x[kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][nc * 16 + (lane >> 4) * 8]);
            Mma<T>::run(acc[nc * 2], p[kk], b[0], b[1]);
            Mma<T>::run(acc[nc * 2 + 1], p[kk], b[2], b[3]);
        }
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ uint32_t word_of(const uint4 &w, int idx) {
    return idx == 0 ? w.x : idx == 1 ? w.y : idx == 2 ? w.z : w.w;
}

__device__ __forceinline__ uint2 drop_key(const AttnParams &p) {
    unsigned long long s = p.seed + (p.seed_base ? *p.seed_base : 0ull);
    return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

// One Philox call yields the 2 x 2 block (i, i+1) x (j, j+1), i and j even.  A thread holds two rows 8 apart of a 2-wide
// column pair, and the lane 4 away (the next row) holds the other row of each block: each of the two lanes draws one
// block and hands the partner the half it needs, so every call's four words are used.

// keep bits of (i0, j), (i0, j+1), (i0+8, j), (i0+8, j+1): rows = queries (forward and dQ layouts), j even
__device__ __forceinline__ void keep_rows4(uint2 key, uint32_t bgh, int i0, int j, uint32_t thr, bool (&k)[4]) {
    const bool odd = i0 & 1;
    const int ib = odd ? i0 + 7 : i0;                       // even row of the block this lane draws
    const uint4 w = philox4x32_10(make_uint4((uint32_t)j >> 1, (uint32_t)ib >> 1, bgh, 0u), key);
    const uint32_t m0 = odd ? w.z : w.x, m1 = odd ? w.w : w.y;  // this lane's row of the block
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, odd ? w.x : w.z, 4);
    const uint32_t r1 = __shfl_xor_sync(0xffffffffu, odd ? w.y : w.w, 4);
    k[0] = (odd ? r0 : m0) >= thr;
    k[1] = (odd ? r1 : m1) >= thr;
    k[2] = (odd ? m0 : r0) >= thr;
    k[3] = (odd ? m1 : r1) >= thr;
}
// keep bits of (i, j0), (i+1, j0), (i, j0+8), (i+1, j0+8): rows = keys (dK / dV layout), i even
__device__ __forceinline__ void keep_cols4(uint2 key, uint32_t bgh, int i, int j0, uint32_t thr, bool (&k)[4]) {
    const bool odd = j0 & 1;
    const int jb = odd ? j0 + 7 : j0;
    const uint4 w = philox4x32_10(make_uint4((uint32_t)jb >> 1, (uint32_t)i >> 1, bgh, 0u), key);
    const uint32_t m0 = odd ? w.y : w.x, m1 = odd ? w.w : w.z;  // this lane's key of the block, queries i, i+1
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, odd ? w.x : w.y, 4);
    const uint32_t r1 = __shfl_xor_sync(0xffffffffu, odd ? w.z : w.w, 4);
    k[0] = (odd ? r0 : m0) >= thr;
    k[1] = (odd ? r1 : m1) >= thr;
    k[2] = (odd ? m0 : r0) >= thr;
    k[3] = (odd ? m1 : r1) >= thr;
}

template <typename T>
__device__ __forceinline__ void store_rows(const float (&acc)[4][4], float mul0, float mul1, T *x, long long ld, int bs,
                                           int b, int h, int tok0, int row, int L, int lane) {
    const int tq = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int r = row + half * 8;
        if (r >= L) continue;
        const float m = half ? mul1 : mul0;
        T *dst = x + ((long long)(tok0 + r) * bs + b) * ld + h * kD + 2 * tq;
#pragma unroll
        for (int c = 0; c < 4; ++c)
            *reinterpret_cast<uint32_t *>(dst + c * 8) = Mma<T>::pack(acc[c][half * 2] * m, acc[c][half * 2 + 1] * m);
    }
}

template <typename T, bool kDrop>
__global__ void __launch_bounds__(kThreads) attn_fwd(const AttnParams p) {
    __shared__ __align__(128) T qs[kTile][kPad];
    __shared__ __align__(128) T ks[2][kTile][kPad];
    __shared__ __align__(128) T vs[2][kTile][kPad];
    const int b = blockIdx.z / p.groups, g = blockIdx.z % p.groups, h = blockIdx.y;
    const int m0 = blockIdx.x * kTile, qtok = g * p.lq, ktok = g * p.lk;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gr = lane >> 2, tq = lane & 3;
    const T *Q = (const T *)p.q, *K = (const T *)p.k, *V = (const T *)p.v;
    const uint32_t bgh = (uint32_t)(blockIdx.z * p.heads + h);
    uint2 key = make_uint2(0u, 0u);
    if (kDrop) key = drop_key(p);

    load_tile(qs, Q, p.ldq, p.bs, b, h, qtok, m0, p.lq);
    load_tile(ks[0], K, p.ldk, p.bs, b, h, ktok, 0, p.lk);
    load_tile(vs[0], V, p.ldv, p.bs, b, h, ktok, 0, p.lk);
    cp_commit();

    const int ntiles = (p.lk + kTile - 1) / kTile;
    uint32_t qf[2][4];
    float o[4][4] = {};
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
    const int i0 = m0 + warp * 16 + gr;        // this thread's rows i0 and i0 + 8 (group-local)
    for (int t = 0; t < ntiles; ++t) {
        if (t + 1 < ntiles) {
            load_tile(ks[(t + 1) & 1], K, p.ldk, p.bs, b, h, ktok, (t + 1) * kTile, p.lk);
            load_tile(vs[(t + 1) & 1], V, p.ldv, p.bs, b, h, ktok, (t + 1) * kTile, p.lk);
            cp_commit();
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        if (t == 0) load_a(qf, qs, warp * 16, lane);
        float s[8][4] = {};
        mma_abt(s, qf, ks[t & 1], lane);
        const int j0 = t * kTile;
        if (j0 + kTile > p.lk) {
#pragma unroll
            for (int n = 0; n < 8; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (j0 + n * 8 + 2 * tq + (e & 1) >= p.lk) s[n][e] = -INFINITY;
        }
        float mx[2] = {mrow[0], mrow[1]};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            mx[0] = fmaxf(mx[0], fmaxf(s[n][0], s[n][1]));
            mx[1] = fmaxf(mx[1], fmaxf(s[n][2], s[n][3]));
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float alpha = exp2f((mrow[r] - mx[r]) * p.scale_log2);
            mrow[r] = mx[r];
            lrow[r] *= alpha;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                o[c][2 * r] *= alpha;
                o[c][2 * r + 1] *= alpha;
            }
        }
        const float msc0 = mx[0] * p.scale_log2, msc1 = mx[1] * p.scale_log2;
        uint32_t pa[4][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            float e0 = exp2f(fmaf(s[n][0], p.scale_log2, -msc0)), e1 = exp2f(fmaf(s[n][1], p.scale_log2, -msc0));
            float e2 = exp2f(fmaf(s[n][2], p.scale_log2, -msc1)), e3 = exp2f(fmaf(s[n][3], p.scale_log2, -msc1));
            lrow[0] += e0 + e1;
            lrow[1] += e2 + e3;
            if (kDrop) {
                const int j = j0 + n * 8 + 2 * tq;
                bool kp[4];
                keep_rows4(key, bgh, i0, j, p.drop_thr, kp);
                e0 = kp[0] ? e0 : 0.f;
                e1 = kp[1] ? e1 : 0.f;
                e2 = kp[2] ? e2 : 0.f;
                e3 = kp[3] ? e3 : 0.f;
            }
            pa[n >> 1][(n & 1) * 2] = Mma<T>::pack(e0, e1);
            pa[n >> 1][(n & 1) * 2 + 1] = Mma<T>::pack(e2, e3);
        }
        mma_ab(o, pa, vs[t & 1], lane);
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
        lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
    }
    const float keep = kDrop ? p.inv_keep : 1.f;
    store_rows(o, keep / lrow[0], keep / lrow[1], (T *)p.out, p.ldo, p.bs, b, h, qtok, i0, p.lq, lane);
    if (tq == 0) {
        float *lse = p.lse + (long long)bgh * p.lq;
        if (i0 < p.lq) lse[i0] = (mrow[0] * p.scale_log2 + log2f(lrow[0])) * kLn2;
        if (i0 + 8 < p.lq) lse[i0 + 8] = (mrow[1] * p.scale_log2 + log2f(lrow[1])) * kLn2;
    }
}

// queries outer: D = rowsum(dO * O) and dQ = scale * dS . K
template <typename T, bool kDrop>
__global__ void __launch_bounds__(kThreads) attn_bwd_dq(const AttnParams p) {
    __shared__ __align__(128) T qs[kTile][kPad];
    __shared__ __align__(128) T dos[kTile][kPad];
    __shared__ __align__(128) T ks[2][kTile][kPad];
    __shared__ __align__(128) T vs[2][kTile][kPad];
    __shared__ float lse_s[kTile], d_s[kTile];
    const int b = blockIdx.z / p.groups, g = blockIdx.z % p.groups, h = blockIdx.y;
    const int m0 = blockIdx.x * kTile, qtok = g * p.lq, ktok = g * p.lk;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gr = lane >> 2, tq = lane & 3;
    const T *Q = (const T *)p.q, *K = (const T *)p.k, *V = (const T *)p.v;
    const T *O = (const T *)p.o, *dO = (const T *)p.dout;
    const uint32_t bgh = (uint32_t)(blockIdx.z * p.heads + h);
    uint2 key = make_uint2(0u, 0u);
    if (kDrop) key = drop_key(p);

    load_tile(qs, Q, p.ldq, p.bs, b, h, qtok, m0, p.lq);
    load_tile(dos, dO, p.lddo, p.bs, b, h, qtok, m0, p.lq);
    load_tile(ks[0], K, p.ldk, p.bs, b, h, ktok, 0, p.lk);
    load_tile(vs[0], V, p.ldv, p.bs, b, h, ktok, 0, p.lk);
    cp_commit();
    {   // D for the tile's rows: two lanes per row, 16 channels each, fixed order
        const int r = threadIdx.x >> 1, part = threadIdx.x & 1, i = m0 + r;
        float d = 0.f, l = 0.f;
        if (i < p.lq) {
            const T *po = O + ((long long)(qtok + i) * p.bs + b) * p.ldo + h * kD + part * 16;
            const T *pd = dO + ((long long)(qtok + i) * p.bs + b) * p.lddo + h * kD + part * 16;
#pragma unroll
            for (int c = 0; c < 16; ++c) d = fmaf(float(po[c]), float(pd[c]), d);
            l = p.lse[(long long)bgh * p.lq + i] * kLog2e;
        }
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        if (part == 0) {
            d_s[r] = d;
            lse_s[r] = l;
            if (i < p.lq) p.delta[(long long)bgh * p.lq + i] = d;
        }
    }

    const int ntiles = (p.lk + kTile - 1) / kTile;
    uint32_t qf[2][4], dof[2][4];
    float dq[4][4] = {};
    float lse2[2], dd[2];
    const int rl = warp * 16 + gr, i0 = m0 + rl;
    for (int t = 0; t < ntiles; ++t) {
        if (t + 1 < ntiles) {
            load_tile(ks[(t + 1) & 1], K, p.ldk, p.bs, b, h, ktok, (t + 1) * kTile, p.lk);
            load_tile(vs[(t + 1) & 1], V, p.ldv, p.bs, b, h, ktok, (t + 1) * kTile, p.lk);
            cp_commit();
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        if (t == 0) {
            load_a(qf, qs, warp * 16, lane);
            load_a(dof, dos, warp * 16, lane);
            lse2[0] = lse_s[rl];
            lse2[1] = lse_s[rl + 8];
            dd[0] = d_s[rl];
            dd[1] = d_s[rl + 8];
        }
        float s[8][4] = {}, dp[8][4] = {};
        mma_abt(s, qf, ks[t & 1], lane);
        mma_abt(dp, dof, vs[t & 1], lane);
        const int j0 = t * kTile;
        uint32_t da[4][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            const int j = j0 + n * 8 + 2 * tq;
            bool kp[4] = {true, true, true, true};
            if (kDrop) {
                keep_rows4(key, bgh, i0, j, p.drop_thr, kp);
            }
            float ds[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pe = (j + (e & 1) < p.lk) ? exp2f(fmaf(s[n][e], p.scale_log2, -lse2[e >> 1])) : 0.f;
                const float dz = kDrop ? (kp[e] ? dp[n][e] * p.inv_keep : 0.f) : dp[n][e];
                ds[e] = pe * (dz - dd[e >> 1]);
            }
            da[n >> 1][(n & 1) * 2] = Mma<T>::pack(ds[0], ds[1]);
            da[n >> 1][(n & 1) * 2 + 1] = Mma<T>::pack(ds[2], ds[3]);
        }
        mma_ab(dq, da, ks[t & 1], lane);
        __syncthreads();
    }
    store_rows(dq, p.scale, p.scale, (T *)p.dq, p.lddq, p.bs, b, h, qtok, i0, p.lq, lane);
}

// keys outer: dV = Z^T . dO and dK = scale * dS^T . Q, with S^T = K . Q^T recomputed tile by tile
template <typename T, bool kDrop>
__global__ void __launch_bounds__(kThreads) attn_bwd_dkv(const AttnParams p) {
    __shared__ __align__(128) T ks[kTile][kPad];
    __shared__ __align__(128) T vs[kTile][kPad];
    __shared__ __align__(128) T qs[2][kTile][kPad];
    __shared__ __align__(128) T dos[2][kTile][kPad];
    __shared__ float lse_s[2][kTile], d_s[2][kTile];
    const int b = blockIdx.z / p.groups, g = blockIdx.z % p.groups, h = blockIdx.y;
    const int n0 = blockIdx.x * kTile, qtok = g * p.lq, ktok = g * p.lk;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gr = lane >> 2, tq = lane & 3;
    const T *Q = (const T *)p.q, *K = (const T *)p.k, *V = (const T *)p.v, *dO = (const T *)p.dout;
    const uint32_t bgh = (uint32_t)(blockIdx.z * p.heads + h);
    const float *lse_g = p.lse + (long long)bgh * p.lq, *d_g = p.delta + (long long)bgh * p.lq;
    uint2 key = make_uint2(0u, 0u);
    if (kDrop) key = drop_key(p);

    auto load_q = [&](int buf, int i0) {
        load_tile(qs[buf], Q, p.ldq, p.bs, b, h, qtok, i0, p.lq);
        load_tile(dos[buf], dO, p.lddo, p.bs, b, h, qtok, i0, p.lq);
        if (threadIdx.x < kTile) {      // rows past the group: P is finite and dO = D = 0, so they add nothing
            const int i = i0 + threadIdx.x;
            lse_s[buf][threadIdx.x] = i < p.lq ? lse_g[i] * kLog2e : 0.f;
            d_s[buf][threadIdx.x] = i < p.lq ? d_g[i] : 0.f;
        }
    };
    load_tile(ks, K, p.ldk, p.bs, b, h, ktok, n0, p.lk);
    load_tile(vs, V, p.ldv, p.bs, b, h, ktok, n0, p.lk);
    load_q(0, 0);
    cp_commit();

    const int ntiles = (p.lq + kTile - 1) / kTile;
    uint32_t kf[2][4], vf[2][4];
    float dk[4][4] = {}, dv[4][4] = {};
    const int j0 = n0 + warp * 16 + gr;       // this thread's keys j0 and j0 + 8
    for (int t = 0; t < ntiles; ++t) {
        const int buf = t & 1;
        if (t + 1 < ntiles) {
            load_q(buf ^ 1, (t + 1) * kTile);
            cp_commit();
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        if (t == 0) {
            load_a(kf, ks, warp * 16, lane);
            load_a(vf, vs, warp * 16, lane);
        }
        float s[8][4] = {}, dp[8][4] = {};
        mma_abt(s, kf, qs[buf], lane);
        mma_abt(dp, vf, dos[buf], lane);
        const int i0 = t * kTile;
        uint32_t za[4][4], da[4][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            const int c = n * 8 + 2 * tq;       // tile-local query column of s[n][0] (and of s[n][2])
            bool kp[4] = {true, true, true, true};
            if (kDrop) keep_cols4(key, bgh, i0 + c, j0, p.drop_thr, kp);  // s[n][0..1]: key j0; [2..3]: j0 + 8
            float pz[4], ds[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pe = exp2f(fmaf(s[n][e], p.scale_log2, -lse_s[buf][c + (e & 1)]));
                const float dz = kDrop ? (kp[e] ? dp[n][e] * p.inv_keep : 0.f) : dp[n][e];
                pz[e] = kDrop ? (kp[e] ? pe * p.inv_keep : 0.f) : pe;
                ds[e] = pe * (dz - d_s[buf][c + (e & 1)]);
            }
            za[n >> 1][(n & 1) * 2] = Mma<T>::pack(pz[0], pz[1]);
            za[n >> 1][(n & 1) * 2 + 1] = Mma<T>::pack(pz[2], pz[3]);
            da[n >> 1][(n & 1) * 2] = Mma<T>::pack(ds[0], ds[1]);
            da[n >> 1][(n & 1) * 2 + 1] = Mma<T>::pack(ds[2], ds[3]);
        }
        mma_ab(dv, za, dos[buf], lane);
        mma_ab(dk, da, qs[buf], lane);
        __syncthreads();
    }
    store_rows(dv, 1.f, 1.f, (T *)p.dv, p.lddv, p.bs, b, h, ktok, j0, p.lk, lane);
    store_rows(dk, p.scale, p.scale, (T *)p.dk, p.lddk, p.bs, b, h, ktok, j0, p.lk, lane);
}

__global__ void attn_dropout_mask_kernel(uint8_t *mask, long long total, int lq, int lk, uint32_t thr,
                                         unsigned long long seed, const unsigned long long *seed_base) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int j = (int)(e % lk);
    const long long r = e / lk;
    const int i = (int)(r % lq);
    const uint32_t bgh = (uint32_t)(r / lq);
    const unsigned long long s = seed + (seed_base ? *seed_base : 0ull);
    const uint4 w = philox4x32_10(make_uint4((uint32_t)j >> 1, (uint32_t)i >> 1, bgh, 0u),
                                  make_uint2((uint32_t)s, (uint32_t)(s >> 32)));
    mask[e] = word_of(w, (i & 1) * 2 + (j & 1)) >= thr ? 1 : 0;
}

uint32_t drop_threshold(float p) {
    const double t = (double)p * 4294967296.0;
    return t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
}

#define ATTN_REQUIRE(cond, msg) do { if (!(cond)) return fail("%s: " msg, who); } while (0)

int check_shape(const char *who, int nq, int nk, int bs, int heads, int head_dim, int groups, float drop_p) {
    ATTN_REQUIRE(head_dim == kD, "head_dim must be 32 (other head sizes are not a kernel case)");
    ATTN_REQUIRE(nq > 0 && nk > 0 && bs > 0 && heads > 0 && groups > 0, "bad dimension");
    ATTN_REQUIRE(nq % groups == 0 && nk % groups == 0, "query and key counts must be multiples of groups");
    ATTN_REQUIRE((long long)bs * groups <= 65535 && heads <= 65535, "batch * groups or heads too large");
    ATTN_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "dropout probability must be in [0, 1)");
    return 0;
}

int check_operand(const char *who, const void *x, long long ld, int heads) {
    ATTN_REQUIRE(x, "null pointer argument");
    ATTN_REQUIRE(aligned16(x), "device pointers must be 16-byte aligned");
    ATTN_REQUIRE(ld % 8 == 0 && ld >= (long long)heads * kD, "row stride must be a multiple of 8 and >= heads * 32");
    return 0;
}

AttnParams make_params(int nq, int nk, int bs, int heads, int groups, float scale, float drop_p, uint64_t seed,
                       const uint64_t *seed_base) {
    AttnParams p{};
    p.bs = bs;
    p.heads = heads;
    p.groups = groups;
    p.lq = nq / groups;
    p.lk = nk / groups;
    p.scale = scale;
    p.scale_log2 = scale * kLog2e;
    p.drop_p = drop_p;
    p.inv_keep = 1.f / (1.f - drop_p);
    p.drop_thr = drop_threshold(drop_p);
    p.seed = seed;
    p.seed_base = reinterpret_cast<const unsigned long long *>(seed_base);
    return p;
}

template <typename T>
void launch_fwd(const AttnParams &p, dim3 grid, cudaStream_t st) {
    if (p.drop_p > 0.f) attn_fwd<T, true><<<grid, kThreads, 0, st>>>(p);
    else attn_fwd<T, false><<<grid, kThreads, 0, st>>>(p);
}

template <typename T>
void launch_bwd(const AttnParams &p, dim3 gq, dim3 gk, cudaStream_t st) {
    if (p.drop_p > 0.f) {
        attn_bwd_dq<T, true><<<gq, kThreads, 0, st>>>(p);
        attn_bwd_dkv<T, true><<<gk, kThreads, 0, st>>>(p);
    } else {
        attn_bwd_dq<T, false><<<gq, kThreads, 0, st>>>(p);
        attn_bwd_dkv<T, false><<<gk, kThreads, 0, st>>>(p);
    }
}

}  // namespace
}  // namespace bevf

using namespace bevf;

extern "C" int bevf_attn_forward(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                 void *out, int64_t ldo, float *lse, int nq, int nk, int bs, int heads, int head_dim,
                                 int groups, float scale, float drop_p, uint64_t seed, const uint64_t *seed_base,
                                 int dtype, void *stream) {
    const char *who = "bevf_attn_forward";
    if (int e = check_shape(who, nq, nk, bs, heads, head_dim, groups, drop_p)) return e;
    ATTN_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F16, "storage must be bf16 or fp16");
    for (auto [x, ld] : {std::pair<const void *, long long>{q, ldq}, {k, ldk}, {v, ldv}, {out, ldo}})
        if (int e = check_operand(who, x, ld, heads)) return e;
    ATTN_REQUIRE(lse, "null pointer argument");
    AttnParams p = make_params(nq, nk, bs, heads, groups, scale, drop_p, seed, seed_base);
    p.q = q; p.k = k; p.v = v; p.out = out; p.lse = lse;
    p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
    const dim3 grid((p.lq + kTile - 1) / kTile, heads, bs * groups);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_BF16) launch_fwd<bf16>(p, grid, st);
    else launch_fwd<__half>(p, grid, st);
    return check_launch(who);
}

extern "C" int bevf_attn_backward(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                  const void *out, int64_t ldo, const void *grad_out, int64_t ldgo, const float *lse,
                                  float *delta, void *dq, int64_t lddq, void *dk, int64_t lddk, void *dv, int64_t lddv,
                                  int nq, int nk, int bs, int heads, int head_dim, int groups, float scale,
                                  float drop_p, uint64_t seed, const uint64_t *seed_base, int dtype, void *stream) {
    const char *who = "bevf_attn_backward";
    if (int e = check_shape(who, nq, nk, bs, heads, head_dim, groups, drop_p)) return e;
    ATTN_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F16, "storage must be bf16 or fp16");
    for (auto [x, ld] : {std::pair<const void *, long long>{q, ldq}, {k, ldk}, {v, ldv}, {out, ldo},
                         {grad_out, ldgo}, {dq, lddq}, {dk, lddk}, {dv, lddv}})
        if (int e = check_operand(who, x, ld, heads)) return e;
    ATTN_REQUIRE(lse && delta, "null pointer argument");
    AttnParams p = make_params(nq, nk, bs, heads, groups, scale, drop_p, seed, seed_base);
    p.q = q; p.k = k; p.v = v; p.o = out; p.dout = grad_out; p.lse = const_cast<float *>(lse); p.delta = delta;
    p.dq = dq; p.dk = dk; p.dv = dv;
    p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo; p.lddo = ldgo; p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    const dim3 gq((p.lq + kTile - 1) / kTile, heads, bs * groups), gk((p.lk + kTile - 1) / kTile, heads, bs * groups);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_BF16) launch_bwd<bf16>(p, gq, gk, st);
    else launch_bwd<__half>(p, gq, gk, st);
    return check_launch(who);
}

extern "C" int bevf_attn_dropout_mask(uint8_t *mask, int nq, int nk, int bs, int heads, int groups, float drop_p,
                                      uint64_t seed, const uint64_t *seed_base, void *stream) {
    const char *who = "bevf_attn_dropout_mask";
    if (int e = check_shape(who, nq, nk, bs, heads, kD, groups, drop_p)) return e;
    ATTN_REQUIRE(mask, "null pointer argument");
    const long long lq = nq / groups, lk = nk / groups;
    const long long total = (long long)bs * groups * heads * lq * lk;
    attn_dropout_mask_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        mask, total, (int)lq, (int)lk, drop_threshold(drop_p), seed, reinterpret_cast<const unsigned long long *>(seed_base));
    return check_launch(who);
}
