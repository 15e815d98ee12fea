// Device helpers shared by the sampler kernels (msda.cu, msda_splat.cuh, msda_dense.cu): the bilinear
// corner arithmetic of SURVEY.md Appendix A, the 16-byte row slices and their fp32 / bf16 math.
#pragma once

#include "common.cuh"

namespace bevf {

constexpr int kMaxLevels = 16;
constexpr int kThreads = 256;

struct Corner {
    int x0, y0;                       // top-left cell, unclamped: x0 in [-1, W-1], y0 in [-1, H-1]
    int pidx;                         // pixel index y0c*W + x0c of the (clamped) top-left corner
    int dx, dy;                       // 1 if the right / bottom neighbour is a distinct in-map pixel
    float w00, w01, w10, w11;         // bilinear weights (zero for corners outside the map / skipped)
    float lx, ly;
    float f00, f01, f10, f11;         // 1 if the corner lies inside the map and the sample counts
    bool valid;
};

// Corner of the sample at pixel coordinates (x, y) (pixel centres at integers).  Range test in float BEFORE any int
// conversion: projected anchors behind a camera reach |x| ~ 1e9.
__device__ __forceinline__ Corner corner_at(float x, float y, int H, int W) {
    Corner c;
    c.valid = (x > -1.f) && (y > -1.f) && (x < (float)W) && (y < (float)H);
    if (!c.valid) { x = 0.f; y = 0.f; }
    const float xf = floorf(x), yf = floorf(y);
    const int x0 = (int)xf, y0 = (int)yf, x1 = x0 + 1, y1 = y0 + 1;
    c.lx = x - xf; c.ly = y - yf;
    const float hx = 1.f - c.lx, hy = 1.f - c.ly;
    const bool x0ok = x0 >= 0, x1ok = x1 <= W - 1, y0ok = y0 >= 0, y1ok = y1 <= H - 1;
    c.f00 = (c.valid && x0ok && y0ok) ? 1.f : 0.f;
    c.f01 = (c.valid && x1ok && y0ok) ? 1.f : 0.f;
    c.f10 = (c.valid && x0ok && y1ok) ? 1.f : 0.f;
    c.f11 = (c.valid && x1ok && y1ok) ? 1.f : 0.f;
    c.w00 = c.f00 * hy * hx;
    c.w01 = c.f01 * hy * c.lx;
    c.w10 = c.f10 * c.ly * hx;
    c.w11 = c.f11 * c.ly * c.lx;
    // Clamp into the map.  When x0 == -1 the only in-map column is x1 == 0: corner "00" then aliases
    // pixel 0 with weight 0 and corner "01" must also address pixel 0, hence dx = 0 (same for y).
    c.x0 = x0; c.y0 = y0;
    c.pidx = max(y0, 0) * W + max(x0, 0);
    c.dx = (x0ok && x1ok) ? 1 : 0;
    c.dy = (y0ok && y1ok) ? 1 : 0;
    return c;
}

// Corner of the sample at normalised location (locx, locy) of an H x W map.
__device__ __forceinline__ Corner make_corner(float locx, float locy, int H, int W) {
    // unfused multiply / add: the sampling cell is floor(x), so x must round exactly like the
    // reference expression loc * W - 0.5 (an FMA would flip floor() for samples on a cell boundary)
    return corner_at(__fadd_rn(__fmul_rn(locx, (float)W), -0.5f), __fadd_rn(__fmul_rn(locy, (float)H), -0.5f), H, W);
}

__device__ __forceinline__ void load_levels(const int64_t *level_hw, const int64_t *level_start,
                                            int L, int *s_h, int *s_w, int *s_start) {
    if ((int)threadIdx.x < L) {
        s_h[threadIdx.x] = (int)level_hw[2 * threadIdx.x];
        s_w[threadIdx.x] = (int)level_hw[2 * threadIdx.x + 1];
        s_start[threadIdx.x] = (int)level_start[threadIdx.x];
    }
    __syncthreads();
}

// Per-level tables for the fast kernels: element offset of the level's first pixel row (times the
// pixel stride) and element stride between image rows, so the inner loop does no multiplies.
struct LevelTab {
    int h[kMaxLevels], w[kMaxLevels], rs[kMaxLevels];
    long long lofs[kMaxLevels];
};
__device__ __forceinline__ void load_level_tab(const int64_t *level_hw, const int64_t *level_start, int L,
                                               int pix, LevelTab &t) {
    if ((int)threadIdx.x < L) {
        const int l = threadIdx.x;
        t.h[l] = (int)level_hw[2 * l];
        t.w[l] = (int)level_hw[2 * l + 1];
        t.rs[l] = t.w[l] * pix;
        t.lofs[l] = (long long)level_start[l] * pix;
    }
    __syncthreads();
}

// The pyramid as the HOST planned with it (dense tensor-core backward, msda_dense.cu).  Both kernels of that path
// evaluate the same predicate on the device -- host shapes == device spatial_shapes / level_start -- so a stale
// host copy degrades to the plain reduction path instead of producing a wrong gradient.
struct HostLevels {
    int h[kMaxLevels], w[kMaxLevels], start[kMaxLevels];
};
__device__ __forceinline__ bool host_levels_match(const HostLevels &hl, const int64_t *level_hw,
                                                  const int64_t *level_start, int L) {
    bool ok = true;
    for (int l = 0; l < L; ++l)
        ok = ok && (int)level_hw[2 * l] == hl.h[l] && (int)level_hw[2 * l + 1] == hl.w[l] &&
             (int)level_start[l] == hl.start[l];
    return ok;
}

// ---- per-storage-type math ---------------------------------------------------------------------
// a * b + c for bf16 a, b with one rounding: widening bf16 to fp32 is exact, so this is the fp32 FMA of the
// widened operands (Hopper has no mixed bf16 x bf16 + fp32 FMA instruction)
__device__ __forceinline__ float fhfma(unsigned short a, unsigned short b, float c) {
    return fmaf(__uint_as_float((uint32_t)a << 16), __uint_as_float((uint32_t)b << 16), c);
}
__device__ __forceinline__ void split16(uint32_t u, unsigned short &lo, unsigned short &hi) {
    asm("mov.b32 {%0, %1}, %2;" : "=h"(lo), "=h"(hi) : "r"(u));
}

template <typename T> struct Vec;          // 16 B of a row as loaded
template <> struct Vec<float> {
    float4 v;
    static constexpr int N = 4;
    __device__ __forceinline__ void load(const float *p) { v = __ldg(reinterpret_cast<const float4 *>(p)); }
    __device__ __forceinline__ void axpy(float w, float (&acc)[4]) const {
        acc[0] = fmaf(w, v.x, acc[0]); acc[1] = fmaf(w, v.y, acc[1]);
        acc[2] = fmaf(w, v.z, acc[2]); acc[3] = fmaf(w, v.w, acc[3]);
    }
    __device__ __forceinline__ float dot(const float (&g)[4]) const {
        return fmaf(g[0], v.x, fmaf(g[1], v.y, fmaf(g[2], v.z, g[3] * v.w)));
    }
};
template <> struct Vec<bf16> {
    uint4 v;
    static constexpr int N = 8;
    __device__ __forceinline__ void load(const bf16 *p) { v = __ldg(reinterpret_cast<const uint4 *>(p)); }
    // acc += w * v with w already rounded to bf16 (products exact, fp32 accumulation)
    __device__ __forceinline__ void axpy_h(unsigned short w, float (&acc)[8]) const {
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            unsigned short lo, hi;
            split16(u[i], lo, hi);
            acc[2 * i] = fhfma(lo, w, acc[2 * i]);
            acc[2 * i + 1] = fhfma(hi, w, acc[2 * i + 1]);
        }
    }
    // <g, v> with g given as packed bf16 (exact products)
    __device__ __forceinline__ float dot_h(const uint4 &g) const {
        const uint32_t u[4] = {v.x, v.y, v.z, v.w}, q[4] = {g.x, g.y, g.z, g.w};
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            unsigned short lo, hi, glo, ghi;
            split16(u[i], lo, hi);
            split16(q[i], glo, ghi);
            d = fhfma(lo, glo, d);
            d = fhfma(hi, ghi, d);
        }
        return d;
    }
    // <g, v> with g in fp32
    __device__ __forceinline__ float dot(const float (&g)[8]) const {
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            d = fmaf(g[2 * i], bf16_lo(u[i]), d);
            d = fmaf(g[2 * i + 1], bf16_hi(u[i]), d);
        }
        return d;
    }
};

// fp16 rows: widened exactly and multiplied with fp32 weights / gradients (no fp16 arithmetic)
template <> struct Vec<__half> {
    uint4 v;
    static constexpr int N = 8;
    __device__ __forceinline__ void load(const __half *p) { v = __ldg(reinterpret_cast<const uint4 *>(p)); }
    __device__ __forceinline__ void axpy(float w, float (&acc)[8]) const {
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            acc[2 * i] = fmaf(w, f16_lo(u[i]), acc[2 * i]);
            acc[2 * i + 1] = fmaf(w, f16_hi(u[i]), acc[2 * i + 1]);
        }
    }
    __device__ __forceinline__ float dot(const float (&g)[8]) const {
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            d = fmaf(g[2 * i], f16_lo(u[i]), d);
            d = fmaf(g[2 * i + 1], f16_hi(u[i]), d);
        }
        return d;
    }
};

template <int LANES> struct GroupMask;
template <> struct GroupMask<4> { static constexpr unsigned kBits = 0x11111111u; };
template <> struct GroupMask<8> { static constexpr unsigned kBits = 0x01010101u; };
template <> struct GroupMask<16> { static constexpr unsigned kBits = 0x00010001u; };

// level of flat sample index s (= s / P) without an integer division: magic = ceil(2^16 / P),
// exact while s * P < 2^16 (checked on the host: L * P * P < 65536).
__device__ __forceinline__ int level_of(int s, int magic) { return (s * magic) >> 16; }

__device__ __forceinline__ int value_map_of(const int *row_map, long long row, int M, int Q) {
    return row_map ? __ldg(row_map + row / M) : (int)(row / ((long long)M * Q));
}


// SpatialCrossAttention's sampling-point prep done inside the row-list sampler (bevf_sca_rows_forward_fused /
// bevf_sca_rows_backward_fused): instead of reading loc / attn, a kernel derives every sample from the head's raw
// offsets|logits, the row's softmax statistics and the camera-projected reference points -- with exactly the
// operations of sca_prep_fwd_m8 (encoder_ops.cu), so the samples are bit-identical to the prep kernel's.
// Sampler row (t, m): pair row t = b * R + r of batch item b, head m; 8 heads, L * P == 32.
struct ScaFuse {
    const float *raw;          // (bs * Nq, 8 * 32 * 3) fp32: per BEV query [offsets (8, L, P, 2) | logits (8, L * P)]
    const float *ref_cam;      // (ncam, bs, Nq, Dz, 2)
    const int *pair_q, *pair_cam, *pair_of;
    float2 *stats;             // (bs * R * 8): softmax max and 1 / sum of every sampler row (written by the forward)
    bf16 *d_raw;               // backward: (bs * Nq, 8 * 32 * 3) gradient of raw
    // forward: the samples of levels [coarse_from, L) as (bs * R * 8, L - coarse_from, P) -- what the dense backward
    // kernel reads (msda_dense.cu), in the loc / attn layout restricted to those levels; coarse_from = L: none
    float2 *coarse_loc;
    float *coarse_attn;
    int coarse_from;
    int bs, Nq, R, Dz, ncam;
};
constexpr int kFuseHeads = 8, kFuseLP = 32;

// inputs of sampler row `row`; false for an unused pair row
struct ScaRow {
    const float *lg, *off;     // the head's logits / offsets in raw
    const float2 *ref;         // reference points of (cam, b, q)
    long long raw_row;         // b * Nq + q
    int q;
};
__device__ __forceinline__ bool sca_row(const ScaFuse &fz, long long row, ScaRow &sr) {
    const long long t = row / kFuseHeads;
    const int m = (int)(row - t * kFuseHeads);
    const int b = (int)(t / fz.R), r = (int)(t - (long long)b * fz.R);
    const int q = __ldg(fz.pair_q + r), cam = __ldg(fz.pair_cam + r);
    if (q < 0) return false;
    sr.q = q;
    sr.raw_row = (long long)b * fz.Nq + q;
    const float *rq = fz.raw + sr.raw_row * (kFuseHeads * kFuseLP * 3);
    sr.off = rq + m * kFuseLP * 2;
    sr.lg = rq + kFuseHeads * kFuseLP * 2 + m * kFuseLP;
    sr.ref = reinterpret_cast<const float2 *>(fz.ref_cam) + (((long long)cam * fz.bs + b) * fz.Nq + q) * fz.Dz;
    return true;
}
// sample k = l * P + p of a row: loc = ref[p mod Dz] + off / (W, H)
__device__ __forceinline__ void sca_loc(const ScaRow &sr, int k, int l, int P, int Dz, int H, int W, float &x,
                                        float &y) {
    const float2 o = __ldg(reinterpret_cast<const float2 *>(sr.off) + k);
    const float2 rf = __ldg(sr.ref + (k - l * P) % Dz);
    x = rf.x + __fdiv_rn(o.x, (float)W);
    y = rf.y + __fdiv_rn(o.y, (float)H);
}
// attn of sample k from the row's softmax statistics: exp(logit - max) * (1 / sum)
__device__ __forceinline__ float sca_attn(const ScaRow &sr, int k, float mx, float inv) {
    return exp_rn(__ldg(sr.lg + k) - mx) * inv;
}
// softmax statistics of a row in sca_prep_fwd_m8's partition: lane `sub` of the row's quad holds logits
// [8 sub, 8 sub + 8), and gets their attention weights in `a`; all 32 lanes must call it
__device__ __forceinline__ float2 sca_row_stats(const ScaRow &sr, bool live, int sub, float (&a)[8]) {
#pragma unroll
    for (int i = 0; i < 8; i += 4) {
        const float4 v = live ? __ldg(reinterpret_cast<const float4 *>(sr.lg + 8 * sub + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
    }
    float mx = a[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, a[i]);
    mx = quad_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a[i] = exp_rn(a[i] - mx); sum += a[i]; }
    const float inv = __frcp_rn(quad_sum(sum));
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] *= inv;
    return make_float2(mx, inv);
}

}  // namespace bevf
