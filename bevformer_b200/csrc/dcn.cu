// Modulated deformable convolution (DCNv2) sampling for sm_90a: the deformable im2col of the forward and its
// backward.  The GEMMs around it are the library's own (gemm.cu, called from ops.py).
//
// Replaces the sampling half of mmcv._ext.modulated_deform_conv_forward / _backward (mmcv-full 1.4.0
// mmcv/ops/modulated_deform_conv.py), which ResNet-101-DCN builds through `dcn=dict(type='DCNv2', ...)`
// (projects/configs/bevformer/bevformer_base.py:43-53).  Arithmetic: SURVEY.md Appendix B.
//
// Layouts.  input is channels-last (N, H, W, C); offset (N, dg*2*kk, Ho, Wo) and mask (N, dg*kk, Ho, Wo) are mmcv's
// NCHW tensors read in place; the columns are (N*Ho*Wo, kk*C), column tap*C + c (K-major for the GEMM).
//
// Mapping.  A warp owns one (tile of 32 output pixels, tap, deform group).  Lane j computes the sample of pixel j of
// the tile ONCE -- position, range test, bilinear weights (corner_at, msda_common.cuh) -- reading offset / mask with
// consecutive lanes on consecutive pixels (coalesced).  The warp then walks the tile's pixels RP at a time: LN lanes
// per pixel take the group's Cg channels in 16-byte slices and receive the sample's scalars with __shfl_sync.
// Backward: the three per-sample sums (grad_mask, the two coordinate derivatives) are reduced over the LN lanes in a
// fixed xor order and handed back to lane j, which stores them (coalesced); grad_input is scattered with 16-byte fp32
// vector reductions, or as 64-bit fixed point in the deterministic form.
#include "msda_common.cuh"

namespace bevf {

struct DcnGeom {
    int N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg;
};

// lanes per pixel: the largest power of two <= min(32, 16-byte slices per group)
__host__ __device__ __forceinline__ int dcn_lanes(int nch) {
    int ln = 1;
    while (ln < 32 && 2 * ln <= nch) ln *= 2;
    return ln;
}

// The sample of (row, tap, group), computed by the lane that owns the row.  Its corners are packed for the shuffle:
// bits 0..3 the in-map flags f00, f01, f10, f11, bit 4 dx, bit 5 dy, bit 6 valid; gp = n * H * W + top-left pixel.
struct DcnSample {
    int gp, bits;
    float lx, ly, m;
};

template <typename T>
__device__ __forceinline__ DcnSample dcn_sample(const T *__restrict__ offset, const T *__restrict__ mask,
                                                const DcnGeom &g, long long row, long long R, int tap, int grp) {
    DcnSample s{0, 0, 0.f, 0.f, 0.f};
    if (row >= R) return s;
    const int hw = g.Ho * g.Wo, kk = g.kh * g.kw;
    const int n = (int)(row / hw), p = (int)(row - (long long)n * hw);
    const int ho = p / g.Wo, wo = p - ho * g.Wo;
    const int i = tap / g.kw, j = tap - i * g.kw;
    const T *op = offset + ((long long)n * g.dg * 2 * kk + grp * 2 * kk + 2 * tap) * hw + p;
    const float oh = Row<T>::load1(op), ow = Row<T>::load1(op + hw);
    s.m = Row<T>::load1(mask + ((long long)n * g.dg * kk + grp * kk + tap) * hw + p);
    // one fp32 add of an exact integer base and the widened offset: floor() picks the cell the restatement picks
    const float y = __fadd_rn((float)(ho * g.sh - g.ph + i * g.dh), oh);
    const float x = __fadd_rn((float)(wo * g.sw - g.pw + j * g.dw), ow);
    const Corner c = corner_at(x, y, g.H, g.W);
    s.gp = n * g.H * g.W + c.pidx;
    s.bits = (c.f00 != 0.f) | (c.f01 != 0.f) << 1 | (c.f10 != 0.f) << 2 | (c.f11 != 0.f) << 3 | c.dx << 4 | c.dy << 5 |
             (int)c.valid << 6;
    s.lx = c.lx;
    s.ly = c.ly;
    return s;
}

__device__ __forceinline__ DcnSample shfl_sample(const DcnSample &s, int src) {
    DcnSample t;
    t.gp = __shfl_sync(0xffffffffu, s.gp, src);
    t.bits = __shfl_sync(0xffffffffu, s.bits, src);
    t.lx = __shfl_sync(0xffffffffu, s.lx, src);
    t.ly = __shfl_sync(0xffffffffu, s.ly, src);
    t.m = __shfl_sync(0xffffffffu, s.m, src);
    return t;
}

// bilinear weights of a shuffled sample, with make_corner's arithmetic (zero for corners outside the map)
struct DcnWeights {
    float w00, w01, w10, w11, hx, hy;
};
__device__ __forceinline__ DcnWeights dcn_weights(const DcnSample &s) {
    DcnWeights w;
    w.hx = 1.f - s.lx;
    w.hy = 1.f - s.ly;
    w.w00 = (s.bits & 1) ? w.hy * w.hx : 0.f;
    w.w01 = (s.bits & 2) ? w.hy * s.lx : 0.f;
    w.w10 = (s.bits & 4) ? s.ly * w.hx : 0.f;
    w.w11 = (s.bits & 8) ? s.ly * s.lx : 0.f;
    return w;
}

// element offsets of the four corners of a shuffled sample (channel 0 of the image row)
__device__ __forceinline__ void dcn_corners(const DcnSample &s, const DcnGeom &g, long long (&o)[4]) {
    o[0] = (long long)s.gp * g.C;
    o[1] = o[0] + ((s.bits & 16) ? g.C : 0);
    const long long oy = (s.bits & 32) ? (long long)g.W * g.C : 0;
    o[2] = o[0] + oy;
    o[3] = o[1] + oy;
}

static unsigned dcn_grid(long long warps) {
    const long long g = (warps + kThreads / 32 - 1) / (kThreads / 32), cap = (long long)device_sms() * 16;
    return (unsigned)(g < cap ? g : cap);
}

// ------------------------------------------------------------------------------------------------
// sampling forward: cols[row, tap*C + c] = mask * bilinear(input[n, :, :, c], y, x)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
dcn_im2col(const T *__restrict__ input, const T *__restrict__ offset, const T *__restrict__ mask, T *__restrict__ cols,
           const DcnGeom g, long long R, long long tasks) {
    constexpr int VEC = 16 / sizeof(T);
    const int lane = threadIdx.x & 31, kk = g.kh * g.kw, Cg = g.C / g.dg, nch = Cg / VEC;
    const int LN = dcn_lanes(nch), RP = 32 / LN, sub = lane % LN, jr = lane / LN;
    const long long nwarps = (long long)gridDim.x * (kThreads / 32);
    for (long long t = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); t < tasks; t += nwarps) {
        const long long tile = t / (kk * g.dg);
        const int rem = (int)(t - tile * kk * g.dg), tap = rem / g.dg, grp = rem - tap * g.dg;
        const DcnSample mine = dcn_sample(offset, mask, g, tile * 32 + lane, R, tap, grp);
        for (int j0 = 0; j0 < 32; j0 += RP) {
            const int j = j0 + jr;
            const DcnSample s = shfl_sample(mine, j);
            const long long row = tile * 32 + j;
            if (row >= R) continue;
            const DcnWeights w = dcn_weights(s);
            const float q[4] = {w.w00 * s.m, w.w01 * s.m, w.w10 * s.m, w.w11 * s.m};
            long long o[4];
            dcn_corners(s, g, o);
            const T *in = input + grp * Cg;
            T *out = cols + row * kk * g.C + (long long)tap * g.C + grp * Cg;
            for (int ch = sub; ch < nch; ch += LN) {
                float acc[VEC];
#pragma unroll
                for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
                if (s.bits & 64) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        float v[VEC];
                        load_vec<T, VEC>(in + o[c] + ch * VEC, v);
#pragma unroll
                        for (int k = 0; k < VEC; ++k) acc[k] = fmaf(q[c], v[k], acc[k]);
                    }
                }
                store_vec<T, VEC>(out + ch * VEC, acc);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// sampling backward.  TV = float: grad_input accumulated with fp32 vector reductions; TV = long long: 64-bit fixed
// point (deterministic form) with the scale of bounds = {max|mask|, max|dcols|}
// ------------------------------------------------------------------------------------------------
template <typename T, typename TV>
__global__ void __launch_bounds__(kThreads)
dcn_col2im(const T *__restrict__ input, const T *__restrict__ offset, const T *__restrict__ mask,
           const T *__restrict__ dcols, TV *__restrict__ grad_input, T *__restrict__ grad_offset,
           T *__restrict__ grad_mask, const DcnGeom g, long long R, long long tasks,
           const unsigned *__restrict__ fx_bounds, int fx_bits) {
    constexpr int VEC = 16 / sizeof(T);
    constexpr bool kFx = sizeof(TV) == 8;
    double fx_sc = 0.0;
    bool scatter = true;
    if constexpr (kFx) {
        const unsigned bm = __ldg(fx_bounds), bg = __ldg(fx_bounds + 1);
        scatter = fx_bounds_finite(bm, bg);
        if (scatter) fx_sc = fx_pow2(fx_bits - fx_exponent(bm, bg));
    }
    const int lane = threadIdx.x & 31, kk = g.kh * g.kw, Cg = g.C / g.dg, nch = Cg / VEC, hw = g.Ho * g.Wo;
    const int LN = dcn_lanes(nch), RP = 32 / LN, sub = lane % LN, jr = lane / LN;
    const long long nwarps = (long long)gridDim.x * (kThreads / 32);
    for (long long t = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); t < tasks; t += nwarps) {
        const long long tile = t / (kk * g.dg);
        const int rem = (int)(t - tile * kk * g.dg), tap = rem / g.dg, grp = rem - tap * g.dg;
        const DcnSample mine = dcn_sample(offset, mask, g, tile * 32 + lane, R, tap, grp);
        float my_gm = 0.f, my_gx = 0.f, my_gy = 0.f;
        for (int j0 = 0; j0 < 32; j0 += RP) {
            const int j = j0 + jr;
            const DcnSample s = shfl_sample(mine, j);
            const long long row = tile * 32 + j;
            float gm = 0.f, gx = 0.f, gy = 0.f;
            if (row < R && (s.bits & 64)) {
                const DcnWeights w = dcn_weights(s);
                const float q[4] = {w.w00 * s.m, w.w01 * s.m, w.w10 * s.m, w.w11 * s.m};
                long long o[4];
                dcn_corners(s, g, o);
                const T *in = input + grp * Cg;
                TV *gi = grad_input + grp * Cg;
                const T *dc = dcols + row * kk * g.C + (long long)tap * g.C + grp * Cg;
                for (int ch = sub; ch < nch; ch += LN) {
                    float d[VEC], v[4][VEC];
                    load_vec<T, VEC>(dc + ch * VEC, d);
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        load_vec<T, VEC>(in + o[c] + ch * VEC, v[c]);
#pragma unroll
                        for (int k = 0; k < VEC; ++k) v[c][k] = (s.bits & (1 << c)) ? v[c][k] : 0.f;
                    }
#pragma unroll
                    for (int k = 0; k < VEC; ++k) {
                        gm = fmaf(d[k], w.hy * (w.hx * v[0][k] + s.lx * v[1][k]) + s.ly * (w.hx * v[2][k] + s.lx * v[3][k]), gm);
                        gx = fmaf(d[k], w.hy * (v[1][k] - v[0][k]) + s.ly * (v[3][k] - v[2][k]), gx);
                        gy = fmaf(d[k], w.hx * (v[2][k] - v[0][k]) + s.lx * (v[3][k] - v[1][k]), gy);
                    }
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        if (q[c] == 0.f) continue;
                        TV *p = gi + o[c] + ch * VEC;
                        if constexpr (kFx) {
                            if (scatter) {
#pragma unroll
                                for (int k = 0; k < VEC; ++k) red_add_fx(p + k, q[c], d[k], fx_sc);
                            }
                        } else {
#pragma unroll
                            for (int k = 0; k < VEC; k += 4)
                                red_add_v4(p + k, q[c] * d[k], q[c] * d[k + 1], q[c] * d[k + 2], q[c] * d[k + 3]);
                        }
                    }
                }
            }
            // fixed-order reduction over the row's LN lanes (every lane takes part: the count is warp-uniform)
            for (int sft = LN / 2; sft > 0; sft >>= 1) {
                gm += __shfl_xor_sync(0xffffffffu, gm, sft);
                gx += __shfl_xor_sync(0xffffffffu, gx, sft);
                gy += __shfl_xor_sync(0xffffffffu, gy, sft);
            }
            // the sums of row j0 + r sit in lane r * LN; lane j keeps those of row j
            const int src = (lane % RP) * LN;
            const float tm = __shfl_sync(0xffffffffu, gm, src), tx = __shfl_sync(0xffffffffu, gx, src),
                        ty = __shfl_sync(0xffffffffu, gy, src);
            if (lane / RP == j0 / RP) { my_gm = tm; my_gx = tx; my_gy = ty; }
        }
        const long long row = tile * 32 + lane;
        if (row < R) {
            const int n = (int)(row / hw), p = (int)(row - (long long)n * hw);
            T *go = grad_offset + ((long long)n * g.dg * 2 * kk + grp * 2 * kk + 2 * tap) * hw + p;
            Row<T>::store1(go, mine.m * my_gy);
            Row<T>::store1(go + hw, mine.m * my_gx);
            Row<T>::store1(grad_mask + ((long long)n * g.dg * kk + grp * kk + tap) * hw + p, my_gm);
        }
    }
}

// max|mask| and max|dcols| as sign-cleared float bits (an unsigned maximum: NaN / inf dominate every finite value)
template <typename T>
__global__ void __launch_bounds__(kThreads)
dcn_fx_bounds(const T *__restrict__ mask, long long nm, const T *__restrict__ dcols, long long nd,
              unsigned *__restrict__ bounds) {
    unsigned mm = 0, md = 0;
    const long long stride = (long long)gridDim.x * kThreads;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nm; i += stride) mm = max(mm, abs_bits(mask[i]));
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nd; i += stride) md = max(md, abs_bits(dcols[i]));
    mm = __reduce_max_sync(0xffffffffu, mm);
    md = __reduce_max_sync(0xffffffffu, md);
    if ((threadIdx.x & 31) == 0) {
        if (mm) atomicMax(bounds, mm);
        if (md) atomicMax(bounds + 1, md);
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int dcn_check(const char *who, int dtype, const DcnGeom &g, long long &R) {
    if (dtype != BEVF_DTYPE_F32 && dtype != BEVF_DTYPE_BF16 && dtype != BEVF_DTYPE_F16)
        return fail("%s: unsupported dtype code", who);
    if (g.N < 0 || g.H <= 0 || g.W <= 0 || g.C <= 0 || g.Ho < 0 || g.Wo < 0 || g.kh <= 0 || g.kw <= 0 || g.sh <= 0 ||
        g.sw <= 0 || g.ph < 0 || g.pw < 0 || g.dh <= 0 || g.dw <= 0 || g.dg <= 0)
        return fail("%s: negative or zero dimension", who);
    const int ho = (g.H + 2 * g.ph - g.dh * (g.kh - 1) - 1) / g.sh + 1, wo = (g.W + 2 * g.pw - g.dw * (g.kw - 1) - 1) / g.sw + 1;
    if (g.Ho != (ho > 0 ? ho : 0) || g.Wo != (wo > 0 ? wo : 0))
        return fail("%s: Ho, Wo are not the convolution's output size (expected %lld x %lld)", who, ho, wo);
    const int vec = dtype == BEVF_DTYPE_F32 ? 4 : 8;
    if (g.C % g.dg || (g.C / g.dg) % vec)
        return fail("%s: channels per deform group must be a multiple of %lld (16 bytes)", who, vec);
    if ((long long)g.N * g.H * g.W >= (1ll << 31) || (long long)g.Ho * g.Wo * g.kh * g.kw >= (1ll << 31) ||
        (long long)g.H * g.W * g.C >= (1ll << 31))
        return fail("%s: input or output map too large (2^31 pixels)", who);
    R = (long long)g.N * g.Ho * g.Wo;
    return 0;
}

static long long dcn_tasks(const DcnGeom &g, long long R) { return (R + 31) / 32 * g.kh * g.kw * g.dg; }

template <typename T>
static void launch_im2col(const void *input, const void *offset, const void *mask, void *cols, const DcnGeom &g,
                          long long R, cudaStream_t st) {
    const long long tasks = dcn_tasks(g, R);
    dcn_im2col<T><<<dcn_grid(tasks), kThreads, 0, st>>>((const T *)input, (const T *)offset, (const T *)mask, (T *)cols,
                                                         g, R, tasks);
}

template <typename T, typename TV>
static void launch_col2im(const void *input, const void *offset, const void *mask, const void *dcols, TV *gi,
                          void *goff, void *gmask, const DcnGeom &g, long long R, const uint32_t *bounds, int bits,
                          cudaStream_t st) {
    const long long tasks = dcn_tasks(g, R);
    dcn_col2im<T, TV><<<dcn_grid(tasks), kThreads, 0, st>>>((const T *)input, (const T *)offset, (const T *)mask,
                                                             (const T *)dcols, gi, (T *)goff, (T *)gmask, g, R, tasks,
                                                             bounds, bits);
}

template <typename TV>
static int dcn_backward_impl(const char *who, const void *input, const void *offset, const void *mask,
                             const void *dcols, int dtype, TV *grad_input, uint32_t *bounds, int frac_bits,
                             void *grad_offset, void *grad_mask, const DcnGeom &g, void *stream) {
    long long R = 0;
    if (int e = dcn_check(who, dtype, g, R)) return e;
    if (R == 0) return 0;
    if (!input || !offset || !mask || !dcols || !grad_input || !grad_offset || !grad_mask)
        return fail("%s: null pointer argument", who);
    if (!aligned16(input) || !aligned16(dcols) || !aligned16(grad_input))
        return fail("%s: input, dcols and grad_input must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    if constexpr (sizeof(TV) == 8) {
        if (!bounds) return fail("%s: null pointer argument", who);
        const int kmax = bevf_msda_fx_frac_bits((int64_t)g.Ho * g.Wo, 1, g.kh * g.kw);
        if (frac_bits < 0 || frac_bits > kmax)
            return fail("%s: frac_bits must be in [0, %lld] for this launch (bevf_msda_fx_frac_bits(Ho * Wo, 1, kh * kw))",
                        who, kmax);
        cudaMemsetAsync(bounds, 0, 2 * sizeof(uint32_t), st);
        const long long nm = (long long)g.N * g.dg * g.kh * g.kw * g.Ho * g.Wo, nd = R * g.kh * g.kw * g.C;
        const long long blocks = (nd + kThreads - 1) / kThreads, cap = (long long)device_sms() * 16;
        const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
        if (dtype == BEVF_DTYPE_F32) dcn_fx_bounds<float><<<grid, kThreads, 0, st>>>((const float *)mask, nm, (const float *)dcols, nd, bounds);
        else if (dtype == BEVF_DTYPE_BF16) dcn_fx_bounds<bf16><<<grid, kThreads, 0, st>>>((const bf16 *)mask, nm, (const bf16 *)dcols, nd, bounds);
        else dcn_fx_bounds<__half><<<grid, kThreads, 0, st>>>((const __half *)mask, nm, (const __half *)dcols, nd, bounds);
        if (int e = check_launch(who)) return e;
    }
    if (dtype == BEVF_DTYPE_F32)
        launch_col2im<float, TV>(input, offset, mask, dcols, grad_input, grad_offset, grad_mask, g, R, bounds, frac_bits, st);
    else if (dtype == BEVF_DTYPE_BF16)
        launch_col2im<bf16, TV>(input, offset, mask, dcols, grad_input, grad_offset, grad_mask, g, R, bounds, frac_bits, st);
    else
        launch_col2im<__half, TV>(input, offset, mask, dcols, grad_input, grad_offset, grad_mask, g, R, bounds, frac_bits, st);
    return check_launch(who);
}

}  // namespace bevf

using namespace bevf;

#define DCN_GEOM DcnGeom{N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg}

extern "C" int bevf_dcn_sampling_forward(const void *input, const void *offset, const void *mask, int dtype, void *cols,
                                         int N, int H, int W, int C, int Ho, int Wo, int kh, int kw, int sh, int sw,
                                         int ph, int pw, int dh, int dw, int dg, void *stream) {
    const char *who = "bevf_dcn_sampling_forward";
    const DcnGeom g = DCN_GEOM;
    long long R = 0;
    if (int e = dcn_check(who, dtype, g, R)) return e;
    if (R == 0) return 0;
    if (!input || !offset || !mask || !cols) return fail("%s: null pointer argument", who);
    if (!aligned16(input) || !aligned16(cols)) return fail("%s: input and cols must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_F32) launch_im2col<float>(input, offset, mask, cols, g, R, st);
    else if (dtype == BEVF_DTYPE_BF16) launch_im2col<bf16>(input, offset, mask, cols, g, R, st);
    else launch_im2col<__half>(input, offset, mask, cols, g, R, st);
    return check_launch(who);
}

extern "C" int bevf_dcn_sampling_backward(const void *input, const void *offset, const void *mask, const void *dcols,
                                          int dtype, float *grad_input, void *grad_offset, void *grad_mask, int N, int H,
                                          int W, int C, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                                          int dh, int dw, int dg, void *stream) {
    return dcn_backward_impl<float>("bevf_dcn_sampling_backward", input, offset, mask, dcols, dtype, grad_input, nullptr,
                                    0, grad_offset, grad_mask, DCN_GEOM, stream);
}

extern "C" int bevf_dcn_sampling_backward_fx(const void *input, const void *offset, const void *mask, const void *dcols,
                                             int dtype, int64_t *grad_input_fx, uint32_t *bounds, int frac_bits,
                                             void *grad_offset, void *grad_mask, int N, int H, int W, int C, int Ho,
                                             int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                                             int dg, void *stream) {
    return dcn_backward_impl<long long>("bevf_dcn_sampling_backward_fx", input, offset, mask, dcols, dtype,
                                        reinterpret_cast<long long *>(grad_input_fx), bounds, frac_bits, grad_offset,
                                        grad_mask, DCN_GEOM, stream);
}
