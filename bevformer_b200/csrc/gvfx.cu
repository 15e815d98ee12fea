// Helpers of the 64-bit fixed-point grad_value of the deterministic sampler backward (msda.cu:
// bevf_msda_backward_fx / bevf_msda_rows_backward_fx).
//
//   fx_bounds_launch       max|attn| and max|grad_out| over the launch's live rows as sign-cleared float bits in two
//                          device words (an unsigned maximum: order-free, and NaN / inf dominate every finite value)
//   bevf_msda_fx_frac_bits the fraction bits K a launch can use without any possibility of overflow
//   bevf_msda_fx_convert   int64 accumulators -> fp32 / bf16 / fp16 gradient, written or ADDED into the caller's buffer
// The scale is a power of two read from device words (no host synchronisation: capturable in a CUDA graph).
#include "common.cuh"

namespace bevf {

constexpr int kFxThreads = 256;

// one warp per query row; rows with row_map < 0 (unused rows of a fixed-capacity list, never written) are skipped
template <typename TG>
__global__ void __launch_bounds__(kFxThreads)
fx_bounds_kernel(const float *__restrict__ attn, const TG *__restrict__ grad_out, const int *__restrict__ row_map,
                 long long qrows, int n_attn, int n_grad, unsigned *__restrict__ bounds) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (kFxThreads / 32);
    unsigned ma = 0, mg = 0;
    for (long long r = (long long)blockIdx.x * (kFxThreads / 32) + (threadIdx.x >> 5); r < qrows; r += nwarps) {
        if (row_map && __ldg(row_map + r) < 0) continue;                      // warp-uniform
        const float *a = attn + r * n_attn;
        for (int i = lane; i < n_attn; i += 32) ma = max(ma, abs_bits(__ldg(a + i)));
        const TG *g = grad_out + r * n_grad;
        for (int i = lane; i < n_grad; i += 32) mg = max(mg, abs_bits(g[i]));
    }
    ma = __reduce_max_sync(0xffffffffu, ma);
    mg = __reduce_max_sync(0xffffffffu, mg);
    if (lane == 0) {
        if (ma) atomicMax(bounds, ma);
        if (mg) atomicMax(bounds + 1, mg);
    }
}

// out = fx * 2^(fx_exponent - frac_bits) (kAcc: out += ...); non-finite bounds: NaN everywhere
template <typename TO, bool kAcc>
__global__ void __launch_bounds__(kFxThreads)
fx_convert_kernel(const long long *__restrict__ fx, const unsigned *__restrict__ bounds, int frac_bits,
                  TO *__restrict__ out, long long n) {
    const unsigned ba = __ldg(bounds), bg = __ldg(bounds + 1);
    const bool finite = fx_bounds_finite(ba, bg);
    const double inv = finite ? fx_pow2(fx_exponent(ba, bg) - frac_bits) : 0.0;
    for (long long i = (long long)blockIdx.x * kFxThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kFxThreads) {
        float v = finite ? (float)((double)__ldg(fx + i) * inv) : __int_as_float(0x7fffffff);
        if constexpr (sizeof(TO) == 2) {
            if constexpr (kAcc) v += St16<TO>::to_f(out[i]);
            out[i] = St16<TO>::from_f(v);
        } else {
            if constexpr (kAcc) v += out[i];
            out[i] = v;
        }
    }
}

static unsigned fx_grid(long long work, int per_block) {
    const long long g = (work + per_block - 1) / per_block;
    const long long cap = (long long)device_sms() * 16;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

int fx_bounds_launch(const char *who, const float *attn, const void *grad_out, int grad_out_dtype,
                     const int32_t *row_map, long long qrows, int M, int D, int L, int P, uint32_t *bounds,
                     cudaStream_t st) {
    const int na = M * L * P, ng = M * D;
    cudaMemsetAsync(bounds, 0, 2 * sizeof(uint32_t), st);
    const unsigned grid = fx_grid(qrows, kFxThreads / 32);
    if (grad_out_dtype == BEVF_DTYPE_BF16)
        fx_bounds_kernel<bf16><<<grid, kFxThreads, 0, st>>>(attn, (const bf16 *)grad_out, row_map, qrows, na, ng, bounds);
    else if (grad_out_dtype == BEVF_DTYPE_F16)
        fx_bounds_kernel<__half><<<grid, kFxThreads, 0, st>>>(attn, (const __half *)grad_out, row_map, qrows, na, ng, bounds);
    else if (grad_out_dtype == BEVF_DTYPE_F32)
        fx_bounds_kernel<float><<<grid, kFxThreads, 0, st>>>(attn, (const float *)grad_out, row_map, qrows, na, ng, bounds);
    else
        return fail("%s: unsupported dtype code", who);
    return check_launch(who);
}

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_msda_fx_frac_bits(int64_t rows_per_map, int L, int P) {
    if (rows_per_map < 0 || L <= 0 || P <= 0) return -1;
    // an element receives at most one contribution per (row, level, point, corner) of the rows on its map
    const unsigned long long count = (unsigned long long)(rows_per_map > 0 ? rows_per_map : 1) * L * P * 4;
    int lg = 0;
    while (lg < 63 && (1ull << lg) < count) ++lg;                  // ceil(log2(count))
    const int k = 62 - lg;                                         // count * 2^k <= 2^62 < 2^63
    return k < 0 ? -1 : (k < 40 ? k : 40);
}

extern "C" int bevf_msda_fx_convert(const int64_t *grad_value_fx, const uint32_t *bounds, int frac_bits, void *out,
                                    int out_dtype, int accumulate, int64_t n, void *stream) {
    const char *who = "bevf_msda_fx_convert";
    if (n < 0 || frac_bits < 0 || frac_bits > 62) return fail("%s: bad dimension or frac_bits", who);
    if (n == 0) return 0;
    if (!grad_value_fx || !bounds || !out) return fail("%s: null pointer argument", who);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = fx_grid(n, kFxThreads);
    const long long *fx = reinterpret_cast<const long long *>(grad_value_fx);
    if (out_dtype == BEVF_DTYPE_F32) {
        if (accumulate) fx_convert_kernel<float, true><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (float *)out, n);
        else fx_convert_kernel<float, false><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (float *)out, n);
    } else if (out_dtype == BEVF_DTYPE_BF16) {
        if (accumulate) fx_convert_kernel<bf16, true><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (bf16 *)out, n);
        else fx_convert_kernel<bf16, false><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (bf16 *)out, n);
    } else if (out_dtype == BEVF_DTYPE_F16) {
        if (accumulate) fx_convert_kernel<__half, true><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (__half *)out, n);
        else fx_convert_kernel<__half, false><<<grid, kFxThreads, 0, st>>>(fx, bounds, frac_bits, (__half *)out, n);
    } else {
        return fail("%s: unsupported dtype code", who);
    }
    return check_launch(who);
}
