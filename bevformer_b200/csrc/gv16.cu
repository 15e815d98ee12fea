// Helpers of the scaled-fp16 accumulation of grad_value (msda.cu: bevf_msda_rows_backward_f16acc / _mixed).
//
// The sampler backward is bound by L2 reduction sectors; accumulating grad_value in fp16 instead of fp32 halves them
// for the levels where that is accurate enough (few contributions per pixel).  fp16 needs a scale:
//   bevf_abs_max        max|grad_out| as float bits in one device word (block maxima + atomicMax on the bit pattern)
//   gv16_scale()        (common.cuh) the power of two that puts that maximum into [8, 16)
//   bevf_gv16_unscale   fp16 accumulators -> bf16 gradient (divide by the scale), what the value projection consumes
//   bevf_gv_merge       mixed mode: fine levels (scaled fp16) + coarse levels (fp32 side buffer) -> one bf16 gradient
//   bevf_gv_merge_replicated   the same with replicated fp16 levels between them: their copies summed in fp32
// Replaces nothing in the reference one to one: there grad_value is allocated in value's dtype and accumulated with
// atomicAdd (multi_scale_deformable_attn_function.py:146-160); this is the same quantity, another accumulator format.
#include <cuda_fp16.h>

#include "common.cuh"

namespace bevf {

constexpr int kGvThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kGvThreads)
abs_max_kernel(const T *__restrict__ x, long long n8, unsigned *__restrict__ out) {
    // n8 = number of 16-byte groups; bf16: 8 values per group, fp32: 4
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * kGvThreads + threadIdx.x; i < n8; i += (long long)gridDim.x * kGvThreads) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(x) + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (sizeof(T) == 2) {
                m = fmaxf(m, fmaxf(fabsf(bf16_lo(w[j])), fabsf(bf16_hi(w[j]))));
            } else {
                m = fmaxf(m, fabsf(__uint_as_float(w[j])));
            }
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
    __shared__ float s_m[kGvThreads / 32];
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 1; i < kGvThreads / 32; ++i) m = fmaxf(m, s_m[i]);
        // non-negative floats order like their bit patterns; NaN (fmaxf drops it) never gets here
        atomicMax(out, __float_as_uint(m));
    }
}

__global__ void __launch_bounds__(kGvThreads)
gv16_unscale_kernel(const __half *__restrict__ gv16, const unsigned *__restrict__ amax, bf16 *__restrict__ out,
                    long long n8) {
    const float inv = 1.f / gv16_scale(__ldg(amax));                    // exact: a power of two
    for (long long i = (long long)blockIdx.x * kGvThreads + threadIdx.x; i < n8; i += (long long)gridDim.x * kGvThreads) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(gv16) + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint4 o;
        uint32_t *ow = &o.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[j]));
            ow[j] = pack_bf16x2(f.x * inv, f.y * inv);
        }
        reinterpret_cast<uint4 *>(out)[i] = o;
    }
}

// out (B, S, row) bf16  <-  f16 (B, S_fine + k * S_rep, row) scaled fp16  |  side (B, S - S_fine - S_rep, row) fp32;
// row = M * D elements.  Pixel p < S_fine of a map is f16 pixel p; S_fine <= p < S_fine + S_rep is the sum of the k
// copies p + c * S_rep of it (the replicated levels of msda_bwd_d32); the rest are side pixels from p - S_fine - S_rep.
__global__ void __launch_bounds__(kGvThreads)
gv_merge_kernel(const __half *__restrict__ f16, const float *__restrict__ side, const unsigned *__restrict__ amax,
                bf16 *__restrict__ out, long long groups_per_map, long long fine_groups_per_map,
                long long rep_groups_per_map, int k, long long total_groups) {
    // a group = 8 consecutive elements (16 B of bf16 output)
    const float inv = 1.f / gv16_scale(__ldg(amax));
    const long long f16_groups_per_map = fine_groups_per_map + k * rep_groups_per_map;
    const long long side_from = fine_groups_per_map + rep_groups_per_map;
    const long long side_groups_per_map = groups_per_map - side_from;
    for (long long i = (long long)blockIdx.x * kGvThreads + threadIdx.x; i < total_groups; i += (long long)gridDim.x * kGvThreads) {
        const long long b = i / groups_per_map, r = i - b * groups_per_map;
        uint4 o;
        if (r < side_from) {
            const uint4 *vp = reinterpret_cast<const uint4 *>(f16) + b * f16_groups_per_map + r;
            float acc[8];
            const int copies = r < fine_groups_per_map ? 1 : k;
            for (int c = 0; c < copies; ++c) {
                const uint4 v = __ldg(vp + c * rep_groups_per_map);
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[j]));
                    acc[2 * j] = c ? acc[2 * j] + f.x : f.x;
                    acc[2 * j + 1] = c ? acc[2 * j + 1] + f.y : f.y;
                }
            }
            uint32_t *ow = &o.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) ow[j] = pack_bf16x2(acc[2 * j] * inv, acc[2 * j + 1] * inv);
        } else {
            const float4 *sp = reinterpret_cast<const float4 *>(side) + 2 * (b * side_groups_per_map + (r - side_from));
            const float4 a = __ldg(sp), c = __ldg(sp + 1);
            o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
            o.z = pack_bf16x2(c.x, c.y); o.w = pack_bf16x2(c.z, c.w);
        }
        reinterpret_cast<uint4 *>(out)[i] = o;
    }
}

static unsigned gv_grid(long long groups) {
    long long g = (groups + kGvThreads - 1) / kGvThreads;
    const long long cap = (long long)device_sms() * 16;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_abs_max(const void *x, int dtype, int64_t n, uint32_t *amax_bits, void *stream) {
    const char *who = "bevf_abs_max";
    if (n < 0) return fail("%s: bad dimension", who);
    if (!amax_bits || (n > 0 && !x)) return fail("%s: null pointer argument", who);
    if (dtype != BEVF_DTYPE_BF16 && dtype != BEVF_DTYPE_F32) return fail("%s: unsupported dtype code", who);
    const int per = dtype == BEVF_DTYPE_BF16 ? 8 : 4;
    if (n % per || !aligned16(x)) return fail("%s: n must be a multiple of the 16-byte vector and x 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(amax_bits, 0, sizeof(uint32_t), st);
    if (n == 0) return 0;
    const long long groups = n / per;
    if (dtype == BEVF_DTYPE_BF16) abs_max_kernel<bf16><<<gv_grid(groups), kGvThreads, 0, st>>>((const bf16 *)x, groups, amax_bits);
    else abs_max_kernel<float><<<gv_grid(groups), kGvThreads, 0, st>>>((const float *)x, groups, amax_bits);
    return check_launch(who);
}

extern "C" int bevf_gv16_unscale(const void *gv16, const uint32_t *amax_bits, void *out_bf16, int64_t n, void *stream) {
    const char *who = "bevf_gv16_unscale";
    if (n < 0 || n % 8) return fail("%s: n must be a non-negative multiple of 8", who);
    if (n == 0) return 0;
    if (!gv16 || !amax_bits || !out_bf16) return fail("%s: null pointer argument", who);
    if (!aligned16(gv16) || !aligned16(out_bf16)) return fail("%s: device pointers must be 16-byte aligned", who);
    gv16_unscale_kernel<<<gv_grid(n / 8), kGvThreads, 0, (cudaStream_t)stream>>>((const __half *)gv16, amax_bits,
                                                                                (bf16 *)out_bf16, n / 8);
    return check_launch(who);
}

extern "C" int bevf_gv_merge(const void *fine_f16, const float *side_f32, const uint32_t *amax_bits, void *out_bf16,
                             int B, int S, int S_fine, int row_elems, void *stream) {
    const char *who = "bevf_gv_merge";
    if (B < 0 || S <= 0 || S_fine <= 0 || S_fine >= S || row_elems <= 0 || row_elems % 8)
        return fail("%s: bad dimension (0 < S_fine < S, row_elems a multiple of 8)", who);
    if (B == 0) return 0;
    if (!fine_f16 || !side_f32 || !amax_bits || !out_bf16) return fail("%s: null pointer argument", who);
    if (!aligned16(fine_f16) || !aligned16(side_f32) || !aligned16(out_bf16))
        return fail("%s: device pointers must be 16-byte aligned", who);
    const long long gpm = (long long)S * row_elems / 8, fpm = (long long)S_fine * row_elems / 8;
    gv_merge_kernel<<<gv_grid(gpm * B), kGvThreads, 0, (cudaStream_t)stream>>>((const __half *)fine_f16, side_f32, amax_bits,
                                                                             (bf16 *)out_bf16, gpm, fpm, 0, 1, gpm * B);
    return check_launch(who);
}

extern "C" int bevf_gv_merge_replicated(const void *f16, const float *side_f32, const uint32_t *amax_bits,
                                        void *out_bf16, int B, int S, int S_fine, int S_rep, int replicas,
                                        int row_elems, void *stream) {
    const char *who = "bevf_gv_merge_replicated";
    if (B < 0 || S <= 0 || S_fine <= 0 || S_rep < 0 || S_fine + S_rep > S || replicas < 1 || row_elems <= 0 ||
        row_elems % 8)
        return fail("%s: bad dimension (0 < S_fine, 0 <= S_rep, S_fine + S_rep <= S, replicas >= 1, row_elems a "
                    "multiple of 8)", who);
    if (B == 0) return 0;
    const bool has_side = S_fine + S_rep < S;
    if (!f16 || (has_side && !side_f32) || !amax_bits || !out_bf16) return fail("%s: null pointer argument", who);
    if (!aligned16(f16) || !aligned16(side_f32) || !aligned16(out_bf16))
        return fail("%s: device pointers must be 16-byte aligned", who);
    const long long gpm = (long long)S * row_elems / 8, fpm = (long long)S_fine * row_elems / 8,
                    rpm = (long long)S_rep * row_elems / 8;
    gv_merge_kernel<<<gv_grid(gpm * B), kGvThreads, 0, (cudaStream_t)stream>>>((const __half *)f16, side_f32, amax_bits,
                                                                             (bf16 *)out_bf16, gpm, fpm, rpm, replicas,
                                                                             gpm * B);
    return check_launch(who);
}
