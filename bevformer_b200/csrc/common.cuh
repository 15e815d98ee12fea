// Shared device/host helpers for the bevformer_b200 kernels (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <string>

#include "../../include/bevformer_b200.h"

namespace bevf {

// ---- host side: error string + launch accounting ----------------------------------------------
std::string &last_error();
extern std::atomic<int64_t> g_launches;

inline int fail(const char *fmt, const char *a = "", long long x = 0, long long y = 0) {
    char buf[512];
    snprintf(buf, sizeof(buf), fmt, a, x, y);
    last_error() = buf;
    return 1;
}

inline int check_launch(const char *what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();
        char buf[512];
        snprintf(buf, sizeof(buf), "%s: launch failed: %s", what, cudaGetErrorString(e));
        last_error() = buf;
        return 2;
    }
    return 0;
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// SM count of the current device, queried once per process; 132 (an H100 SXM) where no device answers
// (host-only queries such as workspace sizes on a machine without a GPU)
inline int device_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
            cudaGetLastError();
            return 132;
        }
        sms = n;
    }
    return sms;
}

// ---- device side ------------------------------------------------------------------------------
typedef __nv_bfloat16 bf16;

// exp(x) rounded correctly to fp32: evaluated in double, which --use_fast_math leaves alone (a plain expf would become
// the ~10-ulp __expf).  The softmaxes of the sampling heads use it: their gradients feed sums with heavy cancellation.
__device__ __forceinline__ float exp_rn(float x) { return (float)exp((double)x); }

__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    // cvt.rn.bf16x2.f32 d, a, b  puts a in the upper half, b in the lower half
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// A "row" is the 32 contiguous channels of one (pixel, head).  kVec channels per lane, 16 B each.
template <typename T> struct Row;
template <> struct Row<float> {
    static constexpr int kVec = 4;
    __device__ static __forceinline__ void load(const float *p, float (&v)[4]) {
        float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    __device__ static __forceinline__ void store(float *p, const float (&v)[4]) {
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __device__ static __forceinline__ float load1(const float *p) { return __ldg(p); }
    __device__ static __forceinline__ void store1(float *p, float v) { *p = v; }
};
template <> struct Row<bf16> {
    static constexpr int kVec = 8;
    __device__ static __forceinline__ void load(const bf16 *p, float (&v)[8]) {
        uint4 t = __ldg(reinterpret_cast<const uint4 *>(p));
        v[0] = bf16_lo(t.x); v[1] = bf16_hi(t.x); v[2] = bf16_lo(t.y); v[3] = bf16_hi(t.y);
        v[4] = bf16_lo(t.z); v[5] = bf16_hi(t.z); v[6] = bf16_lo(t.w); v[7] = bf16_hi(t.w);
    }
    __device__ static __forceinline__ void store(bf16 *p, const float (&v)[8]) {
        uint4 t;
        t.x = pack_bf16x2(v[0], v[1]); t.y = pack_bf16x2(v[2], v[3]);
        t.z = pack_bf16x2(v[4], v[5]); t.w = pack_bf16x2(v[6], v[7]);
        *reinterpret_cast<uint4 *>(p) = t;
    }
    __device__ static __forceinline__ float load1(const bf16 *p) {
        return __bfloat162float(*p);
    }
    __device__ static __forceinline__ void store1(bf16 *p, float v) { *p = __float2bfloat16_rn(v); }
};

// N consecutive channels (N = 4 or 8) <-> fp32 registers, for either storage type.
template <typename T, int N> __device__ __forceinline__ void load_vec(const T *p, float (&v)[N]);
template <> __device__ __forceinline__ void load_vec<float, 4>(const float *p, float (&v)[4]) {
    Row<float>::load(p, v);
}
template <> __device__ __forceinline__ void load_vec<float, 8>(const float *p, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4 *>(p));
    const float4 b = __ldg(reinterpret_cast<const float4 *>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void load_vec<bf16, 8>(const bf16 *p, float (&v)[8]) {
    Row<bf16>::load(p, v);
}
template <> __device__ __forceinline__ void load_vec<bf16, 4>(const bf16 *p, float (&v)[4]) {
    const uint2 t = __ldg(reinterpret_cast<const uint2 *>(p));
    v[0] = bf16_lo(t.x); v[1] = bf16_hi(t.x); v[2] = bf16_lo(t.y); v[3] = bf16_hi(t.y);
}
template <typename T, int N> __device__ __forceinline__ void store_vec(T *p, const float (&v)[N]);
template <> __device__ __forceinline__ void store_vec<float, 4>(float *p, const float (&v)[4]) {
    Row<float>::store(p, v);
}
template <> __device__ __forceinline__ void store_vec<float, 8>(float *p, const float (&v)[8]) {
    reinterpret_cast<float4 *>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4 *>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
template <> __device__ __forceinline__ void store_vec<bf16, 8>(bf16 *p, const float (&v)[8]) {
    Row<bf16>::store(p, v);
}
template <> __device__ __forceinline__ void store_vec<bf16, 4>(bf16 *p, const float (&v)[4]) {
    *reinterpret_cast<uint2 *>(p) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
}

// 16-byte fp32 vector reduction into global memory (SASS: REDG.E.ADD.F32x4).
__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- grad_value accumulated in SCALED fp16 (msda.cu, gv16.cu) ---------------------------------------
// 16-byte fp16 vector reduction, 8 channels (SASS: REDG.E.ADD.F16x2.RN x4): half the L2 reduction sectors of fp32.
__device__ __forceinline__ void red_add_v4_f16x2(void *p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("red.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// Power-of-two scale that puts max|grad_out| into [8, 16): sums of up to ~4000 unit-weight contributions stay below
// fp16's 65504 and everything down to 2^-17 of the maximum stays a NORMAL fp16 number.  amax_bits = the float bits
// of max|grad_out| (bevf_abs_max); 0 / inf / nan -> 1.
__device__ __forceinline__ float gv16_scale(unsigned amax_bits) {
    const float a = __uint_as_float(amax_bits);
    if (!(a > 0.f) || !(a < 3.0e38f)) return 1.f;
    const int e = (int)((amax_bits >> 23) & 0xffu) - 127;          // floor(log2(a)) for normal a (denormal: -127)
    const int ex = min(127 + 3 - e, 254);                          // (maxima below 2^-124 saturate at 2^127)
    return __uint_as_float((unsigned)ex << 23);                    // 2^(3 - e)
}

// ---- grad_value summed in 64-bit FIXED POINT (deterministic mode; msda.cu, gvfx.cu) --------------------------------
// Integer addition is associative, so red.global.add.u64 of two's-complement values gives the same bits in any order.
// bounds[0] / bounds[1] hold the bits of max|attn| / max|grad_out| with the sign cleared: as unsigned numbers NaN >
// inf > every finite value, so a non-finite input shows in the maximum.  Every contribution w * attn * g (w <= 1) is
// below 2^fx_exponent(bounds) and is stored as round(contribution * 2^(frac_bits - fx_exponent)).
__host__ __device__ __forceinline__ bool fx_bounds_finite(unsigned a_bits, unsigned g_bits) {
    return a_bits < 0x7f800000u && g_bits < 0x7f800000u;
}
__host__ __device__ __forceinline__ int fx_exponent(unsigned a_bits, unsigned g_bits) {
    // a value with biased exponent field f (f = 0: zero or denormal) is below 2^(max(f, 1) - 126)
    const int ea = (int)(a_bits >> 23 > 1u ? a_bits >> 23 : 1u) - 126;
    const int eg = (int)(g_bits >> 23 > 1u ? g_bits >> 23 : 1u) - 126;
    return ea + eg;
}
// 2^e as a double, -1022 <= e <= 1023
__device__ __forceinline__ double fx_pow2(int e) { return __longlong_as_double((long long)(1023 + e) << 52); }
// one contribution q * g (exact in double: two fp32 factors) scaled by a power of two and rounded to nearest
__device__ __forceinline__ void red_add_fx(long long *p, float q, float g, double scale) {
    const long long v = __double2ll_rn((double)q * (double)g * scale);
    asm volatile("red.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

}  // namespace bevf
