// GridMask for sm_90a: the detectors' training-time image mask (projects/mmdet3d_plugin/models/utils/grid_mask.py:70-124)
// applied without building it.  The reference draws a (1.5 H, 1.5 W) numpy mask stripe by stripe, crops its centre,
// copies it to the device (a synchronising pageable copy) and multiplies; here the mask of pixel (y, x) is a closed
// form of the drawn integers, evaluated where the pixel is read.
//
// Mapping.  A thread owns VEC = 16 / sizeof(T) consecutive columns of one image row.  It evaluates the row predicate
// and its VEC column predicates once, then walks every plane (camera x channel x sample: the reference shares one
// mask between them) with 16-byte loads and stores.  A chunk that is not full or not 16-byte aligned in every plane
// (W not a multiple of VEC, or an odd plane size) takes the scalar loop instead.  Memory-bound: one read and one write
// of every element.
//
// Arithmetic.  out = x * m with m in {0, 1} in fp32 (mul.rn.f32 without flush-to-zero), rounded to T with cvt.rn:
// what torch's `x * mask.to(x.dtype)` computes on the device, so inf * 0 and NaN give NaN and -x * 0 keeps its sign.
#include "common.cuh"

namespace bevf {

struct GridMaskGeom {
    int H, W, d, l, st_h, st_w, use_h, use_w, mode;
    int oy, ox;   // offset of the crop in the padded frame: ((hh - H) / 2, (ww - W) / 2), hh = int(1.5 * H)
    int nh, nw;   // stripes the loop draws: hh / d, ww / d
};

// The reference's stripe loop zeroes [d * k + st, min(d * k + st + l, n_pad)) for k in [0, n_pad / d); c < n_pad.
__device__ __forceinline__ bool in_stripe(int c, int st, int d, int l, int stripes) {
    const int t = c - st;
    if (t < 0) return false;
    const int k = t / d;
    return k < stripes && t - k * d < l;
}

__device__ __forceinline__ float mul_rn(float a, float b) {
    float r;
    asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

template <typename T> __device__ __forceinline__ float widen(T v);
template <> __device__ __forceinline__ float widen<float>(float v) { return v; }
template <> __device__ __forceinline__ float widen<bf16>(bf16 v) { return __uint_as_float((uint32_t)__bfloat16_as_ushort(v) << 16); }
template <> __device__ __forceinline__ float widen<__half>(__half v) { return __half2float(v); }

template <typename T> __device__ __forceinline__ T narrow(float v);
template <> __device__ __forceinline__ float narrow<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 narrow<bf16>(float v) {
    unsigned short r;
    asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(v));
    return __ushort_as_bfloat16(r);
}
template <> __device__ __forceinline__ __half narrow<__half>(float v) {
    unsigned short r;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(r) : "f"(v));
    return __ushort_as_half(r);
}

// 16 bytes of T times the VEC mask values
template <typename T> __device__ __forceinline__ uint4 mul_vec(uint4 v, const float (&m)[16 / sizeof(T)]) {
    if constexpr (sizeof(T) == 4) {
        return make_uint4(__float_as_uint(mul_rn(__uint_as_float(v.x), m[0])),
                          __float_as_uint(mul_rn(__uint_as_float(v.y), m[1])),
                          __float_as_uint(mul_rn(__uint_as_float(v.z), m[2])),
                          __float_as_uint(mul_rn(__uint_as_float(v.w), m[3])));
    } else {
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
            w[i] = St16<T>::pack(mul_rn(St16<T>::lo(w[i]), m[2 * i]), mul_rn(St16<T>::hi(w[i]), m[2 * i + 1]));
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
grid_mask_kernel(const T *__restrict__ x, T *__restrict__ out, long long planes, const GridMaskGeom g, int chunks) {
    constexpr int VEC = 16 / sizeof(T);
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)g.H * chunks) return;
    const int y = (int)(idx / chunks), x0 = (int)(idx - (long long)y * chunks) * VEC;
    const int n = min(VEC, g.W - x0);
    const bool row0 = g.use_h && in_stripe(y + g.oy, g.st_h, g.d, g.l, g.nh);
    float m[VEC];
    unsigned ones = 0;   // bit j: m[j] == 1 (the scalar loop indexes it at run time)
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
        const bool keep = !(row0 || (g.use_w && in_stripe(x0 + j + g.ox, g.st_w, g.d, g.l, g.nw)));
        m[j] = (keep != (g.mode != 0)) ? 1.f : 0.f;
        ones |= (m[j] != 0.f) << j;
    }
    const long long plane = (long long)g.H * g.W, off = (long long)y * g.W + x0;
    const bool vec = n == VEC && (plane * (long long)sizeof(T)) % 16 == 0 &&
                     ((reinterpret_cast<uintptr_t>(x + off) | reinterpret_cast<uintptr_t>(out + off)) & 15u) == 0;
    if (vec) {
#pragma unroll 4
        for (long long p = 0; p < planes; ++p) {
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(x + p * plane + off));
            *reinterpret_cast<uint4 *>(out + p * plane + off) = mul_vec<T>(v, m);
        }
    } else {
        for (long long p = 0; p < planes; ++p)
            for (int j = 0; j < n; ++j)
                out[p * plane + off + j] = narrow<T>(mul_rn(widen<T>(x[p * plane + off + j]), (ones >> j) & 1u ? 1.f : 0.f));
    }
}

template <typename T>
static void launch_grid_mask(const void *x, void *out, long long planes, const GridMaskGeom &g, cudaStream_t st) {
    constexpr int VEC = 16 / sizeof(T);
    const int chunks = (g.W + VEC - 1) / VEC;
    const long long threads = (long long)g.H * chunks;
    grid_mask_kernel<T><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>((const T *)x, (T *)out, planes, g, chunks);
}

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_grid_mask(const void *x, void *out, int dtype, int64_t planes, int H, int W, int d, int l,
                              int st_h, int st_w, int use_h, int use_w, int mode, void *stream) {
    const char *who = "bevf_grid_mask";
    if (dtype != BEVF_DTYPE_F32 && dtype != BEVF_DTYPE_BF16 && dtype != BEVF_DTYPE_F16)
        return fail("%s: dtype must be f32, bf16 or f16", who);
    if (planes < 0 || H < 0 || W < 0 || (long long)H * W >= (1ll << 31) || H > (1 << 30) || W > (1 << 30))
        return fail("%s: planes, H and W must be non-negative, H * W below 2^31 and H, W at most 2^30", who);
    if (d < 1 || l < 0 || st_h < 0 || st_h >= d || st_w < 0 || st_w >= d)
        return fail("%s: need d >= 1, l >= 0 and 0 <= st_h, st_w < d (got d = %lld, l = %lld)", who, d, l);
    if (mode != 0 && mode != 1) return fail("%s: mode must be 0 or 1", who);
    if (planes == 0 || H == 0 || W == 0) return 0;
    if (!x || !out) return fail("%s: null pointer argument", who);
    const int hh = H + H / 2, ww = W + W / 2;   // int(1.5 * H), int(1.5 * W)
    const GridMaskGeom g{H, W, d, l, st_h, st_w, use_h != 0, use_w != 0, mode, (hh - H) / 2, (ww - W) / 2,
                         hh / d, ww / d};
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_F32) launch_grid_mask<float>(x, out, planes, g, st);
    else if (dtype == BEVF_DTYPE_BF16) launch_grid_mask<bf16>(x, out, planes, g, st);
    else launch_grid_mask<__half>(x, out, planes, g, st);
    return check_launch(who);
}
