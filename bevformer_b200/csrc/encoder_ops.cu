// Fused memory-bound pieces of one BEVFormer encoder layer (everything between the GEMMs and the
// sampler).  Each kernel replaces a run of ATen launches in the reference; see the per-function
// comments in include/bevformer_b200.h for the Python lines.  All are HBM-bound streaming kernels:
// 16 B vector accesses, one pass over each tensor, fp32 math.
#include <curand_kernel.h>

#include "common.cuh"

namespace bevf {

constexpr int kEThreads = 256;


__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// ------------------------------------------------------------------------------------------------
// SCA sampling-point preparation
// raw row (per query): [ offsets (M, L, P, 2) | logits (M, L*P) ]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEThreads)
sca_prep_fwd(const float *__restrict__ raw, const float *__restrict__ ref_cam,
             const int *__restrict__ pair_q, const int *__restrict__ pair_cam,
             const int64_t *__restrict__ level_hw, float *__restrict__ loc, float *__restrict__ attn,
             int B, int Nq, int R, int M, int L, int P, int D, int ncam) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * R * M;
    if (t >= total) return;
    const int m = (int)(t % M);
    const long long br = t / M;
    const int r = (int)(br % R), b = (int)(br / R);
    const int q = pair_q[r], cam = pair_cam[r];
    if (q < 0) return;                                // unused row of a fixed-capacity pair list
    const int LP = L * P, nout = M * LP * 3;
    const float *rq = raw + ((long long)b * Nq + q) * nout;
    const float *off = rq + (long long)m * LP * 2;
    const float *lg = rq + (long long)M * LP * 2 + (long long)m * LP;
    const float *rc = ref_cam + (((long long)cam * B + b) * Nq + q) * D * 2;
    // softmax over the L*P logits of this head
    float mx = -INFINITY;
    for (int k = 0; k < LP; ++k) mx = fmaxf(mx, lg[k]);
    float sum = 0.f;
    for (int k = 0; k < LP; ++k) sum += exp_rn(lg[k] - mx);
    const float inv = __frcp_rn(sum);
    float *lo = loc + t * LP * 2;
    float *at = attn + t * LP;
    for (int l = 0; l < L; ++l) {
        const float fw = (float)level_hw[2 * l + 1], fh = (float)level_hw[2 * l];
        for (int p = 0; p < P; ++p) {
            const int k = l * P + p, z = p % D;          // point p uses Z-anchor p mod D (quirk 3)
            const float2 o = *reinterpret_cast<const float2 *>(off + 2 * k);
            const float2 rf = *reinterpret_cast<const float2 *>(rc + 2 * z);
            *reinterpret_cast<float2 *>(lo + 2 * k) = make_float2(rf.x + __fdiv_rn(o.x, fw), rf.y + __fdiv_rn(o.y, fh));
            at[k] = exp_rn(lg[k] - mx) * inv;
        }
    }
}

// scalar / pair stores into an f32 or bf16 gradient tensor
__device__ __forceinline__ void st1(float *p, float v) { *p = v; }
__device__ __forceinline__ void st1(bf16 *p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void st2(float *p, float a, float b) { *reinterpret_cast<float2 *>(p) = make_float2(a, b); }
__device__ __forceinline__ void st2(bf16 *p, float a, float b) { *reinterpret_cast<uint32_t *>(p) = pack_bf16x2(a, b); }

// d_raw for every query: sums over the cameras that see it (pair_of[cam][q] = row or -1)
template <typename TO>
__global__ void __launch_bounds__(kEThreads)
sca_prep_bwd(const float *__restrict__ raw, const float *__restrict__ grad_loc,
             const float *__restrict__ grad_attn, const int *__restrict__ pair_of,
             const int64_t *__restrict__ level_hw, TO *__restrict__ d_raw, int B, int Nq, int R,
             int M, int L, int P, int ncam) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Nq * M;
    if (t >= total) return;
    const int m = (int)(t % M);
    const long long bq = t / M;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    const int LP = L * P, nout = M * LP * 3;
    const float *lg = raw + bq * nout + (long long)M * LP * 2 + (long long)m * LP;
    TO *d_off = d_raw + bq * nout + (long long)m * LP * 2;
    TO *d_lg = d_raw + bq * nout + (long long)M * LP * 2 + (long long)m * LP;
    int rows[16];
    int n = 0;
    for (int c = 0; c < ncam && c < 16; ++c) {
        const int r = pair_of[(long long)c * Nq + q];
        if (r >= 0) rows[n++] = r;
    }
    float mx = -INFINITY;
    for (int k = 0; k < LP; ++k) mx = fmaxf(mx, lg[k]);
    float sum = 0.f;
    for (int k = 0; k < LP; ++k) sum += exp_rn(lg[k] - mx);
    const float inv = __frcp_rn(sum);
    // dot = sum_k a_k * Ga_k
    float dot = 0.f;
    for (int k = 0; k < LP; ++k) {
        float ga = 0.f;
        for (int i = 0; i < n; ++i) ga += grad_attn[(((long long)b * R + rows[i]) * M + m) * LP + k];
        dot += exp_rn(lg[k] - mx) * inv * ga;
    }
    for (int l = 0; l < L; ++l) {
        const float fw = (float)level_hw[2 * l + 1], fh = (float)level_hw[2 * l];
        for (int p = 0; p < P; ++p) {
            const int k = l * P + p;
            float ga = 0.f, gx = 0.f, gy = 0.f;
            for (int i = 0; i < n; ++i) {
                const long long s = (((long long)b * R + rows[i]) * M + m) * LP + k;
                ga += grad_attn[s];
                const float2 g2 = *reinterpret_cast<const float2 *>(grad_loc + 2 * s);
                gx += g2.x; gy += g2.y;
            }
            const float a = exp_rn(lg[k] - mx) * inv;
            st1(d_lg + k, a * (ga - dot));
            st2(d_off + 2 * k, __fdiv_rn(gx, fw), __fdiv_rn(gy, fh));
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Warp-cooperative SCA prep for num_heads == 8: one warp per row, lane = (head m = lane / 4,
// quarter sub = lane % 4), each lane owns PPL = L*P/4 consecutive sampling points of its head.
// Every global access is a 16 B vector and a quad covers a head's contiguous 32*PPL/8.. bytes, so
// the warp reads / writes whole 128 B lines; the softmax reduces over the quad with two shuffles.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
template <int N> __device__ __forceinline__ void ldv(const float *p, float (&v)[N]) {
    if constexpr (N % 4 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 4) {
            const float4 t = __ldg(reinterpret_cast<const float4 *>(p + i));
            v[i] = t.x; v[i + 1] = t.y; v[i + 2] = t.z; v[i + 3] = t.w;
        }
    } else if constexpr (N % 2 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 2) {
            const float2 t = __ldg(reinterpret_cast<const float2 *>(p + i));
            v[i] = t.x; v[i + 1] = t.y;
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i) v[i] = __ldg(p + i);
    }
}
template <int N> __device__ __forceinline__ void stv(float *p, const float (&v)[N]) {
    if constexpr (N % 4 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 4) *reinterpret_cast<float4 *>(p + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
    } else if constexpr (N % 2 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 2) *reinterpret_cast<float2 *>(p + i) = make_float2(v[i], v[i + 1]);
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i) p[i] = v[i];
    }
}

// d_raw may be wanted in bf16 (it feeds the bf16 dX / dW GEMMs of the offsets|logits head): the
// rounding then happens here instead of in a separate cast pass over the tensor
template <int N> __device__ __forceinline__ void stv(bf16 *p, const float (&v)[N]) {
    if constexpr (N % 8 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 8)
            *reinterpret_cast<uint4 *>(p + i) = make_uint4(pack_bf16x2(v[i], v[i + 1]), pack_bf16x2(v[i + 2], v[i + 3]),
                                                           pack_bf16x2(v[i + 4], v[i + 5]), pack_bf16x2(v[i + 6], v[i + 7]));
    } else if constexpr (N % 4 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 4)
            *reinterpret_cast<uint2 *>(p + i) = make_uint2(pack_bf16x2(v[i], v[i + 1]), pack_bf16x2(v[i + 2], v[i + 3]));
    } else if constexpr (N % 2 == 0) {
#pragma unroll
        for (int i = 0; i < N; i += 2) *reinterpret_cast<uint32_t *>(p + i) = pack_bf16x2(v[i], v[i + 1]);
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i) p[i] = __float2bfloat16_rn(v[i]);
    }
}

template <int PPL>
__global__ void __launch_bounds__(kEThreads)
sca_prep_fwd_m8(const float *__restrict__ raw, const float *__restrict__ ref_cam,
                const int *__restrict__ pair_q, const int *__restrict__ pair_cam,
                const int64_t *__restrict__ level_hw, float *__restrict__ loc, float *__restrict__ attn,
                int B, int Nq, int R, int L, int P, int D, int pmagic) {
    constexpr int M = 8;
    __shared__ float s_w[16], s_h[16];
    if ((int)threadIdx.x < L) { s_h[threadIdx.x] = (float)level_hw[2 * threadIdx.x]; s_w[threadIdx.x] = (float)level_hw[2 * threadIdx.x + 1]; }
    __syncthreads();
    const int lane = threadIdx.x & 31, m = lane >> 2, sub = lane & 3;
    const long long t = (long long)blockIdx.x * (kEThreads / 32) + (threadIdx.x >> 5);   // row b*R + r
    if (t >= (long long)B * R) return;
    const int r = (int)(t % R), b = (int)(t / R);
    const int q = __ldg(pair_q + r), cam = __ldg(pair_cam + r);
    if (q < 0) return;                                // unused row of a fixed-capacity pair list (warp-uniform)
    const int LP = 4 * PPL, k0 = sub * PPL;
    const float *rq = raw + ((long long)b * Nq + q) * (M * LP * 3);
    float lg[PPL], off[2 * PPL];
    ldv<PPL>(rq + M * LP * 2 + m * LP + k0, lg);
    ldv<2 * PPL>(rq + (m * LP + k0) * 2, off);
    float mx = lg[0];
#pragma unroll
    for (int i = 1; i < PPL; ++i) mx = fmaxf(mx, lg[i]);
    mx = quad_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PPL; ++i) { lg[i] = exp_rn(lg[i] - mx); sum += lg[i]; }
    const float inv = __frcp_rn(quad_sum(sum));
    const float *rc = ref_cam + (((long long)cam * B + b) * Nq + q) * D * 2;
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
        const int k = k0 + i;
        const int l = (k * pmagic) >> 16;                  // k / P
        const int z = (k - l * P) % D;
        const float2 rf = __ldg(reinterpret_cast<const float2 *>(rc) + z);
        off[2 * i] = rf.x + __fdiv_rn(off[2 * i], s_w[l]);
        off[2 * i + 1] = rf.y + __fdiv_rn(off[2 * i + 1], s_h[l]);
        lg[i] *= inv;
    }
    stv<2 * PPL>(loc + ((t * M + m) * LP + k0) * 2, off);
    stv<PPL>(attn + (t * M + m) * LP + k0, lg);
}

template <int PPL, typename TO>
__global__ void __launch_bounds__(kEThreads)
sca_prep_bwd_m8(const float *__restrict__ raw, const float *__restrict__ grad_loc,
                const float *__restrict__ grad_attn, const int *__restrict__ pair_of,
                const int64_t *__restrict__ level_hw, TO *__restrict__ d_raw, int B, int Nq, int R,
                int L, int P, int ncam, int pmagic) {
    constexpr int M = 8;
    __shared__ float s_w[16], s_h[16];
    if ((int)threadIdx.x < L) { s_h[threadIdx.x] = (float)level_hw[2 * threadIdx.x]; s_w[threadIdx.x] = (float)level_hw[2 * threadIdx.x + 1]; }
    __syncthreads();
    const int lane = threadIdx.x & 31, m = lane >> 2, sub = lane & 3;
    const long long bq = (long long)blockIdx.x * (kEThreads / 32) + (threadIdx.x >> 5);
    if (bq >= (long long)B * Nq) return;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    const int LP = 4 * PPL, k0 = sub * PPL;
    const long long rbase = bq * (M * LP * 3);
    float a[PPL];
    ldv<PPL>(raw + rbase + M * LP * 2 + m * LP + k0, a);
    float mx = a[0];
#pragma unroll
    for (int i = 1; i < PPL; ++i) mx = fmaxf(mx, a[i]);
    mx = quad_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PPL; ++i) { a[i] = exp_rn(a[i] - mx); sum += a[i]; }
    const float inv = __frcp_rn(quad_sum(sum));
    float ga[PPL], gl[2 * PPL];
#pragma unroll
    for (int i = 0; i < PPL; ++i) { ga[i] = 0.f; gl[2 * i] = 0.f; gl[2 * i + 1] = 0.f; }
    // pair rows of this query under every camera, fetched up front: the loads are independent, whereas
    // "load row id -> test -> load gradients" per camera would serialise ncam round trips (a query is
    // seen by 1.1 cameras on average, so most of them only find out that there is nothing to add)
    constexpr int kCamBatch = 8;
    for (int c0 = 0; c0 < ncam; c0 += kCamBatch) {
        int rid[kCamBatch];
#pragma unroll
        for (int c = 0; c < kCamBatch; ++c)
            rid[c] = (c0 + c < ncam) ? __ldg(pair_of + (long long)(c0 + c) * Nq + q) : -1;   // warp-uniform
#pragma unroll
        for (int c = 0; c < kCamBatch; ++c) {
            if (rid[c] < 0) continue;
            const long long s = (((long long)b * R + rid[c]) * M + m) * LP + k0;
            float t1[PPL], t2[2 * PPL];
            ldv<PPL>(grad_attn + s, t1);
            ldv<2 * PPL>(grad_loc + 2 * s, t2);
#pragma unroll
            for (int i = 0; i < PPL; ++i) { ga[i] += t1[i]; gl[2 * i] += t2[2 * i]; gl[2 * i + 1] += t2[2 * i + 1]; }
        }
    }
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < PPL; ++i) { a[i] *= inv; dot += a[i] * ga[i]; }
    dot = quad_sum(dot);
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
        const int k = k0 + i;
        const int l = (k * pmagic) >> 16;
        ga[i] = a[i] * (ga[i] - dot);
        gl[2 * i] = __fdiv_rn(gl[2 * i], s_w[l]);
        gl[2 * i + 1] = __fdiv_rn(gl[2 * i + 1], s_h[l]);
    }
    stv<PPL>(d_raw + rbase + M * LP * 2 + m * LP + k0, ga);
    stv<2 * PPL>(d_raw + rbase + (m * LP + k0) * 2, gl);
}

// column sums of a (rows, C) matrix into fp32 (bias gradients): out[c] += sum_r x[r, c]
// thread -> (column vector cv, row lane rl); consecutive threads walk along a row (coalesced 16 B
// loads), four rows in flight per thread; row lanes are combined through shared memory without
// atomics, then one global atomicAdd per column per CTA -- or, with `part` (deterministic mode), the CTA's row of
// column sums stored into part[blockIdx.x] for partials_add_kernel.
template <typename T>
__global__ void __launch_bounds__(kEThreads)
colsum_kernel(const T *__restrict__ x, float *__restrict__ out, long long rows, int C, int rows_per_cta,
              float *__restrict__ part = nullptr) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    const int per_row = C / VEC;
    const int cv = threadIdx.x % per_row, rl = threadIdx.x / per_row, rstep = kEThreads / per_row;
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
    const long long r0 = (long long)blockIdx.x * rows_per_cta;
    const long long r1 = min(rows, r0 + rows_per_cta);
    if (rl < rstep) {
        long long r = r0 + rl;
        for (; r + 3ll * rstep < r1; r += 4ll * rstep) {
            float v0[VEC], v1[VEC], v2[VEC], v3[VEC];
            load_vec<T, VEC>(x + r * C + cv * VEC, v0);
            load_vec<T, VEC>(x + (r + rstep) * C + cv * VEC, v1);
            load_vec<T, VEC>(x + (r + 2ll * rstep) * C + cv * VEC, v2);
            load_vec<T, VEC>(x + (r + 3ll * rstep) * C + cv * VEC, v3);
#pragma unroll
            for (int k = 0; k < VEC; ++k) acc[k] += (v0[k] + v1[k]) + (v2[k] + v3[k]);
        }
        for (; r < r1; r += rstep) {
            float v[VEC];
            load_vec<T, VEC>(x + r * C + cv * VEC, v);
#pragma unroll
            for (int k = 0; k < VEC; ++k) acc[k] += v[k];
        }
    }
    extern __shared__ float s_part[];                  // rstep x C floats
    if (rl < rstep) {
#pragma unroll
        for (int k = 0; k < VEC; ++k) s_part[rl * C + cv * VEC + k] = acc[k];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kEThreads) {
        float t = 0.f;
        for (int j = 0; j < rstep; ++j) t += s_part[j * C + c];
        if (part) part[(long long)blockIdx.x * C + c] = t;
        else atomicAdd(out + c, t);
    }
}

// d_pre = dy * scale wherever the saved activation h is non-zero: the joint backward of
// dropout(relu(z)) given h = dropout(relu(z)) (h != 0 <=> z > 0 and the element was kept)
template <typename T>
__global__ void __launch_bounds__(kEThreads)
relu_dropout_bwd_kernel(const T *__restrict__ dy, const T *__restrict__ h, T *__restrict__ out,
                        long long n_vec, float scale) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_vec) return;
    float g[VEC], a[VEC];
    load_vec<T, VEC>(dy + i * VEC, g);
    load_vec<T, VEC>(h + i * VEC, a);
#pragma unroll
    for (int k = 0; k < VEC; ++k) g[k] = a[k] != 0.f ? g[k] * scale : 0.f;
    store_vec<T, VEC>(out + i * VEC, g);
}

// in-place inverted dropout with Philox bits (no mask tensor): x *= keep / (1 - p)
template <typename T>
__global__ void __launch_bounds__(kEThreads)
dropout_inplace_kernel(T *__restrict__ x, long long n_vec, float p, unsigned long long seed,
                       const unsigned long long *__restrict__ seed_base) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_vec) return;
    if (seed_base) seed += *seed_base;
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)i, 0ull, &st);
    const float scale = 1.f / (1.f - p);
    float v[VEC];
    load_vec<T, VEC>(x + i * VEC, v);
#pragma unroll
    for (int k = 0; k < VEC; k += 4) {
        const float4 u = curand_uniform4(&st);
        v[k] = u.x >= p ? v[k] * scale : 0.f; v[k + 1] = u.y >= p ? v[k + 1] * scale : 0.f;
        v[k + 2] = u.z >= p ? v[k + 2] * scale : 0.f; v[k + 3] = u.w >= p ? v[k + 3] * scale : 0.f;
    }
    store_vec<T, VEC>(x + i * VEC, v);
}

// ------------------------------------------------------------------------------------------------
// TSA sampling-point preparation.  raw row: [ offsets (M, 2, L, P, 2) | logits (M, 2, L*P) ]
// out rows ordered (b, queue j, q): loc (B*2, Nq, M, L, P, 2), attn (B*2, Nq, M, L, P)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEThreads)
tsa_prep_fwd(const float *__restrict__ raw, const float *__restrict__ ref2d,
             const int64_t *__restrict__ level_hw, float *__restrict__ loc, float *__restrict__ attn,
             int B, int Nq, int M, int L, int P) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Nq * M * 2;
    if (t >= total) return;
    const int j = (int)(t & 1);
    const long long t2 = t >> 1;
    const int m = (int)(t2 % M);
    const long long bq = t2 / M;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    const int LP = L * P, nout = M * 2 * LP * 3;
    const float *off = raw + bq * nout + ((long long)m * 2 + j) * LP * 2;
    const float *lg = raw + bq * nout + (long long)M * 2 * LP * 2 + ((long long)m * 2 + j) * LP;
    const long long orow = (((long long)b * 2 + j) * Nq + q);
    const float *rf = ref2d + orow * L * 2;
    float mx = -INFINITY;
    for (int k = 0; k < LP; ++k) mx = fmaxf(mx, lg[k]);
    float sum = 0.f;
    for (int k = 0; k < LP; ++k) sum += exp_rn(lg[k] - mx);
    const float inv = __frcp_rn(sum);
    float *lo = loc + (orow * M + m) * LP * 2;
    float *at = attn + (orow * M + m) * LP;
    for (int l = 0; l < L; ++l) {
        const float fw = (float)level_hw[2 * l + 1], fh = (float)level_hw[2 * l];
        const float rx = rf[2 * l], ry = rf[2 * l + 1];
        for (int p = 0; p < P; ++p) {
            const int k = l * P + p;
            const float2 o = *reinterpret_cast<const float2 *>(off + 2 * k);
            *reinterpret_cast<float2 *>(lo + 2 * k) = make_float2(rx + __fdiv_rn(o.x, fw), ry + __fdiv_rn(o.y, fh));
            at[k] = exp_rn(lg[k] - mx) * inv;
        }
    }
}

template <typename TO>
__global__ void __launch_bounds__(kEThreads)
tsa_prep_bwd(const float *__restrict__ raw, const float *__restrict__ grad_loc,
             const float *__restrict__ grad_attn, const int64_t *__restrict__ level_hw,
             TO *__restrict__ d_raw, int B, int Nq, int M, int L, int P) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Nq * M * 2;
    if (t >= total) return;
    const int j = (int)(t & 1);
    const long long t2 = t >> 1;
    const int m = (int)(t2 % M);
    const long long bq = t2 / M;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    const int LP = L * P, nout = M * 2 * LP * 3;
    const long long o_off = bq * nout + ((long long)m * 2 + j) * LP * 2;
    const long long o_lg = bq * nout + (long long)M * 2 * LP * 2 + ((long long)m * 2 + j) * LP;
    const float *lg = raw + o_lg;
    const long long orow = (((long long)b * 2 + j) * Nq + q);
    const float *gl = grad_loc + (orow * M + m) * LP * 2;
    const float *ga = grad_attn + (orow * M + m) * LP;
    float mx = -INFINITY;
    for (int k = 0; k < LP; ++k) mx = fmaxf(mx, lg[k]);
    float sum = 0.f;
    for (int k = 0; k < LP; ++k) sum += exp_rn(lg[k] - mx);
    const float inv = __frcp_rn(sum);
    float dot = 0.f;
    for (int k = 0; k < LP; ++k) dot += exp_rn(lg[k] - mx) * inv * ga[k];
    for (int l = 0; l < L; ++l) {
        const float fw = (float)level_hw[2 * l + 1], fh = (float)level_hw[2 * l];
        for (int p = 0; p < P; ++p) {
            const int k = l * P + p;
            const float a = exp_rn(lg[k] - mx) * inv;
            st1(d_raw + o_lg + k, a * (ga[k] - dot));
            const float2 g2 = *reinterpret_cast<const float2 *>(gl + 2 * k);
            st2(d_raw + o_off + 2 * k, __fdiv_rn(g2.x, fw), __fdiv_rn(g2.y, fh));
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over C channels with fused residual add and an optional second output y + pos.
// One warp per row; a lane holds C/32 channels in registers (C <= 1024, C % 128 == 0 fast path for
// 16 B accesses).  Statistics in fp32; eps inside the sqrt.
// ------------------------------------------------------------------------------------------------
// Keep-mask of the fused dropout: Philox4x32-10 keyed by (seed, row * 32 + lane); element i of the
// lane's PER channels uses draw i.  Forward and backward regenerate the same bits, nothing is stored.
template <int PER>
__device__ __forceinline__ void dropout_scale(float (&m)[PER], unsigned long long seed, long long row, int lane,
                                              float p) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)row * 32ull + (unsigned long long)lane, 0ull, &st);
    const float scale = 1.f / (1.f - p);
#pragma unroll
    for (int i = 0; i < PER; i += 4) {
        const float4 u = curand_uniform4(&st);
        m[i] = u.x >= p ? scale : 0.f; m[i + 1] = u.y >= p ? scale : 0.f;
        m[i + 2] = u.z >= p ? scale : 0.f; m[i + 3] = u.w >= p ? scale : 0.f;
    }
}

// One lane's share of a row as loaded (16 B vectors), so the NEXT row's loads can be in flight while the
// current row is reduced.  Chunk ci holds channels [ci*32*VEC + lane*VEC, +VEC).
template <typename T, int PER> struct RawRow {
    static constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    static constexpr int NCH = PER / VEC;
    uint4 q[NCH];
    __device__ __forceinline__ void load(const T *row_ptr, int lane) {
#pragma unroll
        for (int ci = 0; ci < NCH; ++ci)
            q[ci] = __ldg(reinterpret_cast<const uint4 *>(row_ptr + ci * 32 * VEC + lane * VEC));
    }
    __device__ __forceinline__ void unpack(float (&v)[PER]) const {
#pragma unroll
        for (int ci = 0; ci < NCH; ++ci) {
            if constexpr (sizeof(T) == 2) {
                const uint32_t u[4] = {q[ci].x, q[ci].y, q[ci].z, q[ci].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) { v[ci * 8 + 2 * k] = bf16_lo(u[k]); v[ci * 8 + 2 * k + 1] = bf16_hi(u[k]); }
            } else {
                v[ci * 4] = __uint_as_float(q[ci].x); v[ci * 4 + 1] = __uint_as_float(q[ci].y);
                v[ci * 4 + 2] = __uint_as_float(q[ci].z); v[ci * 4 + 3] = __uint_as_float(q[ci].w);
            }
        }
    }
};

template <typename TP> __device__ __forceinline__ float ldp(const TP *p, int i);
template <> __device__ __forceinline__ float ldp<float>(const float *p, int i) { return __ldg(p + i); }
template <> __device__ __forceinline__ float ldp<bf16>(const bf16 *p, int i) { return __bfloat162float(p[i]); }

constexpr int kLnRowsPerWarp = 4;

template <typename T, typename TP, int C>
__global__ void __launch_bounds__(kEThreads)
layernorm_fwd(const T *__restrict__ x, const T *__restrict__ res, const TP *__restrict__ gamma,
              const TP *__restrict__ beta, const T *__restrict__ pos, T *__restrict__ y,
              T *__restrict__ y2, float *__restrict__ mean_out, float *__restrict__ rstd_out,
              long long rows, float eps, float drop_p, unsigned long long seed,
              const unsigned long long *__restrict__ seed_base) {
    constexpr int PER = C / 32;                 // channels per lane (8 for C = 256)
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    static_assert(PER % VEC == 0, "C must be a multiple of 32 * VEC");
    if (seed_base) seed += *seed_base;          // device-side step counter (CUDA-graph replays)
    const int lane = threadIdx.x & 31;
    const long long row0 = ((long long)blockIdx.x * (kEThreads / 32) + (threadIdx.x >> 5)) * kLnRowsPerWarp;
    if (row0 >= rows) return;
    float gam[PER], bet[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int c = (i / VEC) * 32 * VEC + lane * VEC + (i % VEC);
        gam[i] = ldp<TP>(gamma, c); bet[i] = ldp<TP>(beta, c);
    }
    RawRow<T, PER> xr, rr, xn, rn;
    xr.load(x + row0 * C, lane);
    if (res) rr.load(res + row0 * C, lane);
#pragma unroll 1
    for (int it = 0; it < kLnRowsPerWarp; ++it) {
        const long long row = row0 + it;
        if (row >= rows) break;
        const bool more = (it + 1 < kLnRowsPerWarp) && (row + 1 < rows);
        if (more) {                              // next row's loads go out before this row's math
            xn.load(x + (row + 1) * C, lane);
            if (res) rn.load(res + (row + 1) * C, lane);
        }
        float v[PER];
        xr.unpack(v);
        if (drop_p > 0.f) {
            float msk[PER];
            dropout_scale<PER>(msk, seed, row, lane, drop_p);
#pragma unroll
            for (int i = 0; i < PER; ++i) v[i] *= msk[i];
        }
        if (res) {
            float r2[PER];
            rr.unpack(r2);
#pragma unroll
            for (int i = 0; i < PER; ++i) v[i] += r2[i];
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) s += v[i];
        const float mean = warp_sum(s) * (1.f / C);
        float s2 = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) { const float d = v[i] - mean; s2 += d * d; }
        const float rstd = __frsqrt_rn(warp_sum(s2) * (1.f / C) + eps);
        if (lane == 0) {
            if (mean_out) mean_out[row] = mean;
            if (rstd_out) rstd_out[row] = rstd;
        }
#pragma unroll
        for (int i = 0; i < PER; i += VEC) {
            const int c = (i / VEC) * 32 * VEC + lane * VEC;
            float o[VEC];
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = (v[i + k] - mean) * rstd * gam[i + k] + bet[i + k];
            store_vec<T, VEC>(y + row * C + c, o);
            if (y2) {
                float pz[VEC];
                load_vec<T, VEC>(pos + row * C + c, pz);
#pragma unroll
                for (int k = 0; k < VEC; ++k) pz[k] += o[k];
                store_vec<T, VEC>(y2 + row * C + c, pz);
            }
        }
        xr = xn; rr = rn;
    }
}

// Backward.  xin = dropout(x) + res is recomputed from the saved inputs (same Philox bits); dy2 (grad
// of the y + pos output) is added to dy.  d_sum is the gradient of the LayerNorm input: it is written to
// dres (the residual's gradient) and, times the keep-mask, to dx.  Without dropout and with dres ==
// nullptr only dx is written.  dgamma/dbeta accumulate into fp32 buffers, one atomicAdd per channel per CTA.
// kDet (deterministic mode): the warps are combined in index order and the CTA's [dgamma | dbeta] row is stored into
// part[blockIdx.x] instead; partials_add_kernel then sums the rows in CTA order into dgamma / dbeta.
template <typename T, typename TP, int C, bool kDet = false>
__global__ void __launch_bounds__(kEThreads)
layernorm_bwd(const T *__restrict__ x, const T *__restrict__ res, const TP *__restrict__ gamma,
              const float *__restrict__ mean_in, const float *__restrict__ rstd_in,
              const T *__restrict__ dy, const T *__restrict__ dy2, T *__restrict__ dx,
              T *__restrict__ dres, float *__restrict__ dgamma, float *__restrict__ dbeta, long long rows,
              int rows_per_cta, float drop_p, unsigned long long seed,
              const unsigned long long *__restrict__ seed_base, long long ld2, float *__restrict__ part = nullptr) {
    constexpr int PER = C / 32;
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    if (seed_base) seed += *seed_base;
    __shared__ float s_dg[C], s_db[C];
    for (int i = threadIdx.x; i < C; i += kEThreads) { s_dg[i] = 0.f; s_db[i] = 0.f; }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float adg[PER], adb[PER], gam[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        adg[i] = 0.f; adb[i] = 0.f;
        gam[i] = ldp<TP>(gamma, (i / VEC) * 32 * VEC + lane * VEC + (i % VEC));
    }
    const long long row0 = (long long)blockIdx.x * rows_per_cta;
    const long long row_end = min(rows, row0 + (long long)rows_per_cta);
    constexpr int kStep = kEThreads / 32;
    RawRow<T, PER> xr, rr, gr, g2r, xn, rn, gn, g2n;
    long long row = row0 + warp;
    if (row < row_end) {
        xr.load(x + row * C, lane);
        if (res) rr.load(res + row * C, lane);
        gr.load(dy + row * C, lane);
        if (dy2) g2r.load(dy2 + row * ld2, lane);
    }
#pragma unroll 1
    for (; row < row_end; row += kStep) {
        const long long nxt = row + kStep;
        if (nxt < row_end) {                     // prefetch the next row of this warp
            xn.load(x + nxt * C, lane);
            if (res) rn.load(res + nxt * C, lane);
            gn.load(dy + nxt * C, lane);
            if (dy2) g2n.load(dy2 + nxt * ld2, lane);
        }
        const float mean = mean_in[row], rstd = rstd_in[row];
        float xh[PER], g[PER], msk[PER];
        if (drop_p > 0.f) {
            dropout_scale<PER>(msk, seed, row, lane, drop_p);
        } else {
#pragma unroll
            for (int i = 0; i < PER; ++i) msk[i] = 1.f;
        }
        xr.unpack(xh);
        gr.unpack(g);
#pragma unroll
        for (int i = 0; i < PER; ++i) xh[i] *= msk[i];
        if (res) {
            float r2[PER];
            rr.unpack(r2);
#pragma unroll
            for (int i = 0; i < PER; ++i) xh[i] += r2[i];
        }
        if (dy2) {
            float t2[PER];
            g2r.unpack(t2);
#pragma unroll
            for (int i = 0; i < PER; ++i) g[i] += t2[i];
        }
#pragma unroll
        for (int i = 0; i < PER; ++i) xh[i] = (xh[i] - mean) * rstd;
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            const float gg = g[i] * gam[i];
            s1 += gg; s2 += gg * xh[i];
            adg[i] += g[i] * xh[i]; adb[i] += g[i];
        }
        s1 = warp_sum(s1) * (1.f / C); s2 = warp_sum(s2) * (1.f / C);
#pragma unroll
        for (int i = 0; i < PER; i += VEC) {
            const int c = (i / VEC) * 32 * VEC + lane * VEC;
            float o[VEC], om[VEC];
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                o[k] = rstd * (g[i + k] * gam[i + k] - s1 - xh[i + k] * s2);
                om[k] = o[k] * msk[i + k];
            }
            store_vec<T, VEC>(dx + row * C + c, om);
            if (dres) store_vec<T, VEC>(dres + row * C + c, o);
        }
        xr = xn; rr = rn; gr = gn; g2r = g2n;
    }
    if constexpr (kDet) {
        __shared__ float s_w[kStep][C];
        for (int pass = 0; pass < 2; ++pass) {                 // dgamma, then dbeta
#pragma unroll
            for (int i = 0; i < PER; ++i)
                s_w[warp][(i / VEC) * 32 * VEC + lane * VEC + (i % VEC)] = pass ? adb[i] : adg[i];
            __syncthreads();
            for (int i = threadIdx.x; i < C; i += kEThreads) {
                float t = 0.f;
#pragma unroll
                for (int w = 0; w < kStep; ++w) t += s_w[w][i];
                part[((long long)blockIdx.x * 2 + pass) * C + i] = t;
            }
            __syncthreads();
        }
    } else {
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            const int c = (i / VEC) * 32 * VEC + lane * VEC + (i % VEC);
            atomicAdd(&s_dg[c], adg[i]);
            atomicAdd(&s_db[c], adb[i]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += kEThreads) {
            atomicAdd(dgamma + i, s_dg[i]);
            atomicAdd(dbeta + i, s_db[i]);
        }
    }
}

// Second pass of the deterministic reductions: out[c] += sum over p = 0 .. nparts-1 (in that order) of
// part[p * width + c]; columns [0, C) go to out0, [C, width) to out1.
__global__ void __launch_bounds__(kEThreads)
partials_add_kernel(const float *__restrict__ part, int nparts, int width, int C, float *__restrict__ out0,
                    float *__restrict__ out1) {
    const int c = blockIdx.x * kEThreads + threadIdx.x;
    if (c >= width) return;
    float t = 0.f;
    for (int p = 0; p < nparts; ++p) t += part[(long long)p * width + c];
    if (c < C) out0[c] += t;
    else out1[c - C] += t;
}

// ------------------------------------------------------------------------------------------------
// SCA combine: slots[b,q,:] = inv_count[b,q] * sum over cameras seeing q of out[b*R + r, :]
// and its backward g_out[b*R + r, :] = inv_count[b, q_r] * g_slots[b, q_r, :]
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kEThreads)
sca_combine_fwd(const T *__restrict__ out, const int *__restrict__ pair_of,
                const float *__restrict__ inv_count, T *__restrict__ slots, int B, int Nq, int R,
                int C, int ncam) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    const int per_row = C / VEC;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)B * Nq * per_row) return;
    const int cv = (int)(t % per_row);
    const long long bq = t / per_row;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
    for (int c = 0; c < ncam; ++c) {
        const int r = __ldg(pair_of + (long long)c * Nq + q);
        if (r < 0) continue;
        float v[VEC];
        load_vec<T, VEC>(out + ((long long)b * R + r) * C + cv * VEC, v);
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] += v[k];
    }
    const float ic = inv_count[bq];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] *= ic;
    store_vec<T, VEC>(slots + bq * C + cv * VEC, acc);
}

template <typename T>
__global__ void __launch_bounds__(kEThreads)
sca_combine_bwd(const T *__restrict__ g_slots, const int *__restrict__ pair_q,
                const float *__restrict__ inv_count, T *__restrict__ g_out, int B, int Nq, int R,
                int C) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    const int per_row = C / VEC;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)B * R * per_row) return;
    const int cv = (int)(t % per_row);
    const long long br = t / per_row;
    const int r = (int)(br % R), b = (int)(br / R);
    const int q = __ldg(pair_q + r);
    if (q < 0) return;                                // unused row of a fixed-capacity pair list
    const float ic = inv_count[(long long)b * Nq + q];
    float v[VEC];
    load_vec<T, VEC>(g_slots + ((long long)b * Nq + q) * C + cv * VEC, v);
#pragma unroll
    for (int k = 0; k < VEC; ++k) v[k] *= ic;
    store_vec<T, VEC>(g_out + br * C + cv * VEC, v);
}

// ------------------------------------------------------------------------------------------------
// point sampling: lidar -> image projection of the pillar anchors + in-view mask, fp32
// ------------------------------------------------------------------------------------------------
struct PointSamplingParams {
    float pc[6];
    float zs[16];      // normalised pillar heights (D of them)
    float img_h, img_w;
};

__global__ void __launch_bounds__(kEThreads)
point_sampling_kernel(const float *__restrict__ lidar2img, PointSamplingParams prm,
                      float *__restrict__ ref_cam, unsigned char *__restrict__ mask, int B,
                      int ncam, int H, int W, int D) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int Nq = H * W;
    const long long total = (long long)ncam * B * Nq * D;
    if (t >= total) return;
    const int d = (int)(t % D);
    long long u = t / D;
    const int q = (int)(u % Nq); u /= Nq;
    const int b = (int)(u % B);
    const int cam = (int)(u / B);
    const int i = q / W, j = q % W;
    // reference points exactly as torch.linspace(0.5, n - 0.5, n) / n builds them (encoder.py:62-67): an IEEE
    // division, not the approximate one --use_fast_math gives a plain '/'
    const float xn = __fdiv_rn((float)j + 0.5f, (float)W), yn = __fdiv_rn((float)i + 0.5f, (float)H), zn = prm.zs[d];
    const float X = xn * (prm.pc[3] - prm.pc[0]) + prm.pc[0];
    const float Y = yn * (prm.pc[4] - prm.pc[1]) + prm.pc[1];
    const float Z = zn * (prm.pc[5] - prm.pc[2]) + prm.pc[2];
    const float *m4 = lidar2img + ((long long)b * ncam + cam) * 16;
    // plain (non-fused) fp32 multiply-adds in row order, like a 4x4 @ 4x1 matmul with TF32 off
    const float cx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m4[0], X), __fmul_rn(m4[1], Y)), __fmul_rn(m4[2], Z)), m4[3]);
    const float cy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m4[4], X), __fmul_rn(m4[5], Y)), __fmul_rn(m4[6], Z)), m4[7]);
    const float cz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m4[8], X), __fmul_rn(m4[9], Y)), __fmul_rn(m4[10], Z)), m4[11]);
    const float eps = 1e-5f;
    bool ok = cz > eps;
    const float dz = fmaxf(cz, eps);
    const float px = __fdiv_rn(__fdiv_rn(cx, dz), prm.img_w), py = __fdiv_rn(__fdiv_rn(cy, dz), prm.img_h);
    ok = ok && (py > 0.f) && (py < 1.f) && (px < 1.f) && (px > 0.f);
    const long long o = (((long long)cam * B + b) * Nq + q) * D + d;
    reinterpret_cast<float2 *>(ref_cam)[o] = make_float2(px, py);
    mask[o] = ok ? 1 : 0;
}


// ------------------------------------------------------------------------------------------------
// Warp-cooperative TSA prep for num_heads == 8: one warp per (b, q); lane = (head m = lane / 4,
// queue entry j = (lane / 2) % 2, half = lane % 2); a lane owns PPL = L*P/2 points; the softmax over
// the L*P points of one (head, queue entry) reduces over the lane pair.
// ------------------------------------------------------------------------------------------------
template <int PPL, bool kBackward, typename TO>
__global__ void __launch_bounds__(kEThreads)
tsa_prep_m8(const float *__restrict__ raw, const float *__restrict__ ref2d,
            const float *__restrict__ grad_loc, const float *__restrict__ grad_attn,
            const int64_t *__restrict__ level_hw, float *__restrict__ loc, float *__restrict__ attn,
            TO *__restrict__ d_raw, int B, int Nq, int L, int P, int pmagic, int interleave) {
    constexpr int M = 8;
    __shared__ float s_w[16], s_h[16];
    if ((int)threadIdx.x < L) { s_h[threadIdx.x] = (float)level_hw[2 * threadIdx.x]; s_w[threadIdx.x] = (float)level_hw[2 * threadIdx.x + 1]; }
    __syncthreads();
    const int lane = threadIdx.x & 31, m = lane >> 2, j = (lane >> 1) & 1, half = lane & 1;
    const long long bq = (long long)blockIdx.x * (kEThreads / 32) + (threadIdx.x >> 5);
    if (bq >= (long long)B * Nq) return;
    const int q = (int)(bq % Nq), b = (int)(bq / Nq);
    const int LP = 2 * PPL, k0 = half * PPL;
    const long long rbase = bq * (M * 2 * LP * 3);
    const long long o_off = rbase + ((m * 2 + j) * LP + k0) * 2;
    const long long o_lg = rbase + M * 2 * LP * 2 + (m * 2 + j) * LP + k0;
    const long long orow = ((long long)b * 2 + j) * Nq + q;            // row of ref2d (frame-major)
    // output rows: frame-major (b, j, q) like the reference, or interleaved (b, q, j) so that the two
    // frames of a query are adjacent and their mean folds into the output projection
    const long long out_row = interleave ? (((long long)b * Nq + q) * 2 + j) : orow;
    const long long o_out = (out_row * M + m) * LP + k0;
    float a[PPL];
    ldv<PPL>(raw + o_lg, a);
    float mx = a[0];
#pragma unroll
    for (int i = 1; i < PPL; ++i) mx = fmaxf(mx, a[i]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PPL; ++i) { a[i] = exp_rn(a[i] - mx); sum += a[i]; }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    const float inv = __frcp_rn(sum);
#pragma unroll
    for (int i = 0; i < PPL; ++i) a[i] *= inv;
    if constexpr (!kBackward) {
        float off[2 * PPL];
        ldv<2 * PPL>(raw + o_off, off);
        const float *rf = ref2d + orow * L * 2;
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
            const int l = ((k0 + i) * pmagic) >> 16;
            off[2 * i] = __ldg(rf + 2 * l) + __fdiv_rn(off[2 * i], s_w[l]);
            off[2 * i + 1] = __ldg(rf + 2 * l + 1) + __fdiv_rn(off[2 * i + 1], s_h[l]);
        }
        stv<2 * PPL>(loc + 2 * o_out, off);
        stv<PPL>(attn + o_out, a);
    } else {
        float ga[PPL], gl[2 * PPL];
        ldv<PPL>(grad_attn + o_out, ga);
        ldv<2 * PPL>(grad_loc + 2 * o_out, gl);
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < PPL; ++i) dot += a[i] * ga[i];
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
            const int l = ((k0 + i) * pmagic) >> 16;
            ga[i] = a[i] * (ga[i] - dot);
            gl[2 * i] = __fdiv_rn(gl[2 * i], s_w[l]);
            gl[2 * i + 1] = __fdiv_rn(gl[2 * i + 1], s_h[l]);
        }
        stv<PPL>(d_raw + o_lg, ga);
        stv<2 * PPL>(d_raw + o_off, gl);
    }
}


// ------------------------------------------------------------------------------------------------
// Camera features of one pyramid level, (bs, ncam, C, h*w) as the backbone/FPN emits them, into the
// encoder's (ncam, S, bs, C) layout with the camera and level embeddings added on the way
// (PerceptionTransformer.get_bev_features, transformer.py:161-181: flatten, permute, two broadcast
// adds, cat over the levels, permute = five passes over the 95 MB tensor at base; here one).
// 32 x 32 tiles through shared memory: reads run along h*w, writes along C.
// The two adds round like the reference's tensor adds (embedding cast to T, sum rounded to T).
// ------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float round_to(float v);
template <> __device__ __forceinline__ float round_to<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_to<bf16>(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<bf16>(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(256)
flatten_feats_kernel(const T *__restrict__ feat, const float *__restrict__ cams_embeds,
                     const float *__restrict__ level_embed, T *__restrict__ out, int bs, int ncam, int C,
                     int hw, int S, int level_start) {
    __shared__ float tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int b = blockIdx.z / ncam, cam = blockIdx.z % ncam;
    const T *in = feat + ((long long)(b * ncam + cam) * C) * hw;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + ty + 8 * k, p = p0 + tx;
        if (c < C && p < hw) tile[ty + 8 * k][tx] = to_f<T>(in[(long long)c * hw + p]);
    }
    __syncthreads();
    const int c = c0 + tx;
    if (c >= C) return;
    const float ce = cams_embeds ? round_to<T>(cams_embeds[cam * C + c]) : 0.f;
    const float le = round_to<T>(level_embed[c]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int p = p0 + ty + 8 * k;
        if (p >= hw) continue;
        float v = tile[tx][ty + 8 * k];
        if (cams_embeds) v = round_to<T>(v + ce);
        v = v + le;
        out[(((long long)cam * S + level_start + p) * bs + b) * C + c] = from_f<T>(v);
    }
}

template <bool kBackward, typename TO>
static bool launch_tsa_prep_m8(const float *raw, const float *ref2d, const float *grad_loc,
                               const float *grad_attn, const int64_t *level_hw, float *loc, float *attn,
                               TO *d_raw, int B, int Nq, int M, int L, int P, int interleave,
                               cudaStream_t st) {
    const int LP = L * P;
    if (!(M == 8 && L <= 16 && LP * P < 65536 && (LP == 2 || LP == 4 || LP == 8 || LP == 16 || LP == 32)))
        return false;
    const int pmagic = (65536 + P - 1) / P;
    const unsigned grid = (unsigned)(((long long)B * Nq + kEThreads / 32 - 1) / (kEThreads / 32));
#define BEVF_TSA_CASE(N) tsa_prep_m8<N, kBackward, TO><<<grid, kEThreads, 0, st>>>(raw, ref2d, grad_loc, grad_attn, level_hw, loc, attn, d_raw, B, Nq, L, P, pmagic, interleave)
    switch (LP / 2) {
        case 1: BEVF_TSA_CASE(1); break;
        case 2: BEVF_TSA_CASE(2); break;
        case 4: BEVF_TSA_CASE(4); break;
        case 8: BEVF_TSA_CASE(8); break;
        default: BEVF_TSA_CASE(16); break;
    }
#undef BEVF_TSA_CASE
    return true;
}

}  // namespace bevf

using namespace bevf;

#define BEVF_REQUIRE(cond, who, msg) do { if (!(cond)) return fail("%s: " msg, who); } while (0)

static inline unsigned blocks_for(long long n, int per) { return (unsigned)((n + per - 1) / per); }

extern "C" int bevf_sca_prep_forward(const float *raw, const float *ref_cam, const int32_t *pair_q,
                                     const int32_t *pair_cam, const int64_t *level_hw, float *loc,
                                     float *attn, int B, int Nq, int R, int M, int L, int P, int D,
                                     int ncam, void *stream) {
    const char *who = "bevf_sca_prep_forward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && R >= 0 && M > 0 && L > 0 && P > 0 && D > 0 && ncam > 0, who, "bad dimension");
    BEVF_REQUIRE(P % D == 0, who, "num_points must be a multiple of the number of Z anchors");
    const long long total = (long long)B * R * M;
    if (total == 0) return 0;
    BEVF_REQUIRE(raw && ref_cam && pair_q && pair_cam && level_hw && loc && attn, who, "null pointer argument");
    const int LP = L * P, pmagic = (65536 + P - 1) / P;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned wgrid = blocks_for((long long)B * R, kEThreads / 32);
    if (M == 8 && L <= 16 && LP * P < 65536 && (LP == 4 || LP == 8 || LP == 16 || LP == 32 || LP == 64)) {
        switch (LP / 4) {
            case 1: sca_prep_fwd_m8<1><<<wgrid, kEThreads, 0, st>>>(raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, L, P, D, pmagic); break;
            case 2: sca_prep_fwd_m8<2><<<wgrid, kEThreads, 0, st>>>(raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, L, P, D, pmagic); break;
            case 4: sca_prep_fwd_m8<4><<<wgrid, kEThreads, 0, st>>>(raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, L, P, D, pmagic); break;
            case 8: sca_prep_fwd_m8<8><<<wgrid, kEThreads, 0, st>>>(raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, L, P, D, pmagic); break;
            default: sca_prep_fwd_m8<16><<<wgrid, kEThreads, 0, st>>>(raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, L, P, D, pmagic); break;
        }
    } else {
        sca_prep_fwd<<<blocks_for(total, kEThreads), kEThreads, 0, st>>>(
            raw, ref_cam, pair_q, pair_cam, level_hw, loc, attn, B, Nq, R, M, L, P, D, ncam);
    }
    return check_launch(who);
}

template <typename TO>
static int sca_prep_backward_t(const char *who, const float *raw, const float *grad_loc, const float *grad_attn,
                               const int32_t *pair_of, const int64_t *level_hw, TO *d_raw, int B, int Nq,
                               int R, int M, int L, int P, int ncam, cudaStream_t st) {
    const long long total = (long long)B * Nq * M;
    const int LP = L * P, pmagic = (65536 + P - 1) / P;
    const unsigned wgrid = blocks_for((long long)B * Nq, kEThreads / 32);
    if (M == 8 && L <= 16 && LP * P < 65536 && (LP == 4 || LP == 8 || LP == 16 || LP == 32 || LP == 64)) {
#define BEVF_SCA_CASE(N) sca_prep_bwd_m8<N, TO><<<wgrid, kEThreads, 0, st>>>(raw, grad_loc, grad_attn, pair_of, level_hw, d_raw, B, Nq, R, L, P, ncam, pmagic)
        switch (LP / 4) {
            case 1: BEVF_SCA_CASE(1); break;
            case 2: BEVF_SCA_CASE(2); break;
            case 4: BEVF_SCA_CASE(4); break;
            case 8: BEVF_SCA_CASE(8); break;
            default: BEVF_SCA_CASE(16); break;
        }
#undef BEVF_SCA_CASE
    } else {
        sca_prep_bwd<TO><<<blocks_for(total, kEThreads), kEThreads, 0, st>>>(
            raw, grad_loc, grad_attn, pair_of, level_hw, d_raw, B, Nq, R, M, L, P, ncam);
    }
    return check_launch(who);
}

extern "C" int bevf_sca_prep_backward(const float *raw, const float *grad_loc,
                                      const float *grad_attn, const int32_t *pair_of,
                                      const int64_t *level_hw, void *d_raw, int out_dtype, int B, int Nq,
                                      int R, int M, int L, int P, int ncam, void *stream) {
    const char *who = "bevf_sca_prep_backward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && R >= 0 && M > 0 && L > 0 && P > 0 && ncam > 0 && ncam <= 16, who, "bad dimension (ncam <= 16)");
    BEVF_REQUIRE(out_dtype == BEVF_DTYPE_F32 || out_dtype == BEVF_DTYPE_BF16, who, "unsupported dtype code");
    if ((long long)B * Nq * M == 0) return 0;
    BEVF_REQUIRE(raw && pair_of && level_hw && d_raw && (R == 0 || (grad_loc && grad_attn)), who, "null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (out_dtype == BEVF_DTYPE_BF16)
        return sca_prep_backward_t<bf16>(who, raw, grad_loc, grad_attn, pair_of, level_hw, (bf16 *)d_raw, B, Nq, R, M, L, P, ncam, st);
    return sca_prep_backward_t<float>(who, raw, grad_loc, grad_attn, pair_of, level_hw, (float *)d_raw, B, Nq, R, M, L, P, ncam, st);
}

extern "C" int bevf_tsa_prep_forward(const float *raw, const float *ref2d, const int64_t *level_hw,
                                     float *loc, float *attn, int B, int Nq, int M, int L, int P,
                                     int interleave, void *stream) {
    const char *who = "bevf_tsa_prep_forward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && M > 0 && L > 0 && P > 0, who, "bad dimension");
    const long long total = (long long)B * Nq * M * 2;
    if (total == 0) return 0;
    BEVF_REQUIRE(raw && ref2d && level_hw && loc && attn, who, "null pointer argument");
    if (!launch_tsa_prep_m8<false, float>(raw, ref2d, nullptr, nullptr, level_hw, loc, attn, nullptr, B, Nq, M, L, P,
                                   interleave, (cudaStream_t)stream)) {
        if (interleave) return fail("%s: interleaved rows need num_heads == 8 and L*P in {2,4,8,16,32}", who);
        tsa_prep_fwd<<<blocks_for(total, kEThreads), kEThreads, 0, (cudaStream_t)stream>>>(
            raw, ref2d, level_hw, loc, attn, B, Nq, M, L, P);
    }
    return check_launch(who);
}

template <typename TO>
static int tsa_prep_backward_t(const char *who, const float *raw, const float *grad_loc, const float *grad_attn,
                               const int64_t *level_hw, TO *d_raw, int B, int Nq, int M, int L, int P,
                               int interleave, cudaStream_t st) {
    const long long total = (long long)B * Nq * M * 2;
    if (!launch_tsa_prep_m8<true, TO>(raw, nullptr, grad_loc, grad_attn, level_hw, nullptr, nullptr, d_raw, B, Nq, M,
                                      L, P, interleave, st)) {
        if (interleave) return fail("%s: interleaved rows need num_heads == 8 and L*P in {2,4,8,16,32}", who);
        tsa_prep_bwd<TO><<<blocks_for(total, kEThreads), kEThreads, 0, st>>>(
            raw, grad_loc, grad_attn, level_hw, d_raw, B, Nq, M, L, P);
    }
    return check_launch(who);
}

extern "C" int bevf_tsa_prep_backward(const float *raw, const float *grad_loc,
                                      const float *grad_attn, const int64_t *level_hw, void *d_raw,
                                      int out_dtype, int B, int Nq, int M, int L, int P, int interleave,
                                      void *stream) {
    const char *who = "bevf_tsa_prep_backward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && M > 0 && L > 0 && P > 0, who, "bad dimension");
    BEVF_REQUIRE(out_dtype == BEVF_DTYPE_F32 || out_dtype == BEVF_DTYPE_BF16, who, "unsupported dtype code");
    if ((long long)B * Nq * M * 2 == 0) return 0;
    BEVF_REQUIRE(raw && grad_loc && grad_attn && level_hw && d_raw, who, "null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (out_dtype == BEVF_DTYPE_BF16)
        return tsa_prep_backward_t<bf16>(who, raw, grad_loc, grad_attn, level_hw, (bf16 *)d_raw, B, Nq, M, L, P, interleave, st);
    return tsa_prep_backward_t<float>(who, raw, grad_loc, grad_attn, level_hw, (float *)d_raw, B, Nq, M, L, P, interleave, st);
}

template <typename T, typename TP>
static int ln_fwd_t(const char *who, const void *x, const void *res, const void *gamma, const void *beta,
                    const void *pos, void *y, void *y2, float *mean, float *rstd, long long rows, int C,
                    float eps, float drop_p, unsigned long long seed, const unsigned long long *sb,
                    cudaStream_t st) {
    const unsigned grid = blocks_for(rows, (kEThreads / 32) * kLnRowsPerWarp);
    if (C == 256)
        layernorm_fwd<T, TP, 256><<<grid, kEThreads, 0, st>>>((const T *)x, (const T *)res, (const TP *)gamma, (const TP *)beta, (const T *)pos, (T *)y, (T *)y2, mean, rstd, rows, eps, drop_p, seed, sb);
    else if (C == 512)
        layernorm_fwd<T, TP, 512><<<grid, kEThreads, 0, st>>>((const T *)x, (const T *)res, (const TP *)gamma, (const TP *)beta, (const T *)pos, (T *)y, (T *)y2, mean, rstd, rows, eps, drop_p, seed, sb);
    else
        return fail("%s: embed_dims must be 256 or 512", who);
    return check_launch(who);
}

extern "C" int bevf_layernorm_forward(const void *x, const void *residual, const void *gamma,
                                      const void *beta, int param_dtype, const void *pos, void *y,
                                      void *y_plus_pos, float *mean, float *rstd, int64_t rows, int C,
                                      float eps, float drop_p, uint64_t seed, const uint64_t *seed_base,
                                      int dtype, void *stream) {
    const char *who = "bevf_layernorm_forward";
    const unsigned long long *sb = reinterpret_cast<const unsigned long long *>(seed_base);
    BEVF_REQUIRE(rows >= 0 && C > 0, who, "bad dimension");
    if (rows == 0) return 0;
    BEVF_REQUIRE(x && gamma && beta && y, who, "null pointer argument");
    BEVF_REQUIRE((y_plus_pos == nullptr) == (pos == nullptr), who, "pos and y_plus_pos go together");
    BEVF_REQUIRE(drop_p >= 0.f && drop_p < 1.f, who, "dropout probability must be in [0, 1)");
    cudaStream_t st = (cudaStream_t)stream;
    const bool pb = param_dtype == BEVF_DTYPE_BF16;
    BEVF_REQUIRE(pb || param_dtype == BEVF_DTYPE_F32, who, "unsupported parameter dtype code");
    if (dtype == BEVF_DTYPE_F32) {
        if (pb) return fail("%s: bf16 parameters with fp32 activations are not supported", who);
        return ln_fwd_t<float, float>(who, x, residual, gamma, beta, pos, y, y_plus_pos, mean, rstd, rows, C, eps, drop_p, seed, sb, st);
    }
    if (dtype == BEVF_DTYPE_BF16) {
        if (pb) return ln_fwd_t<bf16, bf16>(who, x, residual, gamma, beta, pos, y, y_plus_pos, mean, rstd, rows, C, eps, drop_p, seed, sb, st);
        return ln_fwd_t<bf16, float>(who, x, residual, gamma, beta, pos, y, y_plus_pos, mean, rstd, rows, C, eps, drop_p, seed, sb, st);
    }
    return fail("%s: unsupported dtype code", who);
}

// rows per CTA and grid of the LayerNorm backward, shared by the launch and the workspace query
static unsigned ln_bwd_plan(long long rows, int &rows_per_cta) {
    // ~4 CTAs per SM worth of row chunks keeps the per-channel atomics few
    rows_per_cta = (int)((rows + device_sms() * 4 - 1) / (device_sms() * 4));
    rows_per_cta = ((rows_per_cta + 7) / 8) * 8;
    if (rows_per_cta < 8) rows_per_cta = 8;
    return blocks_for(rows, rows_per_cta);
}

template <typename T, typename TP>
static int ln_bwd_t(const char *who, const void *x, const void *res, const void *gamma, const float *mean,
                    const float *rstd, const void *dy, const void *dy2, void *dx, void *dres, float *dgamma,
                    float *dbeta, long long rows, int C, float drop_p, unsigned long long seed,
                    const unsigned long long *sb, long long ld2, cudaStream_t st, float *part = nullptr) {
    int rows_per_cta;
    const unsigned grid = ln_bwd_plan(rows, rows_per_cta);
    if (C != 256 && C != 512) return fail("%s: embed_dims must be 256 or 512", who);
    auto kernel = C == 256 ? (part ? layernorm_bwd<T, TP, 256, true> : layernorm_bwd<T, TP, 256, false>)
                           : (part ? layernorm_bwd<T, TP, 512, true> : layernorm_bwd<T, TP, 512, false>);
    kernel<<<grid, kEThreads, 0, st>>>((const T *)x, (const T *)res, (const TP *)gamma, mean, rstd, (const T *)dy,
                                       (const T *)dy2, (T *)dx, (T *)dres, dgamma, dbeta, rows, rows_per_cta, drop_p, seed,
                                       sb, ld2, part);
    if (int e = check_launch(who)) return e;
    if (part) {
        partials_add_kernel<<<(unsigned)((2 * C + kEThreads - 1) / kEThreads), kEThreads, 0, st>>>(part, (int)grid, 2 * C,
                                                                                                   C, dgamma, dbeta);
        return check_launch(who);
    }
    return 0;
}

static int layernorm_backward_impl(const char *who, const void *x, const void *residual, const void *gamma,
                                   int param_dtype, const float *mean, const float *rstd, const void *dy,
                                   const void *dy_plus_pos, int64_t dy_plus_pos_ld, void *dx, void *dres, float *dgamma,
                                   float *dbeta, int64_t rows, int C, float drop_p, uint64_t seed,
                                   const uint64_t *seed_base, int dtype, void *stream, float *part = nullptr) {
    const unsigned long long *sb = reinterpret_cast<const unsigned long long *>(seed_base);
    BEVF_REQUIRE(rows >= 0 && C > 0, who, "bad dimension");
    if (rows == 0) return 0;
    BEVF_REQUIRE(x && gamma && mean && rstd && dy && dx && dgamma && dbeta, who, "null pointer argument");
    const long long ld2 = dy_plus_pos_ld > 0 ? (long long)dy_plus_pos_ld : (long long)C;
    BEVF_REQUIRE(ld2 >= C && ld2 % (dtype == BEVF_DTYPE_BF16 ? 8 : 4) == 0, who, "bad row stride of dy_plus_pos");
    BEVF_REQUIRE(drop_p == 0.f || dres != nullptr || residual == nullptr, who, "dropout with a residual needs a separate dres buffer");
    cudaStream_t st = (cudaStream_t)stream;
    const bool pb = param_dtype == BEVF_DTYPE_BF16;
    BEVF_REQUIRE(pb || param_dtype == BEVF_DTYPE_F32, who, "unsupported parameter dtype code");
    if (dtype == BEVF_DTYPE_F32) {
        if (pb) return fail("%s: bf16 parameters with fp32 activations are not supported", who);
        return ln_bwd_t<float, float>(who, x, residual, gamma, mean, rstd, dy, dy_plus_pos, dx, dres, dgamma, dbeta, rows, C, drop_p, seed, sb, ld2, st, part);
    }
    if (dtype == BEVF_DTYPE_BF16) {
        if (pb) return ln_bwd_t<bf16, bf16>(who, x, residual, gamma, mean, rstd, dy, dy_plus_pos, dx, dres, dgamma, dbeta, rows, C, drop_p, seed, sb, ld2, st, part);
        return ln_bwd_t<bf16, float>(who, x, residual, gamma, mean, rstd, dy, dy_plus_pos, dx, dres, dgamma, dbeta, rows, C, drop_p, seed, sb, ld2, st, part);
    }
    return fail("%s: unsupported dtype code", who);
}

extern "C" int bevf_layernorm_backward(const void *x, const void *residual, const void *gamma,
                                       int param_dtype, const float *mean, const float *rstd,
                                       const void *dy, const void *dy_plus_pos, int64_t dy_plus_pos_ld, void *dx,
                                       void *dres,
                                       float *dgamma, float *dbeta, int64_t rows, int C, float drop_p,
                                       uint64_t seed, const uint64_t *seed_base, int dtype,
                                       void *stream) {
    return layernorm_backward_impl("bevf_layernorm_backward", x, residual, gamma, param_dtype, mean, rstd, dy,
                                   dy_plus_pos, dy_plus_pos_ld, dx, dres, dgamma, dbeta, rows, C, drop_p, seed,
                                   seed_base, dtype, stream);
}

extern "C" int64_t bevf_layernorm_backward_workspace_bytes(int64_t rows, int C) {
    if (rows <= 0 || C <= 0) return 0;
    int rows_per_cta;
    return (int64_t)ln_bwd_plan(rows, rows_per_cta) * 2 * C * sizeof(float);
}

extern "C" int bevf_layernorm_backward_det(const void *x, const void *residual, const void *gamma,
                                           int param_dtype, const float *mean, const float *rstd,
                                           const void *dy, const void *dy_plus_pos, int64_t dy_plus_pos_ld, void *dx,
                                           void *dres, float *dgamma, float *dbeta, void *workspace,
                                           int64_t workspace_bytes, int64_t rows, int C, float drop_p, uint64_t seed,
                                           const uint64_t *seed_base, int dtype, void *stream) {
    const char *who = "bevf_layernorm_backward_det";
    if (rows <= 0) return layernorm_backward_impl(who, x, residual, gamma, param_dtype, mean, rstd, dy, dy_plus_pos,
                                                  dy_plus_pos_ld, dx, dres, dgamma, dbeta, rows, C, drop_p, seed,
                                                  seed_base, dtype, stream);
    BEVF_REQUIRE(workspace && aligned16(workspace), who, "workspace must be a 16-byte aligned device buffer");
    const int64_t need = bevf_layernorm_backward_workspace_bytes(rows, C);
    if (workspace_bytes < need) return fail("%s: workspace too small (need %lld bytes)", who, need);
    return layernorm_backward_impl(who, x, residual, gamma, param_dtype, mean, rstd, dy, dy_plus_pos, dy_plus_pos_ld,
                                   dx, dres, dgamma, dbeta, rows, C, drop_p, seed, seed_base, dtype, stream,
                                   reinterpret_cast<float *>(workspace));
}

extern "C" int bevf_sca_combine_forward(const void *out, const int32_t *pair_of,
                                        const float *inv_count, void *slots, int B, int Nq, int R,
                                        int C, int ncam, int dtype, void *stream) {
    const char *who = "bevf_sca_combine_forward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && R >= 0 && C > 0 && C % 8 == 0 && ncam > 0, who, "bad dimension");
    if ((long long)B * Nq == 0) return 0;
    BEVF_REQUIRE(pair_of && inv_count && slots && (R == 0 || out), who, "null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_F32) {
        sca_combine_fwd<float><<<blocks_for((long long)B * Nq * (C / 4), kEThreads), kEThreads, 0, st>>>((const float *)out, pair_of, inv_count, (float *)slots, B, Nq, R, C, ncam);
    } else if (dtype == BEVF_DTYPE_BF16) {
        sca_combine_fwd<bf16><<<blocks_for((long long)B * Nq * (C / 8), kEThreads), kEThreads, 0, st>>>((const bf16 *)out, pair_of, inv_count, (bf16 *)slots, B, Nq, R, C, ncam);
    } else {
        return fail("%s: unsupported dtype code", who);
    }
    return check_launch(who);
}

extern "C" int bevf_sca_combine_backward(const void *g_slots, const int32_t *pair_q,
                                         const float *inv_count, void *g_out, int B, int Nq, int R,
                                         int C, int dtype, void *stream) {
    const char *who = "bevf_sca_combine_backward";
    BEVF_REQUIRE(B >= 0 && Nq >= 0 && R >= 0 && C > 0 && C % 8 == 0, who, "bad dimension");
    if ((long long)B * R == 0) return 0;
    BEVF_REQUIRE(g_slots && pair_q && inv_count && g_out, who, "null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_F32) {
        sca_combine_bwd<float><<<blocks_for((long long)B * R * (C / 4), kEThreads), kEThreads, 0, st>>>((const float *)g_slots, pair_q, inv_count, (float *)g_out, B, Nq, R, C);
    } else if (dtype == BEVF_DTYPE_BF16) {
        sca_combine_bwd<bf16><<<blocks_for((long long)B * R * (C / 8), kEThreads), kEThreads, 0, st>>>((const bf16 *)g_slots, pair_q, inv_count, (bf16 *)g_out, B, Nq, R, C);
    } else {
        return fail("%s: unsupported dtype code", who);
    }
    return check_launch(who);
}

extern "C" int bevf_point_sampling(const float *lidar2img, const float *pc_range,
                                   const float *z_norm, float img_h, float img_w, float *ref_cam,
                                   uint8_t *bev_mask, int B, int ncam, int bev_h, int bev_w, int D,
                                   void *stream) {
    const char *who = "bevf_point_sampling";
    BEVF_REQUIRE(B >= 0 && ncam > 0 && bev_h > 0 && bev_w > 0 && D > 0 && D <= 16, who, "bad dimension (D <= 16)");
    const long long total = (long long)ncam * B * bev_h * bev_w * D;
    if (total == 0) return 0;
    BEVF_REQUIRE(lidar2img && pc_range && z_norm && ref_cam && bev_mask, who, "null pointer argument");
    PointSamplingParams prm;
    for (int i = 0; i < 6; ++i) prm.pc[i] = pc_range[i];     // HOST arrays
    for (int i = 0; i < D; ++i) prm.zs[i] = z_norm[i];
    prm.img_h = img_h; prm.img_w = img_w;
    point_sampling_kernel<<<blocks_for(total, kEThreads), kEThreads, 0, (cudaStream_t)stream>>>(
        lidar2img, prm, ref_cam, bev_mask, B, ncam, bev_h, bev_w, D);
    return check_launch(who);
}

extern "C" int bevf_flatten_feats(const void *feat, const float *cams_embeds, const float *level_embed,
                                  void *out, int bs, int ncam, int C, int hw, int S, int level_start,
                                  int dtype, void *stream) {
    const char *who = "bevf_flatten_feats";
    BEVF_REQUIRE(bs >= 0 && ncam > 0 && C > 0 && hw >= 0 && S >= 0 && level_start >= 0, who, "bad dimension");
    BEVF_REQUIRE(level_start + hw <= S, who, "the level does not fit the flattened pyramid");
    BEVF_REQUIRE((long long)bs * ncam <= 65535, who, "bs * ncam exceeds the grid limit");
    if ((long long)bs * hw == 0) return 0;
    BEVF_REQUIRE(feat && level_embed && out, who, "null pointer argument");
    const dim3 grid((unsigned)((hw + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)(bs * ncam));
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_F32)
        flatten_feats_kernel<float><<<grid, 256, 0, st>>>((const float *)feat, cams_embeds, level_embed, (float *)out, bs, ncam, C, hw, S, level_start);
    else if (dtype == BEVF_DTYPE_BF16)
        flatten_feats_kernel<bf16><<<grid, 256, 0, st>>>((const bf16 *)feat, cams_embeds, level_embed, (bf16 *)out, bs, ncam, C, hw, S, level_start);
    else
        return fail("%s: unsupported dtype code", who);
    return check_launch(who);
}

// out = sum of up to 8 equally-shaped bf16 / f32 tensors, fp32 accumulation, one pass (the input gradients
// of the layers that share an input: n reads + 1 write instead of n-1 pairwise add kernels)
struct SumPtrs { const void *p[8]; };
template <typename T>
__global__ void __launch_bounds__(kEThreads)
sum_n_kernel(SumPtrs src, int n, T *__restrict__ out, long long vecs) {
    constexpr int VEC = (sizeof(T) == 2) ? 8 : 4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < vecs;
         i += (long long)gridDim.x * blockDim.x) {
        float acc[VEC];
        load_vec<T, VEC>(reinterpret_cast<const T *>(src.p[0]) + i * VEC, acc);
        for (int k = 1; k < n; ++k) {
            float v[VEC];
            load_vec<T, VEC>(reinterpret_cast<const T *>(src.p[k]) + i * VEC, v);
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] += v[j];
        }
        store_vec<T, VEC>(out + i * VEC, acc);
    }
}

extern "C" int bevf_sum_tensors(const void *const *srcs, int n, void *out, int64_t numel, int dtype, void *stream) {
    const char *who = "bevf_sum_tensors";
    BEVF_REQUIRE(n >= 1 && n <= 8 && numel >= 0, who, "1..8 tensors");
    if (numel == 0) return 0;
    BEVF_REQUIRE(srcs && out, who, "null pointer argument");
    BEVF_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F32, who, "unsupported dtype code");
    const int vec = dtype == BEVF_DTYPE_BF16 ? 8 : 4;
    BEVF_REQUIRE(numel % vec == 0, who, "numel must be a multiple of 16 bytes");
    SumPtrs sp;
    for (int k = 0; k < 8; ++k) {
        sp.p[k] = srcs[k < n ? k : 0];
        BEVF_REQUIRE(sp.p[k] && aligned16(sp.p[k]), who, "source pointers must be non-null and 16-byte aligned");
    }
    BEVF_REQUIRE(aligned16(out), who, "out must be 16-byte aligned");
    const long long vecs = numel / vec;
    long long blocks = (vecs + kEThreads - 1) / kEThreads;
    if (blocks > device_sms() * 16) blocks = device_sms() * 16;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_BF16)
        sum_n_kernel<bf16><<<(unsigned)blocks, kEThreads, 0, st>>>(sp, n, (bf16 *)out, vecs);
    else
        sum_n_kernel<float><<<(unsigned)blocks, kEThreads, 0, st>>>(sp, n, (float *)out, vecs);
    return check_launch(who);
}

static unsigned colsum_plan(long long rows, long long &rows_per_cta) {
    rows_per_cta = (rows + device_sms() * 4 - 1) / (device_sms() * 4);
    if (rows_per_cta < 64) rows_per_cta = 64;
    return blocks_for(rows, (int)rows_per_cta);
}

static int colsum_impl(const char *who, const void *x, float *out, int64_t rows, int C, int dtype, void *stream,
                       float *part = nullptr) {
    BEVF_REQUIRE(rows >= 0 && C > 0, who, "bad dimension");
    if (rows == 0) return 0;
    BEVF_REQUIRE(x && out, who, "null pointer argument");
    const int vec = dtype == BEVF_DTYPE_BF16 ? 8 : 4;
    BEVF_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F32, who, "unsupported dtype code");
    BEVF_REQUIRE(C % vec == 0 && C / vec <= kEThreads, who, "C must be a multiple of the vector width and <= 2048");
    long long rows_per_cta;
    const unsigned grid = colsum_plan(rows, rows_per_cta);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sm = (size_t)(kEThreads / (C / vec)) * C * sizeof(float);
    BEVF_REQUIRE(sm <= 48 * 1024, who, "C too large for the row-lane staging");
    if (dtype == BEVF_DTYPE_BF16)
        colsum_kernel<bf16><<<grid, kEThreads, sm, st>>>((const bf16 *)x, out, rows, C, (int)rows_per_cta, part);
    else
        colsum_kernel<float><<<grid, kEThreads, sm, st>>>((const float *)x, out, rows, C, (int)rows_per_cta, part);
    if (int e = check_launch(who)) return e;
    if (part) {
        partials_add_kernel<<<blocks_for(C, kEThreads), kEThreads, 0, st>>>(part, (int)grid, C, C, out, nullptr);
        return check_launch(who);
    }
    return 0;
}

extern "C" int bevf_colsum(const void *x, float *out, int64_t rows, int C, int dtype, void *stream) {
    return colsum_impl("bevf_colsum", x, out, rows, C, dtype, stream);
}

extern "C" int64_t bevf_colsum_workspace_bytes(int64_t rows, int C) {
    if (rows <= 0 || C <= 0) return 0;
    long long rows_per_cta;
    return (int64_t)colsum_plan(rows, rows_per_cta) * C * sizeof(float);
}

extern "C" int bevf_colsum_det(const void *x, float *out, void *workspace, int64_t workspace_bytes, int64_t rows, int C,
                               int dtype, void *stream) {
    const char *who = "bevf_colsum_det";
    if (rows <= 0) return colsum_impl(who, x, out, rows, C, dtype, stream);
    BEVF_REQUIRE(workspace && aligned16(workspace), who, "workspace must be a 16-byte aligned device buffer");
    const int64_t need = bevf_colsum_workspace_bytes(rows, C);
    if (workspace_bytes < need) return fail("%s: workspace too small (need %lld bytes)", who, need);
    return colsum_impl(who, x, out, rows, C, dtype, stream, reinterpret_cast<float *>(workspace));
}

extern "C" int bevf_relu_dropout_backward(const void *dy, const void *h, void *out, int64_t n, float scale,
                                          int dtype, void *stream) {
    const char *who = "bevf_relu_dropout_backward";
    BEVF_REQUIRE(n >= 0, who, "bad dimension");
    if (n == 0) return 0;
    BEVF_REQUIRE(dy && h && out, who, "null pointer argument");
    const int vec = dtype == BEVF_DTYPE_BF16 ? 8 : 4;
    BEVF_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F32, who, "unsupported dtype code");
    BEVF_REQUIRE(n % vec == 0, who, "element count must be a multiple of the vector width");
    const long long nv = n / vec;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BEVF_DTYPE_BF16)
        relu_dropout_bwd_kernel<bf16><<<blocks_for(nv, kEThreads), kEThreads, 0, st>>>((const bf16 *)dy, (const bf16 *)h, (bf16 *)out, nv, scale);
    else
        relu_dropout_bwd_kernel<float><<<blocks_for(nv, kEThreads), kEThreads, 0, st>>>((const float *)dy, (const float *)h, (float *)out, nv, scale);
    return check_launch(who);
}

extern "C" int bevf_dropout_inplace(void *x, int64_t n, float p, uint64_t seed, const uint64_t *seed_base,
                                    int dtype, void *stream) {
    const char *who = "bevf_dropout_inplace";
    BEVF_REQUIRE(n >= 0, who, "bad dimension");
    BEVF_REQUIRE(p >= 0.f && p < 1.f, who, "dropout probability must be in [0, 1)");
    if (n == 0 || p == 0.f) return 0;
    BEVF_REQUIRE(x, who, "null pointer argument");
    const int vec = dtype == BEVF_DTYPE_BF16 ? 8 : 4;
    BEVF_REQUIRE(dtype == BEVF_DTYPE_BF16 || dtype == BEVF_DTYPE_F32, who, "unsupported dtype code");
    BEVF_REQUIRE(n % vec == 0, who, "element count must be a multiple of the vector width");
    const long long nv = n / vec;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned long long *sb = reinterpret_cast<const unsigned long long *>(seed_base);
    if (dtype == BEVF_DTYPE_BF16)
        dropout_inplace_kernel<bf16><<<blocks_for(nv, kEThreads), kEThreads, 0, st>>>((bf16 *)x, nv, p, seed, sb);
    else
        dropout_inplace_kernel<float><<<blocks_for(nv, kEThreads), kEThreads, 0, st>>>((float *)x, nv, p, seed, sb);
    return check_launch(who);
}
