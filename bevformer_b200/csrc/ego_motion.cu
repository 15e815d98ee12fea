// Once-per-frame ego-motion block of PerceptionTransformer.get_bev_features on the device: the BEV shift, the
// CAN-bus MLP input, forward_test's delta state, and the nearest-neighbour rotation of prev_bev.  The reference
// does this arithmetic on the host (numpy float64 + torchvision's rotate); with everything read from and written
// to device memory a video frame has no host arithmetic left and can be captured in a CUDA graph.
//
// Double-precision steps that the host performs as separate IEEE operations are written with the __d*_rn
// intrinsics, which the compiler never contracts into FMAs: the results then differ from numpy's only where
// sin / cos / atan2 themselves do (last bit).
#include "common.cuh"

namespace bevf {

#define BEVF_REQUIRE(cond, who, msg) do { if (!(cond)) return fail("%s: " msg, who); } while (0)

struct EgoState {            // include/bevformer_b200.h: 40 bytes
    double prev_pos[3];
    double prev_angle;
    long long has_history;
};

constexpr double kPi = 3.141592653589793;       // numpy's np.pi and CPython's math.pi

// what torch's Tensor.new_tensor(float64 data) stores: double -> float -> storage type, each round-to-nearest
template <typename TQ> __device__ __forceinline__ TQ round_to(double v);
template <> __device__ __forceinline__ float round_to<float>(double v) { return (float)v; }
template <> __device__ __forceinline__ bf16 round_to<bf16>(double v) { return __float2bfloat16_rn((float)v); }
template <> __device__ __forceinline__ __half round_to<__half>(double v) { return __float2half_rn((float)v); }
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }

struct EgoParams {
    int bs, bev_h, bev_w, use_shift, mode;
    double grid_h, grid_w, center_x, center_y;
};

// one thread per sample; the stream state belongs to sample 0 (forward_test edits img_metas[0] only)
template <typename TQ>
__global__ void ego_motion_kernel(const double *__restrict__ can_bus, EgoState *__restrict__ state,
                                  float *__restrict__ shift, float *__restrict__ rot, TQ *__restrict__ mlp_in,
                                  EgoParams p) {
    for (int b = threadIdx.x; b < p.bs; b += blockDim.x) {
        double cb[18];
#pragma unroll
        for (int i = 0; i < 18; ++i) cb[i] = can_bus[b * 18 + i];
        if (b == 0 && p.mode != BEVF_EGO_DELTAS) {            // detectors/bevformer.py:254-268
            const double px = cb[0], py = cb[1], pz = cb[2], pa = cb[17];
            if (p.mode == BEVF_EGO_CONTINUE && state->has_history) {
                cb[0] = __dsub_rn(cb[0], state->prev_pos[0]);
                cb[1] = __dsub_rn(cb[1], state->prev_pos[1]);
                cb[2] = __dsub_rn(cb[2], state->prev_pos[2]);
                cb[17] = __dsub_rn(cb[17], state->prev_angle);
            } else {
                cb[0] = 0.0; cb[1] = 0.0; cb[2] = 0.0; cb[17] = 0.0;
            }
            state->prev_pos[0] = px; state->prev_pos[1] = py; state->prev_pos[2] = pz;
            state->prev_angle = pa;
            state->has_history = 1;
        }
#pragma unroll
        for (int i = 0; i < 18; ++i) mlp_in[b * 18 + i] = round_to<TQ>(cb[i]);

        // shift (transformer.py:122-140), operation by operation as numpy evaluates it
        const double dx = cb[0], dy = cb[1];
        const double ego = __dmul_rn(__ddiv_rn(cb[16], kPi), 180.0);
        const double length = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        const double bev_angle = __dsub_rn(ego, __dmul_rn(__ddiv_rn(atan2(dy, dx), kPi), 180.0));
        const double ang = __dmul_rn(__ddiv_rn(bev_angle, 180.0), kPi);
        const double sy = __ddiv_rn(__ddiv_rn(__dmul_rn(length, cos(ang)), p.grid_h), (double)p.bev_h);
        const double sx = __ddiv_rn(__ddiv_rn(__dmul_rn(length, sin(ang)), p.grid_w), (double)p.bev_w);
        const double use = p.use_shift ? 1.0 : 0.0;
        shift[b * 2] = widen(round_to<TQ>(__dmul_rn(sx, use)));
        shift[b * 2 + 1] = widen(round_to<TQ>(__dmul_rn(sy, use)));

        // torchvision rotate(img, angle, center): _get_inverse_affine_matrix(center_f, -angle, [0, 0], 1, [0, 0])
        // without shear is [cos, sin, tx, -sin, cos, ty]; then float32 and _gen_affine_grid's division
        const double cx = __dsub_rn(p.center_x, __dmul_rn((double)p.bev_w, 0.5));
        const double cy = __dsub_rn(p.center_y, __dmul_rn((double)p.bev_h, 0.5));
        const double r = __dmul_rn(-cb[17], kPi / 180.0);       // math.radians
        const double c = cos(r), s = sin(r);
        const double m0 = c, m1 = s, m3 = -s, m4 = c;
        const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(m0, -cx), __dmul_rn(m1, -cy)), cx);
        const double m5 = __dadd_rn(__dadd_rn(__dmul_rn(m3, -cx), __dmul_rn(m4, -cy)), cy);
        const float hw = 0.5f * (float)p.bev_w, hh = 0.5f * (float)p.bev_h;
        float *o = rot + b * 6;
        o[0] = __fdiv_rn((float)m0, hw); o[1] = __fdiv_rn((float)m1, hw); o[2] = __fdiv_rn((float)m2, hw);
        o[3] = __fdiv_rn((float)m3, hh); o[4] = __fdiv_rn((float)m4, hh); o[5] = __fdiv_rn((float)m5, hh);
    }
}

// ------------------------------------------------------------------------------------------------
// prev_bev rotated in one pass: out[q, b, :] = prev[src(q, b), b, :] or 0.  One warp per output row (a cell's C
// channels), 16-byte loads and stores, grid-stride over the rows.  The source cell is computed in fp32 whatever
// the storage type, in the order torchvision + grid_sample(mode="nearest", align_corners=False) use.
// ------------------------------------------------------------------------------------------------
constexpr int kRotThreads = 256;

template <typename TI, typename TO>
__global__ void __launch_bounds__(kRotThreads)
rotate_bev_kernel(const TI *__restrict__ prev, long long stride_q, long long stride_b,
                  const float *__restrict__ rot, TO *__restrict__ out, int bs, int H, int W, int C) {
    const int lane = threadIdx.x & 31;
    const long long rows = (long long)H * W * bs;
    const long long step = (long long)gridDim.x * (kRotThreads / 32);
    for (long long row = (long long)blockIdx.x * (kRotThreads / 32) + (threadIdx.x >> 5); row < rows; row += step) {
        const int b = (int)(row % bs);
        const int q = (int)(row / bs);
        const int i = q / W, j = q - i * W;
        const float *m = rot + b * 6;
        const float bx = (float)j + 0.5f - 0.5f * (float)W, by = (float)i + 0.5f - 0.5f * (float)H;
        const float gx = __fadd_rn(__fmaf_rn(by, __ldg(m + 1), __fmul_rn(bx, __ldg(m))), __ldg(m + 2));
        const float gy = __fadd_rn(__fmaf_rn(by, __ldg(m + 4), __fmul_rn(bx, __ldg(m + 3))), __ldg(m + 5));
        const float fx = __fmul_rn(__fmaf_rn(__fadd_rn(gx, 1.f), (float)W, -1.f), 0.5f);
        const float fy = __fmul_rn(__fmaf_rn(__fadd_rn(gy, 1.f), (float)H, -1.f), 0.5f);
        const float rx = rintf(fx), ry = rintf(fy);            // nearest, ties to even (nearbyint)
        const bool inside = rx >= 0.f && rx <= (float)(W - 1) && ry >= 0.f && ry <= (float)(H - 1);
        TO *dst = out + row * C;
        if (inside) {
            const TI *src = prev + ((long long)ry * W + (long long)rx) * stride_q + (long long)b * stride_b;
            for (int c = lane * 8; c < C; c += 256) {
                float v[8];
                load_vec<TI, 8>(src + c, v);
                store_vec<TO, 8>(dst + c, v);
            }
        } else {
            const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int c = lane * 8; c < C; c += 256) store_vec<TO, 8>(dst + c, z);
        }
    }
}

template <typename TI, typename TO>
static int rotate_launch(const char *who, const void *prev, long long sq, long long sb, const float *rot, void *out,
                         int bs, int H, int W, int C, cudaStream_t st) {
    const long long rows = (long long)H * W * bs;
    long long blocks = (rows + kRotThreads / 32 - 1) / (kRotThreads / 32);
    if (blocks > (long long)device_sms() * 16) blocks = (long long)device_sms() * 16;
    rotate_bev_kernel<TI, TO><<<(unsigned)blocks, kRotThreads, 0, st>>>((const TI *)prev, sq, sb, rot, (TO *)out, bs,
                                                                         H, W, C);
    return check_launch(who);
}

template <typename TI>
static int rotate_dispatch_out(const char *who, const void *prev, long long sq, long long sb, const float *rot,
                               void *out, int out_dtype, int bs, int H, int W, int C, cudaStream_t st) {
    if (out_dtype == BEVF_DTYPE_F32) return rotate_launch<TI, float>(who, prev, sq, sb, rot, out, bs, H, W, C, st);
    if (out_dtype == BEVF_DTYPE_BF16) return rotate_launch<TI, bf16>(who, prev, sq, sb, rot, out, bs, H, W, C, st);
    return rotate_launch<TI, __half>(who, prev, sq, sb, rot, out, bs, H, W, C, st);
}

static bool dtype_ok(int d) { return d == BEVF_DTYPE_F32 || d == BEVF_DTYPE_BF16 || d == BEVF_DTYPE_F16; }

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_ego_motion(const double *can_bus, void *state, int mode, float *shift, float *rot,
                               void *can_bus_out, int out_dtype, int bs, int bev_h, int bev_w, double grid_h,
                               double grid_w, double center_x, double center_y, int use_shift, void *stream) {
    const char *who = "bevf_ego_motion";
    BEVF_REQUIRE(bs >= 0 && bev_h > 0 && bev_w > 0, who, "bad dimension");
    BEVF_REQUIRE(grid_h > 0.0 && grid_w > 0.0, who, "grid_length must be positive");
    BEVF_REQUIRE(dtype_ok(out_dtype), who, "unsupported dtype code");
    BEVF_REQUIRE(mode == BEVF_EGO_DELTAS || mode == BEVF_EGO_CONTINUE || mode == BEVF_EGO_NEW_SCENE, who,
                 "unknown history mode");
    if (bs == 0) return 0;
    BEVF_REQUIRE(can_bus && shift && rot && can_bus_out, who, "null pointer argument");
    BEVF_REQUIRE(mode == BEVF_EGO_DELTAS || state, who, "null pointer argument (a stream mode needs the state block)");
    BEVF_REQUIRE((reinterpret_cast<uintptr_t>(can_bus) & 7u) == 0 && (reinterpret_cast<uintptr_t>(state) & 7u) == 0 &&
                 (reinterpret_cast<uintptr_t>(shift) & 3u) == 0 && (reinterpret_cast<uintptr_t>(rot) & 3u) == 0 &&
                 (reinterpret_cast<uintptr_t>(can_bus_out) & 3u) == 0, who, "misaligned pointer argument");
    EgoParams p{bs, bev_h, bev_w, use_shift, mode, grid_h, grid_w, center_x, center_y};
    cudaStream_t st = (cudaStream_t)stream;
    EgoState *s = (EgoState *)state;
    if (out_dtype == BEVF_DTYPE_F32)
        ego_motion_kernel<float><<<1, 32, 0, st>>>(can_bus, s, shift, rot, (float *)can_bus_out, p);
    else if (out_dtype == BEVF_DTYPE_BF16)
        ego_motion_kernel<bf16><<<1, 32, 0, st>>>(can_bus, s, shift, rot, (bf16 *)can_bus_out, p);
    else
        ego_motion_kernel<__half><<<1, 32, 0, st>>>(can_bus, s, shift, rot, (__half *)can_bus_out, p);
    return check_launch(who);
}

extern "C" int bevf_rotate_bev(const void *prev, int in_dtype, int64_t stride_q, int64_t stride_b, const float *rot,
                               void *out, int out_dtype, int bs, int bev_h, int bev_w, int C, void *stream) {
    const char *who = "bevf_rotate_bev";
    BEVF_REQUIRE(bs >= 0 && bev_h > 0 && bev_w > 0 && C > 0, who, "bad dimension");
    BEVF_REQUIRE(C % 8 == 0, who, "C must be a multiple of 8 (16-byte vectors)");
    BEVF_REQUIRE(dtype_ok(in_dtype) && dtype_ok(out_dtype), who, "unsupported dtype code");
    BEVF_REQUIRE(stride_q >= 0 && stride_b >= 0 && stride_q % 8 == 0 && stride_b % 8 == 0, who,
                 "strides must be non-negative multiples of 8 elements");
    if (bs == 0) return 0;
    BEVF_REQUIRE(prev && rot && out, who, "null pointer argument");
    BEVF_REQUIRE(aligned16(prev) && aligned16(out) && (reinterpret_cast<uintptr_t>(rot) & 3u) == 0, who,
                 "prev and out must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (in_dtype == BEVF_DTYPE_F32)
        return rotate_dispatch_out<float>(who, prev, stride_q, stride_b, rot, out, out_dtype, bs, bev_h, bev_w, C, st);
    if (in_dtype == BEVF_DTYPE_BF16)
        return rotate_dispatch_out<bf16>(who, prev, stride_q, stride_b, rot, out, out_dtype, bs, bev_h, bev_w, C, st);
    return rotate_dispatch_out<__half>(who, prev, stride_q, stride_b, rot, out, out_dtype, bs, bev_h, bev_w, C, st);
}
