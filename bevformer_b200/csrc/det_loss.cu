// Training loss of BEVFormerHead on the device, around the host's Hungarian assignment.
//
//   bevf_det_match_cost      HungarianAssigner3D.assign's cost (core/bbox/assigners/hungarian_assigner_3d.py:106-116):
//                            mmdet 2.14 FocalLossCost + BBox3DL1Cost / SmoothL1Cost (core/bbox/match_costs/
//                            match_cost.py:7-90) on normalize_bbox(gt) (core/bbox/util.py:4-24), for every
//                            (decoder layer, sample) in one launch; a query group is a range of rows of the same matrix
//   bevf_det_loss_forward    BEVFormerHead.loss_single after the assignment (dense_heads/bevformer_head.py:215-393):
//                            targets of the PseudoSampler, mmcv's CUDA sigmoid_focal_loss, L1Loss / SmoothL1Loss with
//                            code weights over the rows whose normalised target is finite, weight_reduce_loss with the
//                            avg factors, nan_to_num; one scalar pair per (layer, group) slot
//   bevf_det_loss_backward   the gradient of those slot scalars with respect to the logits and boxes
//
// Arithmetic: the sigmoid is rounded to fp32 exactly as torch.sigmoid and mmcv's kernel compute it (libdevice expf,
// IEEE division) because that rounding is what decides the reference's costs for confident logits (1 - p carries the
// absolute error of p); the fp32 sums 1 - p and p + eps are kept for the same reason.  Everything after them -- log,
// pow, the 8-term regression sum, the reductions -- is evaluated in double and rounded once, so the results do not
// depend on --use_fast_math.  The reductions run in a fixed order (one CTA per slot, a shared-memory tree), with no
// floating-point atomics: the outputs repeat bit for bit from run to run.
#include "common.cuh"

#include <cfloat>

namespace bevf {

constexpr int kDlThreads = 256;
constexpr int kDcTileQ = 32;                   // queries per CTA of the cost kernel
constexpr int kDlMaxCls = 64;
constexpr int kDcMaxSmem = 200 * 1024;

extern "C" __device__ float __nv_expf(float);

__device__ __forceinline__ float dl_ld(const void *p, int dt, long long i) {
    if (dt == BEVF_DTYPE_BF16) return __bfloat162float(reinterpret_cast<const bf16 *>(p)[i]);
    if (dt == BEVF_DTYPE_F16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
    return reinterpret_cast<const float *>(p)[i];
}

__device__ __forceinline__ void dl_st(void *p, int dt, long long i, float v) {
    if (dt == BEVF_DTYPE_BF16) reinterpret_cast<bf16 *>(p)[i] = __float2bfloat16_rn(v);
    else if (dt == BEVF_DTYPE_F16) reinterpret_cast<__half *>(p)[i] = __float2half_rn(v);
    else reinterpret_cast<float *>(p)[i] = v;
}

// torch.sigmoid / mmcv's p in fp32: 1 / (1 + expf(-x))
__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, __nv_expf(-x))); }

// normalize_bbox of one gravity-centred box (x, y, z, w, l, h, rot, vx, vy): (cx, cy, log w, log l, cz, log h,
// sin rot, cos rot, vx, vy), each rounded to fp32 as the reference's fp32 tensor holds it
__device__ __forceinline__ void normalize_gt(const float *g, float (&t)[10]) {
    t[0] = g[0]; t[1] = g[1];
    t[2] = (float)log((double)g[3]); t[3] = (float)log((double)g[4]);
    t[4] = g[2]; t[5] = (float)log((double)g[5]);
    t[6] = (float)sin((double)g[6]); t[7] = (float)cos((double)g[6]);
    t[8] = g[7]; t[9] = g[8];
}

struct FocalCfg {
    double alpha, gamma;
};

// mmcv 1.4 sigmoid_focal_loss_forward_cuda_kernel, one element: -alpha (1-p)^g log(max(p, FLT_MIN)) for the target
// class, -(1-alpha) p^g log(max(1-p, FLT_MIN)) for the others
__device__ __forceinline__ double focal_loss(float x, bool pos, const FocalCfg &f) {
    const float p = sigmoid_ref(x), q = __fsub_rn(1.f, p);
    if (pos) return -f.alpha * pow((double)q, f.gamma) * log((double)fmaxf(p, FLT_MIN));
    return -(1.0 - f.alpha) * pow((double)p, f.gamma) * log((double)fmaxf(q, FLT_MIN));
}

// mmcv 1.4 sigmoid_focal_loss_backward_cuda_kernel, one element
__device__ __forceinline__ double focal_grad(float x, bool pos, const FocalCfg &f) {
    const float p = sigmoid_ref(x), q = __fsub_rn(1.f, p);
    const double pd = p, qd = q;
    if (pos) return -f.alpha * pow(qd, f.gamma) * (qd - f.gamma * pd * log((double)fmaxf(p, FLT_MIN)));
    return -(1.0 - f.alpha) * pow(pd, f.gamma) * (f.gamma * qd * log((double)fmaxf(q, FLT_MIN)) - pd);
}

// ---- matching cost ---------------------------------------------------------------------------------------------
struct CostParams {
    const void *cls, *box;
    int cls_dt, box_dt;
    const float *gt;               // (bs, G, 9)
    const long long *labels;       // (bs, G)
    const int *n_gt;               // (bs)
    float *cost;                   // (P, nq, G)
    int P, bs, nq, ncls, G, tiles, reg_kind;
    double w_cls, w_reg, alpha, gamma;
    float eps;
};

__global__ void __launch_bounds__(kDlThreads) det_match_cost_kernel(const __grid_constant__ CostParams p) {
    extern __shared__ double dc_smem[];
    double *s_cls = dc_smem;                                   // [kDcTileQ][ncls] weighted focal cost per class
    float *s_box = reinterpret_cast<float *>(s_cls + kDcTileQ * p.ncls);   // [kDcTileQ][8]
    float *s_gt = s_box + kDcTileQ * 8;                        // [G][8] normalised ground truth
    int *s_lab = reinterpret_cast<int *>(s_gt + p.G * 8);      // [G]
    const int pi = blockIdx.x / p.tiles, tile = blockIdx.x - pi * p.tiles;
    const int b = pi % p.bs, q0 = tile * kDcTileQ, nrow = min(kDcTileQ, p.nq - q0);
    const int ng = min(max(p.n_gt[b], 0), p.G);
    const int tid = threadIdx.x;
    for (int g = tid; g < ng; g += kDlThreads) {
        float t[10];
        normalize_gt(p.gt + ((long long)b * p.G + g) * 9, t);
#pragma unroll
        for (int c = 0; c < 8; ++c) s_gt[g * 8 + c] = t[c];
        const long long lab = p.labels[(long long)b * p.G + g];
        s_lab[g] = lab >= 0 && lab < p.ncls ? (int)lab : -1;
    }
    const long long row0 = (long long)pi * p.nq + q0;
    for (int e = tid; e < nrow * p.ncls; e += kDlThreads) {
        // FocalLossCost: pos = -log(p + eps) alpha (1 - p)^g, neg = -log(1 - p + eps) (1 - alpha) p^g
        const float pr = sigmoid_ref(dl_ld(p.cls, p.cls_dt, row0 * p.ncls + e));
        const float q = __fsub_rn(1.f, pr);
        const double pos = -log((double)__fadd_rn(pr, p.eps)) * p.alpha * pow((double)q, p.gamma);
        const double neg = -log((double)__fadd_rn(q, p.eps)) * (1.0 - p.alpha) * pow((double)pr, p.gamma);
        s_cls[e] = (pos - neg) * p.w_cls;
    }
    for (int e = tid; e < nrow * 8; e += kDlThreads)
        s_box[e] = dl_ld(p.box, p.box_dt, (row0 + e / 8) * 10 + e % 8);
    __syncthreads();
    float *out = p.cost + row0 * p.G;
    for (int e = tid; e < nrow * p.G; e += kDlThreads) {
        const int q = e / p.G, g = e - q * p.G;
        if (g >= ng) { out[e] = 0.f; continue; }
        const int lab = s_lab[g];
        if (lab < 0) { out[e] = __int_as_float(0x7fc00000); continue; }   // a label outside [0, ncls): NaN
        double reg = 0.0;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const double d = fabs((double)s_box[q * 8 + c] - (double)s_gt[g * 8 + c]);
            reg += p.reg_kind == BEVF_DET_REG_L1 ? d : (d < 1.0 ? 0.5 * d * d : d - 0.5);
        }
        out[e] = (float)(s_cls[q * p.ncls + lab] + reg * p.w_reg);
    }
}

// ---- losses ----------------------------------------------------------------------------------------------------
struct LossParams {
    const void *cls, *box;
    int cls_dt, box_dt;
    const int *assign;             // (P, nq): ground-truth index or -1
    const float *gt;               // (bs, G, 9)
    const long long *labels;       // (bs, G)
    const int *n_gt;               // (bs)
    const float *code_w;           // (10)
    const float *avg;              // (S, 2): cls / regression avg factors before max(., 1)
    float *loss, *loss_raw;        // (S, 2)
    const float *grad_loss;        // (S, 2)
    void *grad_cls, *grad_box;
    int L, bs, nq, groups, nqg, ncls, G, reg_kind;
    double lw_cls, lw_box, beta;
    FocalCfg focal;
};

// the row's label (-1: background) and, for a positive row, its normalised target and whether all of it is finite
struct RowTarget {
    int label;
    bool box_ok;
    float t[10];
};

__device__ __forceinline__ RowTarget row_target(const LossParams &p, int b, long long row) {
    RowTarget r;
    r.label = -1;
    r.box_ok = false;
    const int j = p.assign[row];
    const int ng = min(max(p.n_gt[b], 0), p.G);
    if (j < 0 || j >= ng) return r;
    const long long lab = p.labels[(long long)b * p.G + j];
    r.label = lab >= 0 && lab < p.ncls ? (int)lab : p.ncls;    // mmcv: a label no channel equals is all-negative
    normalize_gt(p.gt + ((long long)b * p.G + j) * 9, r.t);
    r.box_ok = true;
#pragma unroll
    for (int c = 0; c < 10; ++c) r.box_ok = r.box_ok && isfinite(r.t[c]);
    return r;
}

__device__ __forceinline__ double reg_term(double d, const LossParams &p) {
    const double a = fabs(d);
    return p.reg_kind == BEVF_DET_REG_L1 ? a : (a < p.beta ? 0.5 * a * a / p.beta : a - 0.5 * p.beta);
}
__device__ __forceinline__ double reg_deriv(double d, const LossParams &p) {
    const double s = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0);
    return p.reg_kind == BEVF_DET_REG_L1 ? s : (fabs(d) < p.beta ? d / p.beta : s);
}

__device__ __forceinline__ float nan_to_num_f(float v) {
    if (isnan(v)) return 0.f;
    if (isinf(v)) return v > 0.f ? FLT_MAX : -FLT_MAX;
    return v;
}

// one CTA per slot (layer l, group g): rows (b, q) for every sample b and q in the group's query range
__global__ void __launch_bounds__(kDlThreads) det_loss_forward_kernel(const __grid_constant__ LossParams p) {
    __shared__ double red[2][kDlThreads];
    const int s = blockIdx.x, l = s / p.groups, grp = s - l * p.groups;
    const int tid = threadIdx.x;
    double acc_cls = 0.0, acc_box = 0.0;
    for (int r = tid; r < p.bs * p.nqg; r += kDlThreads) {
        const int b = r / p.nqg, q = grp * p.nqg + (r - b * p.nqg);
        const long long row = ((long long)l * p.bs + b) * p.nq + q;
        const RowTarget t = row_target(p, b, row);
        for (int c = 0; c < p.ncls; ++c)
            acc_cls += focal_loss(dl_ld(p.cls, p.cls_dt, row * p.ncls + c), c == t.label, p.focal);
        if (t.box_ok)
#pragma unroll
            for (int c = 0; c < 10; ++c)
                acc_box += reg_term((double)dl_ld(p.box, p.box_dt, row * 10 + c) - (double)t.t[c], p) *
                           (double)p.code_w[c];
    }
    red[0][tid] = acc_cls;
    red[1][tid] = acc_box;
    __syncthreads();
    for (int w = kDlThreads / 2; w > 0; w >>= 1) {
        if (tid < w) {
            red[0][tid] += red[0][tid + w];
            red[1][tid] += red[1][tid + w];
        }
        __syncthreads();
    }
    if (tid < 2) {
        const double avg = fmax((double)p.avg[2 * s + tid], 1.0);
        const float v = (float)(red[tid][0] / avg * (tid == 0 ? p.lw_cls : p.lw_box));
        p.loss_raw[2 * s + tid] = v;
        p.loss[2 * s + tid] = nan_to_num_f(v);
    }
}

// one thread per row (l, b, q): the row's ncls logit gradients and 10 box gradients
__global__ void __launch_bounds__(kDlThreads) det_loss_backward_kernel(const __grid_constant__ LossParams p) {
    const long long row = (long long)blockIdx.x * kDlThreads + threadIdx.x;
    if (row >= (long long)p.L * p.bs * p.nq) return;
    const int q = (int)(row % p.nq);
    const int b = (int)((row / p.nq) % p.bs), l = (int)(row / ((long long)p.nq * p.bs));
    const int s = l * p.groups + q / p.nqg;
    // d(slot scalar) / d(sum of elementwise terms), with nan_to_num's mask: no gradient through a non-finite loss
    const double gc = (double)p.grad_loss[2 * s] * (isfinite(p.loss_raw[2 * s]) ? 1.0 : 0.0) * p.lw_cls /
                      fmax((double)p.avg[2 * s], 1.0);
    const double gb = (double)p.grad_loss[2 * s + 1] * (isfinite(p.loss_raw[2 * s + 1]) ? 1.0 : 0.0) * p.lw_box /
                      fmax((double)p.avg[2 * s + 1], 1.0);
    const RowTarget t = row_target(p, b, row);
    for (int c = 0; c < p.ncls; ++c) {
        const double g = focal_grad(dl_ld(p.cls, p.cls_dt, row * p.ncls + c), c == t.label, p.focal) * gc;
        dl_st(p.grad_cls, p.cls_dt, row * p.ncls + c, (float)g);
    }
#pragma unroll
    for (int c = 0; c < 10; ++c) {
        float g = 0.f;
        if (t.box_ok)
            g = (float)(reg_deriv((double)dl_ld(p.box, p.box_dt, row * 10 + c) - (double)t.t[c], p) *
                        (double)p.code_w[c] * gb);
        dl_st(p.grad_box, p.box_dt, row * 10 + c, g);
    }
}

static bool dl_dt_ok(int dt) { return dt == BEVF_DTYPE_F32 || dt == BEVF_DTYPE_BF16 || dt == BEVF_DTYPE_F16; }

}  // namespace bevf

using namespace bevf;

#define BEVF_REQUIRE(cond, who, msg) do { if (!(cond)) return fail("%s: " msg, who); } while (0)

extern "C" int64_t bevf_det_match_cost_smem_bytes(int ncls, int G) {
    return (int64_t)kDcTileQ * ncls * 8 + kDcTileQ * 8 * 4 + (int64_t)G * 8 * 4 + (int64_t)G * 4;
}

extern "C" int bevf_det_match_cost(const void *cls, int cls_dtype, const void *box, int box_dtype, const float *gt,
                                   const int64_t *gt_labels, const int *n_gt, float *cost, int P, int bs, int nq,
                                   int ncls, int G, int reg_kind, float cls_weight, float reg_weight, float alpha,
                                   float gamma, float eps, void *stream) {
    const char *who = "bevf_det_match_cost";
    BEVF_REQUIRE(P > 0 && bs > 0 && P % bs == 0 && nq > 0 && G > 0, who, "bad dimension (P a multiple of bs, G > 0)");
    BEVF_REQUIRE(ncls > 0 && ncls <= kDlMaxCls, who, "need 1 <= ncls <= 64");
    BEVF_REQUIRE(reg_kind == BEVF_DET_REG_L1 || reg_kind == BEVF_DET_REG_SMOOTH_L1, who, "unknown regression cost");
    BEVF_REQUIRE(dl_dt_ok(cls_dtype) && dl_dt_ok(box_dtype), who, "unsupported dtype code");
    BEVF_REQUIRE(cls && box && gt && gt_labels && n_gt && cost, who, "null pointer argument");
    const int64_t smem = bevf_det_match_cost_smem_bytes(ncls, G);
    BEVF_REQUIRE(smem <= kDcMaxSmem, who, "too many ground-truth boxes for the shared-memory tile");
    const int tiles = (nq + kDcTileQ - 1) / kDcTileQ;
    BEVF_REQUIRE((long long)P * tiles < (1LL << 31), who, "too many rows");
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(det_match_cost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDcMaxSmem) !=
            cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory", who);
        }
        attr = true;
    }
    CostParams p{};
    p.cls = cls; p.box = box; p.cls_dt = cls_dtype; p.box_dt = box_dtype;
    p.gt = gt; p.labels = reinterpret_cast<const long long *>(gt_labels); p.n_gt = n_gt; p.cost = cost;
    p.P = P; p.bs = bs; p.nq = nq; p.ncls = ncls; p.G = G; p.tiles = tiles; p.reg_kind = reg_kind;
    p.w_cls = cls_weight; p.w_reg = reg_weight; p.alpha = alpha; p.gamma = gamma; p.eps = eps;
    det_match_cost_kernel<<<P * tiles, kDlThreads, (size_t)smem, (cudaStream_t)stream>>>(p);
    return check_launch(who);
}

static int loss_params(LossParams &p, const char *who, const void *cls, int cls_dtype, const void *box,
                       int box_dtype, const int *assign, const float *gt, const int64_t *gt_labels, const int *n_gt,
                       const float *code_weights, const float *avg, int L, int bs, int nq, int groups, int ncls,
                       int G, int reg_kind, float cls_loss_weight, float bbox_loss_weight, float alpha, float gamma,
                       float beta) {
    BEVF_REQUIRE(L > 0 && bs > 0 && nq > 0 && groups > 0 && nq % groups == 0 && G >= 0, who,
                 "bad dimension (nq a multiple of groups)");
    BEVF_REQUIRE(ncls > 0, who, "need ncls >= 1");
    BEVF_REQUIRE((long long)L * bs * nq < (1LL << 40), who, "too many rows");
    BEVF_REQUIRE(reg_kind == BEVF_DET_REG_L1 || reg_kind == BEVF_DET_REG_SMOOTH_L1, who, "unknown regression loss");
    BEVF_REQUIRE(reg_kind == BEVF_DET_REG_L1 || beta > 0.f, who, "smooth-L1 needs beta > 0");
    BEVF_REQUIRE(dl_dt_ok(cls_dtype) && dl_dt_ok(box_dtype), who, "unsupported dtype code");
    BEVF_REQUIRE(cls && box && assign && n_gt && code_weights && avg, who, "null pointer argument");
    BEVF_REQUIRE(G == 0 || (gt && gt_labels), who, "null ground-truth pointer");
    p.cls = cls; p.box = box; p.cls_dt = cls_dtype; p.box_dt = box_dtype;
    p.assign = assign; p.gt = gt; p.labels = reinterpret_cast<const long long *>(gt_labels); p.n_gt = n_gt;
    p.code_w = code_weights; p.avg = avg;
    p.L = L; p.bs = bs; p.nq = nq; p.groups = groups; p.nqg = nq / groups; p.ncls = ncls; p.G = G;
    p.reg_kind = reg_kind;
    p.lw_cls = cls_loss_weight; p.lw_box = bbox_loss_weight; p.beta = beta;
    p.focal.alpha = alpha; p.focal.gamma = gamma;
    return 0;
}

extern "C" int bevf_det_loss_forward(const void *cls, int cls_dtype, const void *box, int box_dtype,
                                     const int *assign, const float *gt, const int64_t *gt_labels, const int *n_gt,
                                     const float *code_weights, const float *avg, float *loss, float *loss_raw, int L,
                                     int bs, int nq, int groups, int ncls, int G, int reg_kind, float cls_loss_weight,
                                     float bbox_loss_weight, float alpha, float gamma, float beta, void *stream) {
    const char *who = "bevf_det_loss_forward";
    LossParams p{};
    if (loss_params(p, who, cls, cls_dtype, box, box_dtype, assign, gt, gt_labels, n_gt, code_weights, avg, L, bs, nq,
                    groups, ncls, G, reg_kind, cls_loss_weight, bbox_loss_weight, alpha, gamma, beta))
        return 1;
    BEVF_REQUIRE(loss && loss_raw, who, "null pointer argument");
    p.loss = loss; p.loss_raw = loss_raw;
    det_loss_forward_kernel<<<L * groups, kDlThreads, 0, (cudaStream_t)stream>>>(p);
    return check_launch(who);
}

extern "C" int bevf_det_loss_backward(const void *cls, int cls_dtype, const void *box, int box_dtype,
                                      const int *assign, const float *gt, const int64_t *gt_labels, const int *n_gt,
                                      const float *code_weights, const float *avg, const float *loss_raw,
                                      const float *grad_loss, void *grad_cls, void *grad_box, int L, int bs, int nq,
                                      int groups, int ncls, int G, int reg_kind, float cls_loss_weight,
                                      float bbox_loss_weight, float alpha, float gamma, float beta, void *stream) {
    const char *who = "bevf_det_loss_backward";
    LossParams p{};
    if (loss_params(p, who, cls, cls_dtype, box, box_dtype, assign, gt, gt_labels, n_gt, code_weights, avg, L, bs, nq,
                    groups, ncls, G, reg_kind, cls_loss_weight, bbox_loss_weight, alpha, gamma, beta))
        return 1;
    BEVF_REQUIRE(loss_raw && grad_loss && grad_cls && grad_box, who, "null pointer argument");
    p.loss_raw = const_cast<float *>(loss_raw); p.grad_loss = grad_loss;
    p.grad_cls = grad_cls; p.grad_box = grad_box;
    const long long rows = (long long)L * bs * nq;
    det_loss_backward_kernel<<<(unsigned)((rows + kDlThreads - 1) / kDlThreads), kDlThreads, 0,
                               (cudaStream_t)stream>>>(p);
    return check_launch(who);
}
