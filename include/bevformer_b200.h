/*
 * bevformer_b200 -- C ABI of the CUDA-native BEV-encoder hot path (built for sm_90a, H100).
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference reaches its native code through the
 * pybind module `mmcv._ext` (third-party wheel mmcv-full==1.4.0, not in the reference tree):
 *
 *   ext_module.ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc,
 *                                     attn_weight, im2col_step) -> Tensor
 *       projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:118-124
 *   ext_module.ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc,
 *                                      attn_weight, grad_output, grad_value, grad_sampling_loc,
 *                                      grad_attn_weight, im2col_step) -> None   (in place)
 *       .../multi_scale_deformable_attn_function.py:150-160
 *
 * Those two calls are replaced 1:1 by bevf_msda_forward / bevf_msda_backward below.  The remaining
 * entry points are the fused pieces of the encoder layer that the reference spells as ATen /
 * cuBLAS launches inside TemporalSelfAttention / SpatialCrossAttention / BEVFormerLayer /
 * BEVFormerEncoder (each cites the Python lines it replaces).
 *
 * Conventions
 *   - plain C: raw device pointers, sizes, an opaque cudaStream_t passed as void*; no torch types.
 *   - the caller owns every buffer; the library never allocates, frees or synchronises, and keeps no
 *     mutable global state besides a thread-local error string, so every call is re-entrant and
 *     safe under CUDA-graph capture.
 *   - every function returns 0 on success, non-zero on error; bevf_last_error() then holds a
 *     message for the calling thread (the Python wrapper raises RuntimeError with it, which is
 *     what mmcv's TORCH_CHECK failures surface as).
 *   - tensors are dense row-major in the layouts named per function; "dtype" arguments take the
 *     BEVF_DTYPE_* codes.  Device pointers must be 16-byte aligned; the entry points refuse a misaligned
 *     pointer that a kernel accesses with 16 B vectors, while scalar and atomic operands (LayerNorm's mean / rstd /
 *     dgamma / dbeta, bevf_colsum's out, inv_count) may sit at any float offset.
 *   - there is NO CPU implementation behind this ABI.
 */
#ifndef BEVFORMER_B200_H_
#define BEVFORMER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BEVF_ABI_VERSION 3

#if defined(__GNUC__)
#define BEVF_API __attribute__((visibility("default")))
#else
#define BEVF_API
#endif

/* Storage types.  fp16 stores round to nearest and overflow to +-inf (never saturate), so loss scaling sees the
 * overflow; every kernel widens 16-bit inputs exactly and accumulates in fp32. */
enum bevf_dtype { BEVF_DTYPE_F32 = 0, BEVF_DTYPE_BF16 = 1, BEVF_DTYPE_F16 = 2 };

/* ABI version of the loaded library (== BEVF_ABI_VERSION it was built with). */
BEVF_API int bevf_version(void);

/* Message of the last failing call on this thread ("" if none). Never NULL. */
BEVF_API const char *bevf_last_error(void);

/* Number of kernel launches issued through this library by the calling process so far
 * (bench.py reports it as gpu_launches). */
BEVF_API int64_t bevf_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Multi-scale deformable attention sampler.
 *
 * replaces: mmcv._ext.ms_deform_attn_forward, as called at
 *   multi_scale_deformable_attn_function.py:118-124 (from temporal_self_attention.py:247,
 *   spatial_cross_attention.py:390, decoder.py:332).
 *
 *   value        (B, S, M, D)        value_dtype (f32 | bf16 | f16)
 *   level_hw     (L, 2) int64 DEVICE (h, w) per level          -- the reference's spatial_shapes
 *   level_start  (L,)   int64 DEVICE first row of each level   -- the reference's level_start_index
 *   loc          (B, Q, M, L, P, 2) f32, (x, y) normalised to [0,1] over each level
 *   attn         (B, Q, M, L, P)    f32
 *   out          (B, Q, M*D)        out_dtype (f32 | bf16 | f16), fully overwritten; a 16-bit out
 *                                   needs the same value dtype (bf16 value may write f32, f16 value f32)
 *
 * out[b,q,m,:] = sum_l sum_p attn * bilinear(value_l, x = loc_x*W_l - 0.5, y = loc_y*H_l - 0.5),
 * zero padding, a sample contributes only if -1 < x < W_l and -1 < y < H_l (SURVEY.md Appendix A).
 * Accumulation is fp32 for both value dtypes.  `im2col_step` of the reference has no equivalent:
 * the whole batch is one launch.  L <= 16.
 */
BEVF_API int bevf_msda_forward(const void *value, int value_dtype, const int64_t *level_hw,
                      const int64_t *level_start, const float *loc, const float *attn, void *out,
                      int out_dtype, int B, int S, int M, int D, int Q, int L, int P, void *stream);

/*
 * replaces: mmcv._ext.ms_deform_attn_backward, as called at
 *   multi_scale_deformable_attn_function.py:150-160.
 *
 *   grad_out    (B, Q, M*D)  grad_out_dtype (f32 | bf16 | f16; a 16-bit grad_out matches value_dtype)
 *   grad_value  (B, S, M, D) f32 -- ACCUMULATED INTO (caller zero-fills, as the reference does at
 *                                   multi_scale_deformable_attn_function.py:146)
 *   grad_loc    (B, Q, M, L, P, 2) f32 -- fully overwritten (zeros for skipped samples)
 *   grad_attn   (B, Q, M, L, P)    f32 -- fully overwritten
 * grad_value uses vector fp32 reductions in L2; its summation order is not deterministic
 * (bevf_msda_backward_fx below is the deterministic form).
 */
BEVF_API int bevf_msda_backward(const void *value, int value_dtype, const int64_t *level_hw,
                       const int64_t *level_start, const float *loc, const float *attn,
                       const void *grad_out, int grad_out_dtype, float *grad_value,
                       float *grad_loc, float *grad_attn, int B, int S, int M, int D, int Q, int L,
                       int P, void *stream);

/*
 * Row-list form of the sampler: R query rows, each sampling the value map named by row_map[r]
 * (0 <= row_map[r] < B).  bevf_msda_forward is the special case row_map[r] = r / Q.
 *
 * replaces: the zero-padded per-camera re-batching around the op in
 *   spatial_cross_attention.py:138-167 (nonzero -> max_len -> queries_rebatch -> op -> slots +=):
 *   SpatialCrossAttention hands the op only the (camera, query) pairs that are actually in view,
 *   in one launch, instead of num_cams x max_len padded rows.
 *
 *   loc (R, M, L, P, 2) f32; attn (R, M, L, P) f32; out / grad_out (R, M*D); row_map (R,) int32 DEVICE.
 * Other arguments and semantics as for bevf_msda_forward / bevf_msda_backward.
 */
BEVF_API int bevf_msda_rows_forward(const void *value, int value_dtype, const int64_t *level_hw,
                                    const int64_t *level_start, const float *loc, const float *attn,
                                    void *out, int out_dtype, const int32_t *row_map, int B, int S,
                                    int M, int D, int R, int L, int P, void *stream);

BEVF_API int bevf_msda_rows_backward(const void *value, int value_dtype, const int64_t *level_hw,
                                     const int64_t *level_start, const float *loc,
                                     const float *attn, const void *grad_out, int grad_out_dtype,
                                     float *grad_value, float *grad_loc, float *grad_attn,
                                     const int32_t *row_map, int B, int S, int M, int D, int R,
                                     int L, int P, void *stream);

/*
 * Same as bevf_msda_rows_backward, plus `group_order` (R,) int32 (or NULL = identity): a permutation of
 * the rows that lists them so that runs of 64 consecutive entries are spatial neighbours on ONE value map
 * (for the interleaved TSA rows: 8x8 BEV tiles of one frame).  The grad_value half of the backward
 * merges the contributions of such a run in registers before they reach L2 (csrc/msda_splat.cuh); the
 * order changes which additions are merged, never the result beyond fp32 summation order.
 * Level maps must satisfy H_l, W_l < 32768.
 */
BEVF_API int bevf_msda_rows_backward_ordered(const void *value, int value_dtype, const int64_t *level_hw,
                                             const int64_t *level_start, const float *loc,
                                             const float *attn, const void *grad_out,
                                             int grad_out_dtype, float *grad_value, float *grad_loc,
                                             float *grad_attn, const int32_t *row_map,
                                             const int32_t *group_order, int B, int S, int M, int D,
                                             int R, int L, int P, void *stream);

/*
 * grad_value accumulated in SCALED fp16 instead of fp32.  The sampler backward is bound by the L2 reduction-sector
 * rate; an fp16 running sum needs half the sectors (one 16-byte f16x2 vector reduction per lane and corner).
 * fp16 needs a scale: bevf_abs_max puts max|grad_out| (as float bits) into one device word, every kernel of the
 * path derives the same power of two from it (the maximum lands in [8, 16): sums of thousands of contributions stay
 * below 65504, values down to 2^-17 of the maximum stay normal numbers).  The running sum is rounded to 11 bits at
 * every addition, so this is for maps / levels where a (pixel, head) collects few contributions; measured errors
 * in tests/test_msda_gpu.py (bf16 accumulation -- what the reference's fp16 op class does,
 * multi_scale_deformable_attn_function.py:146-160 -- was measured at 1.4e-2 on the TSA launch, above the bar).
 *
 *   bevf_abs_max(x, dtype, n, amax_bits)      *amax_bits = float bits of max|x| (n a multiple of 8 / 4 elements)
 *   bevf_msda_rows_backward_f16acc            bevf_msda_rows_backward_ordered with grad_value_f16 (B, S, M, D) fp16,
 *                                             zero-filled or holding a running sum in the same scale
 *   bevf_gv16_unscale(gv16, amax, out, n)     out (bf16) = gv16 / scale
 *   bevf_msda_rows_backward_mixed             the first num_f16_levels pyramid levels (pixels [0, S_fine) of every
 *                                             map) in scaled fp16 into grad_value_fine_f16 (B, S_fine, M, D), the
 *                                             others in fp32 into grad_value_side (B, S - S_fine, M, D); S_fine is
 *                                             taken from level_hw_host (L, 2) int32 HOST, the kernel re-derives which
 *                                             levels lie before / after it from the DEVICE pyramid (a device level
 *                                             that straddles S_fine is a caller bug and traps)
 *   bevf_msda_rows_backward_mixed_dense       bevf_msda_rows_backward_mixed for row lists grouped by value map
 *                                             (map_range (B, 2) int32 DEVICE, as bevf_msda_rows_backward_dense; no
 *                                             group_order): the side levels [first_dense_level, L) (first_dense_level
 *                                             in [num_f16_levels, L - 1]) come from the dense tensor-core kernel
 *                                             (csrc/msda_dense.cu) instead of fp32 L2 reductions, written into
 *                                             grad_value_side, on the stream bevf_msda_set_dense_backward selects.
 *                                             Only if its bin plan covers exactly those levels, grad_out is
 *                                             bf16 and there are 4 or 8 points per level; otherwise, with the dense
 *                                             mode 0, or when the device pyramid differs from level_hw_host, this is
 *                                             exactly bevf_msda_rows_backward_mixed.  Same outputs either way; the
 *                                             dense levels' coefficients are rounded to bf16 (2^-9 relative per term).
 *   bevf_gv_merge(fine, side, amax, out, B, S, S_fine, row_elems)   out (B, S, row_elems) bf16 from both
 * All need a bf16 value tensor and head_dim 32 (fp16 value is an error); grad_loc / grad_attn are those of the fp32
 * path bit for bit.
 */
BEVF_API int bevf_abs_max(const void *x, int dtype, int64_t n, uint32_t *amax_bits, void *stream);
BEVF_API int bevf_msda_rows_backward_f16acc(const void *value, int value_dtype, const int64_t *level_hw,
                                            const int64_t *level_start, const float *loc, const float *attn,
                                            const void *grad_out, int grad_out_dtype, void *grad_value_f16,
                                            const uint32_t *amax_bits, float *grad_loc, float *grad_attn,
                                            const int32_t *row_map, const int32_t *group_order, int B, int S,
                                            int M, int D, int R, int L, int P, void *stream);
BEVF_API int bevf_gv16_unscale(const void *gv16, const uint32_t *amax_bits, void *out_bf16, int64_t n, void *stream);
BEVF_API int bevf_msda_rows_backward_mixed(const void *value, int value_dtype, const int64_t *level_hw,
                                           const int64_t *level_start, const int32_t *level_hw_host,
                                           const float *loc, const float *attn, const void *grad_out,
                                           int grad_out_dtype, void *grad_value_fine_f16, float *grad_value_side,
                                           const uint32_t *amax_bits, int num_f16_levels, float *grad_loc,
                                           float *grad_attn, const int32_t *row_map, const int32_t *group_order,
                                           int B, int S, int M, int D, int R, int L, int P, void *stream);
BEVF_API int bevf_msda_rows_backward_mixed_dense(const void *value, int value_dtype, const int64_t *level_hw,
                                                 const int64_t *level_start, const int32_t *level_hw_host,
                                                 const float *loc, const float *attn, const void *grad_out,
                                                 int grad_out_dtype, void *grad_value_fine_f16, float *grad_value_side,
                                                 const uint32_t *amax_bits, int num_f16_levels, int first_dense_level,
                                                 float *grad_loc, float *grad_attn, const int32_t *row_map,
                                                 const int32_t *map_range,
                                                 int B, int S, int M, int D, int R, int L, int P, void *stream);
BEVF_API int bevf_gv_merge(const void *fine_f16, const float *side_f32, const uint32_t *amax_bits, void *out_bf16,
                           int B, int S, int S_fine, int row_elems, void *stream);

/*
 * DETERMINISTIC sampler backward: grad_value summed in 64-bit fixed point.  Integer addition is associative, so the
 * result does not depend on the order in which the samples are processed (any row order, any schedule gives the same
 * bits).  grad_loc / grad_attn are those of bevf_msda_backward / bevf_msda_rows_backward bit for bit.
 *
 *   bevf_msda_fx_frac_bits(rows_per_map, L, P)   the fraction bits K for a launch: min(40, 62 - ceil(log2(n_max)))
 *                                                with n_max = rows_per_map * L * P * 4, the most contributions one
 *                                                element can receive (rows_per_map = Q, or R for a row list);
 *                                                n_max * 2^K <= 2^62, so the sum cannot overflow.  -1 if no K fits.
 *   bevf_msda_backward_fx / _rows_backward_fx    arguments as bevf_msda_backward / bevf_msda_rows_backward, plus
 *       grad_value_fx  (B, S, M, D) int64 -- ACCUMULATED INTO (caller zero-fills)
 *       bounds         2 uint32 DEVICE words, written: the bits of max|attn| and max|grad_out| over the launch's rows
 *                      (rows with row_map < 0 excluded), sign cleared; the conversion reads them
 *       frac_bits      K, at most bevf_msda_fx_frac_bits(Q or R, L, P)
 *   bevf_msda_fx_convert(fx, bounds, K, out, out_dtype, accumulate, n)   out (f32 | bf16 | f16) = fx * 2^(E - K), or
 *                                                out += that with accumulate != 0 (bevf_msda_backward's contract)
 * Scale: E = (floor(log2 max|attn|) + 1) + (floor(log2 max|grad_out|) + 1), so every contribution w * attn * g
 * (w <= 1) is below 2^E.  A contribution is formed exactly (the fp32 products w * attn and (w * attn) * g in double),
 * scaled by 2^(K - E) and rounded to the nearest integer once.  PRECISION: an element that receives n contributions
 * differs from their exact sum by at most n * 2^(E - K - 1) before the final rounding to out_dtype (with K = 40:
 * n * 2^-39 of 4 * max|attn| * max|grad_out|).
 * NON-FINITE INPUT: if attn or grad_out holds an inf or NaN in a live row, nothing is accumulated and the conversion
 * makes every element of grad_value NaN (with accumulate: NaN is added).
 */
BEVF_API int bevf_msda_fx_frac_bits(int64_t rows_per_map, int L, int P);
BEVF_API int bevf_msda_backward_fx(const void *value, int value_dtype, const int64_t *level_hw,
                                   const int64_t *level_start, const float *loc, const float *attn,
                                   const void *grad_out, int grad_out_dtype, int64_t *grad_value_fx, uint32_t *bounds,
                                   int frac_bits, float *grad_loc, float *grad_attn, int B, int S, int M, int D, int Q,
                                   int L, int P, void *stream);
BEVF_API int bevf_msda_rows_backward_fx(const void *value, int value_dtype, const int64_t *level_hw,
                                        const int64_t *level_start, const float *loc, const float *attn,
                                        const void *grad_out, int grad_out_dtype, int64_t *grad_value_fx,
                                        uint32_t *bounds, int frac_bits, float *grad_loc, float *grad_attn,
                                        const int32_t *row_map, int B, int S, int M, int D, int R, int L, int P,
                                        void *stream);
BEVF_API int bevf_msda_fx_convert(const int64_t *grad_value_fx, const uint32_t *bounds, int frac_bits, void *out,
                                  int out_dtype, int accumulate, int64_t n, void *stream);

/*
 * bevf_msda_rows_backward for row lists grouped by value map (the SCA pair list), with grad_value of the
 * COARSE pyramid levels computed as a dense product on the tensor cores (csrc/msda_dense.cu) instead of one
 * L2 reduction per (sample, corner): for a (value map, head) the col2im scatter of
 * multi_scale_deformable_attn_function.py:150-160 is  C[pixel, row] x grad_out[row, 32]  with a sparse
 * coefficient matrix C (attention weight x bilinear weight, rounded to bf16); bins of <= 512 pixels keep
 * their fp32 accumulators in registers, the coefficients of 16 rows at a time are written into shared memory
 * by one thread per (row, level) and multiplied with wgmma.  Levels with more than BEVF_DENSE_MAXPIX
 * pixels (default 8192), grad_loc and grad_attn come from the one-kernel backward as before.
 * Used when grad_out is bf16 and head_dim is 32 with 4 or 8 points per level; any other configuration
 * runs exactly bevf_msda_rows_backward (fp16 value or grad_out is an error).  grad_value must be zero-filled or
 * hold a running sum, as there.
 *   level_hw_host  (L, 2) int32 HOST copy of level_hw (the bins are planned on the host; a device-side
 *                  mismatch is a caller bug and traps)
 *   map_range      (B, 2) int32 DEVICE: [first, end) rows of every value map (bevf_sca_plan_build)
 * bevf_msda_set_dense_backward (process-wide): 0 = never use the dense kernel, 1 = on the caller's stream,
 * 2 = on a library-owned second stream next to the reduction kernel (fork / join with events, capturable),
 * -1 = the library default: mode 2 for bevf_msda_rows_backward_mixed_dense, off for bevf_msda_rows_backward_dense.
 * The environment variable BEVF_MSDA_DENSE=0 / 1 replaces the default.  Under the default the second stream is
 * created at the first call that is not being captured; a captured call before that runs on the caller's stream.
 * bevf_msda_get_dense_backward returns the mode bevf_msda_rows_backward_mixed_dense runs in (0, 1 or 2).
 */
BEVF_API int bevf_msda_rows_backward_dense(const void *value, int value_dtype, const int64_t *level_hw,
                                           const int64_t *level_start, const int32_t *level_hw_host,
                                           const float *loc, const float *attn, const void *grad_out,
                                           int grad_out_dtype, float *grad_value, float *grad_loc,
                                           float *grad_attn, const int32_t *row_map, const int32_t *map_range,
                                           int B, int S, int M, int D, int R, int L, int P, void *stream);
BEVF_API int bevf_msda_set_dense_backward(int mode);
BEVF_API int bevf_msda_get_dense_backward(void);
/*
 * Host-only helper: the pixel bins bevf_msda_rows_backward_dense plans for a pyramid.  bins_out receives 7 int32
 * per bin {first pixel, pixel count, number of levels, level ids (4, -1 padded)}; *level_mask the levels covered;
 * returns the number of bins (0: nothing applies), negative on a bad argument.  tiles = 8 or 16 accumulator
 * tiles of 128 pixels per bin.  No device work.
 */
BEVF_API int bevf_msda_dense_plan(const int32_t *level_hw_host, int L, int max_pix, int tiles, int32_t *bins_out,
                                  int bins_cap, uint32_t *level_mask);

/*
 * Selects how bevf_msda_*backward* computes grad_value (process-wide; default 0, or the environment
 * variable BEVF_MSDA_BWD=split).  0: one kernel, one 16 B-vector L2 reduction per corner contribution.
 * 1: gather kernel + a splat kernel that merges the contributions of 64 neighbouring rows in registers
 * before they reach L2 (fewer reductions, more instructions; kept for A/B measurements).
 * 2: hybrid -- the coarse half of the pyramid through the splat kernel on a library-owned second stream
 * (forked from / joined to the caller's stream with events: capturable), the rest in the one kernel.
 * Results agree up to fp32 summation order.  Modes 1 and 2 take fp32 / bf16 only: an fp16 backward under them fails.
 */
BEVF_API int bevf_msda_set_backward_mode(int mode);

/* ------------------------------------------------------------------------------------------------
 * Fused memory-bound pieces of one encoder layer.  "raw" is the fp32 output of the layer's combined
 * sampling_offsets|attention_weights GEMM, one row per BEV query.
 * ---------------------------------------------------------------------------------------------- */

/*
 * In-view (camera, query) pair list of SpatialCrossAttention, built on the device without a host
 * synchronisation (capturable in a CUDA graph; a new lidar2img every frame just changes the contents).
 * replaces spatial_cross_attention.py:138-141 (per-camera nonzero() + max_len: two host syncs per layer)
 * and the zero-padded re-batch at :144-153.
 *   bev_mask   (ncam, B, Nq, D) uint8    the in-view mask bevf_point_sampling writes
 *   qorder     (Nq,) int32 or NULL       order of the queries inside a camera's list (e.g. 8x8 BEV tiles)
 *   pair_q, pair_cam (capacity,) int32   out; camera-major; entries >= num_pairs are -1
 *   pair_of    (ncam, Nq) int32          out; row of (cam, q) or -1
 *   row_map    (B*capacity,) int32       out; value map b*ncam+cam of sampler row b*capacity+r, -1 = unused
 *   inv_count  (B, Nq) f32               out; 1 / max(1, #cameras seeing q in batch item b)  (:169-171)
 *   map_range  (B*ncam, 2) int32         out; [first, end) sampler rows of value map b*ncam+cam (its rows are
 *                                        contiguous) -- what bevf_msda_rows_backward_dense partitions by
 *   counters   (2,) int32                out; [0] = number of pairs found, [1] = 1 if it exceeded capacity
 *                                        (the pairs beyond capacity are dropped: the caller must check)
 *   workspace  bevf_sca_plan_workspace_ints(ncam, Nq) int32
 * The lists come from batch item 0's mask for every batch item, as in the reference (:139).  Every
 * row-list entry point of this library skips rows whose pair_q / row_map entry is -1.
 */
BEVF_API int64_t bevf_sca_plan_workspace_ints(int ncam, int Nq);
BEVF_API int bevf_sca_plan_build(const unsigned char *bev_mask, const int32_t *qorder, int32_t *pair_q,
                                 int32_t *pair_cam, int32_t *pair_of, int32_t *row_map, float *inv_count,
                                 int32_t *map_range, int32_t *counters, int32_t *workspace, int B, int ncam,
                                 int Nq, int D, int capacity, void *stream);

/*
 * SCA sampling points.  replaces spatial_cross_attention.py:338-372 (view, softmax over L*P,
 * offset / (W_l, H_l), Z-anchor broadcast "point p uses anchor p mod D", add) for the in-view
 * (camera, query) pairs only.
 *   raw      (B*Nq, M*L*P*3) f32: [offsets (M,L,P,2) | logits (M,L*P)]
 *   ref_cam  (ncam, B, Nq, D, 2) f32       pair_q, pair_cam (R,) int32
 *   loc      (B*R, M, L, P, 2) f32 out      attn (B*R, M, L, P) f32 out   (row = b*R + r)
 */
BEVF_API int bevf_sca_prep_forward(const float *raw, const float *ref_cam, const int32_t *pair_q,
                                   const int32_t *pair_cam, const int64_t *level_hw, float *loc,
                                   float *attn, int B, int Nq, int R, int M, int L, int P, int D,
                                   int ncam, void *stream);

/* Backward of the above into d_raw (B*Nq, M*L*P*3), fully overwritten, stored as out_dtype (f32, or
 * bf16 when it feeds the bf16 dX / dW GEMMs of the head directly); pair_of (ncam, Nq) int32 holds the
 * pair row of (camera, query) or -1. */
BEVF_API int bevf_sca_prep_backward(const float *raw, const float *grad_loc, const float *grad_attn,
                                    const int32_t *pair_of, const int64_t *level_hw, void *d_raw,
                                    int out_dtype, int B, int Nq, int R, int M, int L, int P, int ncam,
                                    void *stream);

/*
 * SCA's row-list sampler with the sampling-point prep fused in: the kernels derive every sample's loc / attn
 * from raw + ref_cam exactly as bevf_sca_prep_forward does (bit-identical), so loc / attn never go through
 * memory.  8 heads, head_dim 32, L * P == 32, bf16 value / output / grad_out.
 *   value (B, S, 8, 32) bf16 with B = bs * ncam value maps; row_map (R,) as for bevf_msda_rows_forward, R = bs * pairs
 *   raw, ref_cam, pair_q, pair_cam as for bevf_sca_prep_forward (pairs = its R, ncam, Dz = its D)
 *   stats (R * 8, 2) f32 out: softmax max and 1 / sum of every (pair row, head); the backward reads them
 *   coarse_loc (R, 8, L - coarse_from, P, 2), coarse_attn (R, 8, L - coarse_from, P) f32 out: the samples of the levels
 *   [coarse_from, L), which the backward's dense tensor-core kernel reads; coarse_from = L: none (pointers may be NULL)
 */
BEVF_API int bevf_sca_rows_forward_fused(const void *value, int value_dtype, const int64_t *level_hw,
                                         const int64_t *level_start, const float *raw, const float *ref_cam,
                                         const int32_t *pair_q, const int32_t *pair_cam, float *stats,
                                         float *coarse_loc, float *coarse_attn, int coarse_from, void *out,
                                         int out_dtype, const int32_t *row_map, int B, int S, int M, int D, int R,
                                         int L, int P, int bs, int Nq, int pairs, int Dz, int ncam, void *stream);

/* Backward of the above with bevf_msda_rows_backward_mixed_dense's grad_value accumulation (map_range NULL: that
 * of bevf_msda_rows_backward_mixed without the dense kernel; the dense kernel runs only where the forward stored the
 * samples of its levels, coarse_from <= first_dense_level).  The d_raw rows (bf16, layout of raw) of the queries
 * seen by exactly one camera (counted in pair_of) are finished here; the other pair rows store grad_loc / grad_attn
 * ((R, 8, L, P, 2) / (R, 8, L, P) f32 scratch) and bevf_sca_prep_backward_multi completes d_raw from them. */
BEVF_API int bevf_sca_rows_backward_fused(const void *value, int value_dtype, const int64_t *level_hw,
                                          const int64_t *level_start, const int32_t *level_hw_host, const float *raw,
                                          const float *stats, const float *coarse_loc, const float *coarse_attn,
                                          int coarse_from, const float *ref_cam, const int32_t *pair_q,
                                          const int32_t *pair_cam, const int32_t *pair_of, const void *grad_out,
                                          int grad_out_dtype, void *grad_value_fine_f16, float *grad_value_side,
                                          const uint32_t *amax_bits, int num_f16_levels, int first_dense_level,
                                          float *grad_loc, float *grad_attn, void *d_raw, const int32_t *row_map,
                                          const int32_t *map_range, int B, int S, int M, int D, int R, int L, int P,
                                          int bs, int Nq, int pairs, int Dz, int ncam, void *stream);

/* bevf_sca_prep_backward for the queries NOT seen by exactly one camera (0 cameras: zero rows; 2+: the sum over
 * their pair rows in camera order); the rows of one-camera queries are left as they are.  8 heads, L * P == 32,
 * bf16 / fp16 d_raw. */
BEVF_API int bevf_sca_prep_backward_multi(const float *raw, const float *grad_loc, const float *grad_attn,
                                          const int32_t *pair_of, const int64_t *level_hw, void *d_raw,
                                          int out_dtype, int B, int Nq, int R, int M, int L, int P, int ncam,
                                          void *stream);

/*
 * TSA sampling points.  replaces temporal_self_attention.py:206-229 (view, softmax over L*P per
 * queue entry, the two permute+reshape copies, offset / (W, H) + reference point).
 *   raw    (B*Nq, M*2*L*P*3) f32: [offsets (M,2,L,P,2) | logits (M,2,L*P)]
 *   ref2d  (B*2, Nq, L, 2) f32 (the encoder's hybird_ref_2d)
 *   loc    (B*2, Nq, M, L, P, 2) f32 out     attn (B*2, Nq, M, L, P) f32 out
 *   interleave != 0 orders the output rows (b, q, frame) instead of (b, frame, q): the two frames of a
 *   query become adjacent rows, so the row-list sampler's output is (B*Nq, 2*C) and the average over
 *   the frames (temporal_self_attention.py:257-265) folds into the output projection.
 */
BEVF_API int bevf_tsa_prep_forward(const float *raw, const float *ref2d, const int64_t *level_hw,
                                   float *loc, float *attn, int B, int Nq, int M, int L, int P,
                                   int interleave, void *stream);

/* d_raw (B*Nq, M*2*L*P*3) stored as out_dtype (f32 or bf16), fully overwritten. */
BEVF_API int bevf_tsa_prep_backward(const float *raw, const float *grad_loc, const float *grad_attn,
                                    const int64_t *level_hw, void *d_raw, int out_dtype, int B, int Nq,
                                    int M, int L, int P, int interleave, void *stream);

/*
 * The same preparation for F in {1, 2} frames (queue entries); bevf_tsa_prep_* are the F = 2 calls, and the
 * decoder's CustomMSDeformableAttention (decoder.py:300-330: softmax over L*P, offset / (W, H) + reference point)
 * is F = 1.
 *   raw    (B*Nq, M*F*L*P*3) f32: [offsets (M,F,L,P,2) | logits (M,F,L*P)]
 *   ref2d  (B*F, Nq, L, 2) f32
 *   loc    (B*F, Nq, M, L, P, 2) f32 out     attn (B*F, Nq, M, L, P) f32 out   (interleave: rows (b, q, frame))
 *   d_raw  (B*Nq, M*F*L*P*3) as out_dtype (f32, bf16 or f16), fully overwritten.
 */
BEVF_API int bevf_query_prep_forward(const float *raw, const float *ref2d, const int64_t *level_hw,
                                     float *loc, float *attn, int B, int Nq, int M, int L, int P, int F,
                                     int interleave, void *stream);
BEVF_API int bevf_query_prep_backward(const float *raw, const float *grad_loc, const float *grad_attn,
                                      const int64_t *level_hw, void *d_raw, int out_dtype, int B, int Nq, int M,
                                      int L, int P, int F, int interleave, void *stream);

/*
 * Reference-point refinement of DetectionTransformerDecoder (decoder.py:106-118), forward only (the result is
 * detached):  out[r, c] = sigmoid(tmp[r, col_c] + inverse_sigmoid(ref[r, c])), col = (0, 1, 4), eps = 1e-5.
 *   tmp    (rows, >= 5) rows tmp_row_stride elements apart (the regression branch output, read in place)
 *   ref    (rows, 3) contiguous     out (rows, 3) contiguous; tmp, ref, out all in `dtype` (f32 | bf16 | f16)
 *   ref2d  optional (rows, 2) f32 out: the x, y of `out`, the next layer's sampling-point prep input
 */
BEVF_API int bevf_refine_points(const void *tmp, int64_t tmp_row_stride, const void *ref, void *out, float *ref2d,
                                int dtype, int64_t rows, void *stream);

/*
 * y = LayerNorm(dropout(x) + residual) * gamma + beta, optionally also y_plus_pos = y + pos.
 * replaces the `norm` steps of BEVFormerLayer.forward (encoder.py:377-379) together with the
 * preceding "self.dropout(output) + identity" of the attention / FFN
 * (temporal_self_attention.py:272, spatial_cross_attention.py:175, mmcv FFN) and TSA's
 * `query + query_pos` (temporal_self_attention.py:186-187).
 *   x, residual, pos, y, y_plus_pos: (rows, C) in `dtype` (f32 | bf16 | f16); gamma, beta: (C) in `param_dtype`
 *   (f32, or the 16-bit `dtype` itself);
 *   mean, rstd: (rows) f32.  residual / pos / y_plus_pos / mean / rstd may be NULL.  C in {256, 512}.
 *   drop_p in [0,1): inverted dropout on x with keep-mask bits from Philox4x32-10(seed, row*32+lane);
 *   the backward regenerates the same bits from `seed`, no mask tensor exists.  drop_p = 0: no dropout.
 *   seed_base (DEVICE, may be NULL) is added to seed inside the kernel: a step counter kept on the
 *   device lets a captured CUDA graph draw new masks on every replay.
 */
BEVF_API int bevf_layernorm_forward(const void *x, const void *residual, const void *gamma,
                                    const void *beta, int param_dtype, const void *pos, void *y,
                                    void *y_plus_pos, float *mean, float *rstd, int64_t rows, int C,
                                    float eps, float drop_p, uint64_t seed, const uint64_t *seed_base,
                                    int dtype, void *stream);

/* dx (rows, C) = gradient of x, fully overwritten; dres = gradient of residual (may be NULL when
 * drop_p == 0: it then equals dx); dgamma / dbeta (C,) f32 are ACCUMULATED INTO.  dy_plus_pos may be
 * NULL; its rows may be strided (dy_plus_pos_ld elements between rows, 0 = C): it usually arrives as a
 * column slice of the gradient of cat([prev_bev, query + pos]).  drop_p / seed must be the forward call's. */
BEVF_API int bevf_layernorm_backward(const void *x, const void *residual, const void *gamma,
                                     int param_dtype, const float *mean, const float *rstd,
                                     const void *dy, const void *dy_plus_pos, int64_t dy_plus_pos_ld,
                                     void *dx, void *dres, float *dgamma, float *dbeta, int64_t rows,
                                     int C, float drop_p, uint64_t seed, const uint64_t *seed_base,
                                     int dtype, void *stream);

/* Deterministic form of bevf_layernorm_backward: the warps of a CTA are combined in index order and every CTA stores
 * its [dgamma | dbeta] partial row into `workspace`; a second kernel sums the rows in CTA order and adds them into
 * dgamma / dbeta (still ACCUMULATED INTO).  Same results run to run on one GPU model (the partition follows the SM
 * count).  bevf_layernorm_backward_workspace_bytes(rows, C) gives the workspace size. */
BEVF_API int64_t bevf_layernorm_backward_workspace_bytes(int64_t rows, int C);
BEVF_API int bevf_layernorm_backward_det(const void *x, const void *residual, const void *gamma,
                                         int param_dtype, const float *mean, const float *rstd,
                                         const void *dy, const void *dy_plus_pos, int64_t dy_plus_pos_ld,
                                         void *dx, void *dres, float *dgamma, float *dbeta, void *workspace,
                                         int64_t workspace_bytes, int64_t rows, int C, float drop_p, uint64_t seed,
                                         const uint64_t *seed_base, int dtype, void *stream);

/*
 * slots[b,q,:] = inv_count[b,q] * sum_{cameras seeing q} out[b*R + pair_of[cam][q], :]
 * replaces spatial_cross_attention.py:165-172 (python scatter-add loops, count, divide).
 */
BEVF_API int bevf_sca_combine_forward(const void *out, const int32_t *pair_of,
                                      const float *inv_count, void *slots, int B, int Nq, int R,
                                      int C, int ncam, int dtype, void *stream);

BEVF_API int bevf_sca_combine_backward(const void *g_slots, const int32_t *pair_q,
                                       const float *inv_count, void *g_out, int B, int Nq, int R,
                                       int C, int dtype, void *stream);

/*
 * One pyramid level of camera features into the encoder's key/value layout, embeddings added.
 * replaces PerceptionTransformer.get_bev_features' flatten / permute / +cams_embeds / +level_embeds /
 * cat / permute (transformer.py:161-181).
 *   feat (bs, ncam, C, hw) T in;  cams_embeds (ncam, C) f32 or null;  level_embed (C) f32;
 *   out (ncam, S, bs, C) T: rows [level_start, level_start + hw) of every camera are written.
 */
BEVF_API int bevf_flatten_feats(const void *feat, const float *cams_embeds, const float *level_embed,
                                void *out, int bs, int ncam, int C, int hw, int S, int level_start,
                                int dtype, void *stream);

/*
 * Projection of the pillar anchors into every camera + in-view mask, fp32 without FMA contraction.
 * replaces BEVFormerEncoder.get_reference_points(dim='3d') + point_sampling (encoder.py:46-71,
 * 88-149), including the 61 MB repeated-matrix materialisation.
 *   lidar2img (B, ncam, 4, 4) f32 DEVICE; pc_range (6) and z_norm (D) HOST arrays;
 *   ref_cam (ncam, B, Nq, D, 2) f32 out; bev_mask (ncam, B, Nq, D) uint8 out; Nq = bev_h*bev_w.
 */
BEVF_API int bevf_point_sampling(const float *lidar2img, const float *pc_range, const float *z_norm,
                                 float img_h, float img_w, float *ref_cam, uint8_t *bev_mask, int B,
                                 int ncam, int bev_h, int bev_w, int D, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Dense projection on the tensor cores (TMA + wgmma):
 *     y[M,N] = act( x[M,K] . w[N,K]^T + bias[N] ) (+ residual[M,N])
 * replaces nn.Linear (cuBLAS GEMM + bias) and the ReLU / "+ identity" launches that follow it in
 * TemporalSelfAttention (temporal_self_attention.py:198,206-209,267), MSDeformableAttention3D /
 * SpatialCrossAttention (spatial_cross_attention.py:334,338-341,173) and mmcv's FFN.
 *   x (M,K) bf16, w (N,K) bf16 (nn.Linear layout), bias (N) in bias_dtype (f32 | bf16) or NULL,
 *   residual (M,N) bf16 or NULL,
 *   y (M,N) in y_dtype (bf16 | f32, straight from the fp32 accumulator).  relu != 0 applies
 *   max(.,0) before the residual add.  K % 64 == 0, N % 16 == 0.
 */
BEVF_API int bevf_linear_forward(const void *x, const void *w, const void *bias, int bias_dtype,
                                 const void *residual, void *y, int y_dtype, int64_t M, int N, int K,
                                 int relu, void *stream);

/*
 * Input gradient of a projection: dx (M, K) bf16 = dy (M, N) bf16 . w (N, K) bf16 -- the
 * `grad_input = grad_output.mm(weight)` half of F.linear's backward.  Same wgmma kernel as
 * bevf_linear_forward, but the weight is read in place as an MN-major operand (no W^T copy).
 * N and K must be multiples of 64.
 */
BEVF_API int bevf_linear_dgrad(const void *dy, const void *w, void *dx, int64_t M, int N, int K,
                               void *stream);

/*
 * dX = addend + dY . W : the same kernel with a (M, K) bf16 addend read in the epilogue (may alias dx).
 * Layers that share an input (the camera features feed every layer's value_proj; the BEV queue feeds every
 * layer's temporal value_proj) chain their input gradients through it instead of materialising one
 * gradient per layer and summing them with separate element-wise kernels.
 */
BEVF_API int bevf_linear_dgrad_acc(const void *dy, const void *w, const void *addend, void *dx, int64_t M,
                                   int N, int K, void *stream);

/*
 * Weight gradient of the projection above:  dw[N,K] += dy[M,N]^T . x[M,K]   (fp32, ACCUMULATED
 * INTO: the caller zero-fills).  dy, x bf16 row-major; split over the M rows across the SMs, partial
 * tiles combined with 16 B fp32 reductions.  replaces the cuBLAS call autograd makes for
 * nn.Linear.weight.grad.  K % 64 == 0, N % 8 == 0.  db (N) f32, optional: the bias gradient
 * db[n] += sum_m dy[m, n], summed from the dY tiles while they sit in shared memory (no second pass
 * over dy; replaces the at::reduce_kernel behind nn.Linear.bias.grad).
 */
BEVF_API int bevf_linear_wgrad(const void *dy, const void *x, float *dw, float *db, int64_t M, int N,
                               int K, void *stream);

/* out[c] += sum over rows of x[r, c]  (fp32, ACCUMULATED INTO).  The bias gradient of the projections:
 * replaces the at::reduce_kernel autograd launches for nn.Linear.bias.grad.  x (rows, C) f32 | bf16 | f16. */
/* out = srcs[0] + ... + srcs[n-1] (n <= 8 device tensors of `numel` elements, f32, bf16 or f16, fp32 accumulation):
 * the one-pass sum of the per-layer input gradients of a shared input (replaces autograd's chain of
 * pairwise add kernels).  `srcs` is a HOST array of device pointers. */
BEVF_API int bevf_sum_tensors(const void *const *srcs, int n, void *out, int64_t numel, int dtype, void *stream);

BEVF_API int bevf_colsum(const void *x, float *out, int64_t rows, int C, int dtype, void *stream);

/* Deterministic form of bevf_colsum: per-CTA column sums stored into `workspace`, then summed in CTA order and added
 * into out.  bevf_colsum_workspace_bytes(rows, C) gives the workspace size. */
BEVF_API int64_t bevf_colsum_workspace_bytes(int64_t rows, int C);
BEVF_API int bevf_colsum_det(const void *x, float *out, void *workspace, int64_t workspace_bytes, int64_t rows, int C,
                             int dtype, void *stream);

/*
 * The FFN's hidden dropout (mmcv FFN: Linear -> ReLU -> Dropout; the ReLU itself is fused into
 * bevf_linear_forward's epilogue) and the joint backward of dropout(relu(z)).
 *   bevf_dropout_inplace: x *= keep / (1 - p) with Philox4x32-10(seed [+ *seed_base], element / vec) bits,
 *     no mask tensor.  replaces at::native::fused_dropout.
 *   bevf_relu_dropout_backward: out = dy * scale where h != 0, else 0, with h the SAVED forward
 *     activation dropout(relu(z)) (h != 0 <=> z > 0 and kept) and scale = 1 / (1 - p).  replaces
 *     masked_scale + threshold_backward.  dy, h, out: n elements in `dtype`.
 */
BEVF_API int bevf_dropout_inplace(void *x, int64_t n, float p, uint64_t seed, const uint64_t *seed_base,
                                  int dtype, void *stream);
BEVF_API int bevf_relu_dropout_backward(const void *dy, const void *h, void *out, int64_t n, float scale,
                                        int dtype, void *stream);

/*
 * Two-pass form of the weight (+ bias) gradient: every split of the M rows stores its partial 128-row
 * tiles into its own slab of `workspace` with plain stores (no SM-count-way contended reductions), then a
 * small kernel sums the slabs and writes dw (N, K) and db (N) -- fully OVERWRITTEN, in grad_dtype
 * (f32 | bf16, i.e. the parameter's dtype: no zero-fill and no cast launch around the call).
 * bevf_linear_wgrad_workspace_bytes gives the scratch size for a problem; db may be NULL.
 */
BEVF_API int64_t bevf_linear_wgrad_workspace_bytes(int64_t M, int N, int K);
BEVF_API int bevf_linear_wgrad_out(const void *dy, const void *x, void *dw, void *db, int grad_dtype,
                                   void *workspace, int64_t workspace_bytes, int64_t M, int N, int K,
                                   void *stream);
/* The same two passes, ACCUMULATING into fp32 dw (N, K) / db (N) (the gradient arena).  Both passes sum in a fixed
 * order (the bias column sums of pass 1 too), so this and bevf_linear_wgrad_out are deterministic run to run on one
 * GPU model; the workspace is bevf_linear_wgrad_workspace_bytes(M, N, K). */
BEVF_API int bevf_linear_wgrad_into(const void *dy, const void *x, float *dw, float *db, void *workspace,
                                    int64_t workspace_bytes, int64_t M, int N, int K, void *stream);

/*
 * The projections above with the operand type as an argument: `dtype` = BEVF_DTYPE_BF16 or BEVF_DTYPE_F16 for x, w,
 * dy, the residual / addend and 16-bit outputs (wgmma .f16 / .bf16 with fp32 accumulation; the kernels and their
 * speed are the same for both).  bias_dtype is f32 or `dtype`, y_dtype f32 or `dtype`, grad_dtype (wgrad_out) f32,
 * bf16 or f16.  The names without _dt are these with dtype = BEVF_DTYPE_BF16.
 */
BEVF_API int bevf_linear_forward_dt(const void *x, const void *w, const void *bias, int bias_dtype,
                                    const void *residual, void *y, int y_dtype, int64_t M, int N, int K,
                                    int relu, int dtype, void *stream);
BEVF_API int bevf_linear_dgrad_dt(const void *dy, const void *w, void *dx, int64_t M, int N, int K, int dtype,
                                  void *stream);
BEVF_API int bevf_linear_dgrad_acc_dt(const void *dy, const void *w, const void *addend, void *dx, int64_t M,
                                      int N, int K, int dtype, void *stream);
BEVF_API int bevf_linear_wgrad_dt(const void *dy, const void *x, float *dw, float *db, int64_t M, int N,
                                  int K, int dtype, void *stream);
BEVF_API int bevf_linear_wgrad_out_dt(const void *dy, const void *x, void *dw, void *db, int grad_dtype,
                                      void *workspace, int64_t workspace_bytes, int64_t M, int N, int K,
                                      int dtype, void *stream);
BEVF_API int bevf_linear_wgrad_into_dt(const void *dy, const void *x, float *dw, float *db, void *workspace,
                                       int64_t workspace_bytes, int64_t M, int N, int K, int dtype,
                                       void *stream);

/*
 * Grouped ("block-diagonal") multi-head softmax attention, head_dim 32, bf16 / fp16 storage (dtype), fp32
 * accumulation.  Replaces the split / cat along the batch axis around nn.MultiheadAttention in
 * GroupMultiheadAttention.forward (projects/mmdet3d_plugin/bevformer/modules/group_attention.py:117-162): the
 * `groups` equal slices of nq queries each attend only to the same slice of the nk keys.
 *
 * Layout (sequence-first, read and written in place): element (token t, batch b, head h, channel c) of an operand X
 * with row stride ldx (elements, multiple of 8, >= heads * 32) is X[(t * bs + b) * ldx + h * 32 + c].  Q, K, V and
 * their gradients each have their own pointer and stride, so [Q | K] may be one (N, bs, 2C) buffer.
 *
 * bevf_attn_forward writes out (nq, bs, ldo) and lse (bs, groups, heads, nq / groups), the natural-log log-sum-exp of
 * the scaled scores in fp32.  drop_p > 0 drops attention probabilities (inverted dropout, torch's
 * nn.MultiheadAttention semantics; the normaliser uses the undropped probabilities).  The keep bits come from
 * Philox4x32-10 keyed by seed + *seed_base (seed_base may be NULL; a device word so CUDA-graph replays draw new
 * masks) and the indices (b, group, head, query, key); nothing is stored.
 *
 * bevf_attn_backward writes dq, dk, dv (fully overwritten, same layout) from the forward's out and lse and the
 * output gradient.  It runs two passes without atomics (queries outer for dQ and D = rowsum(dO * O), written to
 * delta (bs, groups, heads, nq / groups) fp32 scratch; keys outer for dK and dV), so the result repeats bit for bit.
 * seed, seed_base and drop_p must be the forward's.
 *
 * Other head dims and fp32 storage are not kernel cases and return an error.
 */
BEVF_API int bevf_attn_forward(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                               void *out, int64_t ldo, float *lse, int nq, int nk, int bs, int heads, int head_dim,
                               int groups, float scale, float drop_p, uint64_t seed, const uint64_t *seed_base,
                               int dtype, void *stream);
BEVF_API int bevf_attn_backward(const void *q, int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                const void *out, int64_t ldo, const void *grad_out, int64_t ldgo, const float *lse,
                                float *delta, void *dq, int64_t lddq, void *dk, int64_t lddk, void *dv, int64_t lddv,
                                int nq, int nk, int bs, int heads, int head_dim, int groups, float scale, float drop_p,
                                uint64_t seed, const uint64_t *seed_base, int dtype, void *stream);
/* Test and debugging aid: the keep-mask (1 = kept) that bevf_attn_forward / _backward apply for these arguments,
 * as uint8 (bs, groups, heads, nq / groups, nk / groups). */
BEVF_API int bevf_attn_dropout_mask(uint8_t *mask, int nq, int nk, int bs, int heads, int groups, float drop_p,
                                    uint64_t seed, const uint64_t *seed_base, void *stream);

/* ------------------------------------------------------------------------------------------------
 * The once-per-frame ego-motion block of PerceptionTransformer.get_bev_features on the device
 * (transformer.py:122-153, detectors/bevformer.py:254-268): no host arithmetic, so a video frame can be
 * captured in a CUDA graph and replayed with a new CAN-bus vector.
 *
 * bevf_ego_motion, one launch per frame:
 *   can_bus (bs, 18) f64 DEVICE: [0:3] ego translation, [16] ego yaw (rad), [17] yaw (deg).
 *   mode    BEVF_EGO_DELTAS    can_bus already holds deltas to the previous frame; state is not touched (may be NULL)
 *           BEVF_EGO_CONTINUE  can_bus is absolute: sample 0's position / angle become deltas against the state
 *                              when it has history (zeros when it has not), then the state takes this frame's
 *                              absolute values
 *           BEVF_EGO_NEW_SCENE can_bus is absolute, first frame of a scene: sample 0's position / angle become
 *                              zeros, the state takes this frame's absolute values
 *   state   40 bytes, 8-byte aligned: double prev_pos[3]; double prev_angle; int64 has_history (all-zero = empty).
 *   shift (bs, 2) f32 out: the BEV shift (x, y) in float64, rounded to out_dtype and widened to f32 (what
 *           bev_queries.new_tensor(shift) followed by the encoder's .float() holds); zeros with use_shift == 0.
 *   rot   (bs, 6) f32 out: torchvision's rotate(img, angle = can_bus[17], center) as the rows of its sampling
 *           grid: _get_inverse_affine_matrix(center - size / 2, -angle) in float64, rounded to f32, x row divided by
 *           0.5 * bev_w and y row by 0.5 * bev_h (_gen_affine_grid).  center = (center_x, center_y) in pixels.
 *   can_bus_out (bs, 18) out_dtype: the CAN-bus MLP input (deltas applied).
 *
 * bevf_rotate_bev: out[q, b, :] = prev[src(q), b, :], or zeros where src falls outside the map; src is the
 * nearest cell (ties to even) of grid_sample(align_corners=False) under the grid `rot` describes, computed in f32
 * for every storage type.  prev: element (q, b, c) at prev[q * stride_q + b * stride_b + c] (so (Nq, bs, C) and
 * (bs, Nq, C) are both read in place), in_dtype; out (Nq, bs, C) contiguous, out_dtype.  C % 8 == 0, strides % 8 == 0.
 * Values are copied, so apart from the cast the result is exact.  out must not alias prev.
 */
enum bevf_ego_mode { BEVF_EGO_DELTAS = 0, BEVF_EGO_CONTINUE = 1, BEVF_EGO_NEW_SCENE = 2 };
BEVF_API int bevf_ego_motion(const double *can_bus, void *state, int mode, float *shift, float *rot,
                             void *can_bus_out, int out_dtype, int bs, int bev_h, int bev_w, double grid_h,
                             double grid_w, double center_x, double center_y, int use_shift, void *stream);
BEVF_API int bevf_rotate_bev(const void *prev, int in_dtype, int64_t stride_q, int64_t stride_b, const float *rot,
                             void *out, int out_dtype, int bs, int bev_h, int bev_w, int C, void *stream);

/*
 * Detection head (BEVFormerHead.forward after the transformer, dense_heads/bevformer_head.py:171-203), inference only:
 * per decoder level l the classification branch (Linear-LayerNorm-ReLU x 2, Linear -> ncls) and the regression branch
 * (Linear-ReLU x 2, Linear -> 10) on the level's decoder states, then on the regression output
 *   out[c] = sigmoid(tmp[c] + inverse_sigmoid(ref[c'])) * (pc_range[c' + 3] - pc_range[c']) + pc_range[c'],
 *   (c, c') in {(0, 0), (1, 1), (4, 2)}, inverse_sigmoid with eps 1e-5, evaluated in fp32 and rounded once.
 * One launch, one CTA per (level, branch, 64-row tile); the hidden activations stay in shared memory.
 *   x          decoder states (L, nq, bs, C = 256) in `dtype` (bf16 | f16): element (l, q, b, c) at
 *              x[l * stride_l + q * stride_q + b * stride_b + c]; strides multiples of 8
 *   ref0       (bs, nq, 3) initial reference points; refs (L, bs, nq, 3) the decoder's, level l > 0 reads refs[l - 1];
 *              both in ref_dtype (f32 | bf16 | f16)
 *   params     HOST array of L * 16 device pointers, per level: cls W0 b0 gamma0 beta0 W1 b1 gamma1 beta1 W2 b2, then
 *              reg W0 b0 W1 b1 W2 b2; weights row-major (out, 256); all in param_dtype (`dtype` or f32: fp32 weights
 *              and Linear biases are rounded to `dtype`, as autocast's Linear rounds them; LayerNorm's in fp32).  Copied into the kernel's parameters at the call, so a
 *              captured launch keeps reading the same parameter tensors.
 *   cls_out    (L, bs, nq, ncls) and box_out (L, bs, nq, 10) in `dtype`
 *   1 <= L <= 8, ncls <= 16, code_size == 10; ln_eps the LayerNorms' eps; pc_range HOST array of 6 doubles.
 */
BEVF_API int bevf_det_branches_forward(const void *x, int64_t stride_l, int64_t stride_q, int64_t stride_b, int dtype,
                                       const void *ref0, const void *refs, int ref_dtype, const void *const *params,
                                       int param_dtype, void *cls_out, void *box_out, int L, int bs, int nq, int C,
                                       int ncls, int code_size, float ln_eps, const double *pc_range, void *stream);

/*
 * NMSFreeCoder.decode (core/bbox/coders/nms_free_coder.py:40-121) for a batch, one CTA per sample, no host
 * synchronisation.  cls (bs, nq, ncls) logits and box (bs, nq, 10) normalised boxes, contiguous, any dtype code
 * (widened to fp32).  scores = 1 / (1 + expf(-x)) in IEEE fp32 (torch.sigmoid's arithmetic, subnormal results
 * included); the max_num largest of the nq * ncls scores are
 * selected and ordered by (score descending, flat index ascending) -- a tie rule torch.topk leaves unspecified;
 * label = idx % ncls, box = denormalize_bbox(box[idx / ncls]) = (cx, cy, cz, exp w, exp l, exp h,
 * atan2(sin, cos), vx, vy).  With has_threshold (a threshold that is given and non-zero) the reference's decay loop
 * picks the mask: score > t, else score >= t * 0.9^i (t * 0.9^i in double, compared in fp32) for the first i
 * the top score passes, else (t * 0.9^i < 0.01) score > -1.  Kept: centre within post_center_range (HOST float[6],
 * inclusive) and the threshold mask.  Outputs, in candidate order, compacted: bboxes (bs, max_num, 9) f32,
 * scores (bs, max_num) f32, labels (bs, max_num) i64, num (bs) i32; slots past num are zero.  z_shift: z -= h / 2
 * (BEVFormerHead.get_bboxes).  max_num <= nq * ncls and bevf_nms_free_decode_smem_bytes(...) <= 200 KiB.
 */
BEVF_API int bevf_nms_free_decode(const void *cls, int cls_dtype, const void *box, int box_dtype, int bs, int nq,
                                  int ncls, int code_size, int max_num, const float *post_center_range,
                                  int has_threshold, double score_threshold, int z_shift, float *bboxes,
                                  float *scores, int64_t *labels, int *num, void *stream);
BEVF_API int64_t bevf_nms_free_decode_smem_bytes(int nq, int ncls, int max_num);

/*
 * Training loss of BEVFormerHead / BEVFormerHead_GroupDETR around a host-side Hungarian assignment.
 * Common arguments:
 *   cls        (P, nq, ncls) logits, box (P, nq, 10) normalised boxes, contiguous, any dtype code (widened to fp32);
 *              P = L * bs, row p = l * bs + b (all_cls_scores / all_bbox_preds flattened over layer and sample)
 *   gt         (bs, G, 9) f32 gravity-centred boxes (x, y, z, w, l, h, rot, vx, vy), gt_labels (bs, G) int64,
 *              n_gt (bs) int32: sample b's first n_gt[b] boxes are real, the rest padding; the kernels normalise
 *              them (normalize_bbox, core/bbox/util.py:4-24: cx, cy, log w, log l, cz, log h, sin rot, cos rot, vx, vy)
 *   reg_kind   BEVF_DET_REG_L1 (BBox3DL1Cost / L1Loss) or BEVF_DET_REG_SMOOTH_L1 (SmoothL1Cost / SmoothL1Loss)
 *   alpha, gamma  the focal parameters (mmdet's FocalLossCost / FocalLoss)
 * The sigmoid is rounded to fp32 as torch.sigmoid computes it (libdevice expf, IEEE division), as are 1 - p and
 * p + eps; the rest is evaluated in double and rounded once.
 */
enum bevf_det_reg { BEVF_DET_REG_L1 = 0, BEVF_DET_REG_SMOOTH_L1 = 1 };

/*
 * HungarianAssigner3D.assign's cost (core/bbox/assigners/hungarian_assigner_3d.py:106-116) for every (layer, sample)
 * in one launch:
 *   cost[p, q, g] = cls_weight * (pos - neg)[label_g] + reg_weight * reg(box[p, q, :8], normalize_bbox(gt[b, g])[:8])
 *   pos = -log(p + eps) alpha (1 - p)^gamma, neg = -log(1 - p + eps) (1 - alpha) p^gamma   (mmdet 2.14 FocalLossCost)
 *   reg = sum |d| (BBox3DL1Cost, match_costs/match_cost.py:7-29) or sum smooth-L1(d, beta 1) (SmoothL1Cost, :32-90)
 * cost (P, nq, G) f32; columns g >= n_gt[b] are 0 and a label outside [0, ncls) gives NaN.  Query groups are ranges
 * of q.  1 <= ncls <= 64, G >= 1 and bevf_det_match_cost_smem_bytes(ncls, G) <= 200 KiB.
 */
BEVF_API int bevf_det_match_cost(const void *cls, int cls_dtype, const void *box, int box_dtype, const float *gt,
                                 const int64_t *gt_labels, const int *n_gt, float *cost, int P, int bs, int nq,
                                 int ncls, int G, int reg_kind, float cls_weight, float reg_weight, float alpha,
                                 float gamma, float eps, void *stream);
BEVF_API int64_t bevf_det_match_cost_smem_bytes(int ncls, int G);

/*
 * BEVFormerHead.loss_single after the assignment (dense_heads/bevformer_head.py:215-393) for every slot s = l * groups
 * + group in one launch; the slot's rows are (b, q) for all samples and q in [group * nq / groups, (group + 1) * nq /
 * groups).
 *   assign     (P, nq) int32: the ground-truth index matched to the query, or -1 (PseudoSampler: matched rows are
 *              positive, with label gt_labels[b, assign]; the others have label num_classes = ncls)
 *   loss_cls   mmcv 1.4's CUDA sigmoid_focal_loss (-alpha (1-p)^gamma log(max(p, FLT_MIN)) on the label's channel,
 *              -(1-alpha) p^gamma log(max(1-p, FLT_MIN)) on the others), summed, / max(avg[s, 0], 1) * cls_loss_weight
 *   loss_bbox  sum over positive rows whose normalised target is all finite (the reference's isnotnan) of
 *              code_weights[c] * l(box - target) with l = |d| or smooth-L1 (beta), / max(avg[s, 1], 1)
 *              * bbox_loss_weight
 *   code_weights (10) f32; avg (S, 2) f32 in device memory; loss (S, 2) = nan_to_num of the values, loss_raw (S, 2) the
 *   values before it (the backward reads them).  S = L * groups; one CTA per slot, fixed-order double sums.
 */
BEVF_API int bevf_det_loss_forward(const void *cls, int cls_dtype, const void *box, int box_dtype, const int *assign,
                                   const float *gt, const int64_t *gt_labels, const int *n_gt,
                                   const float *code_weights, const float *avg, float *loss, float *loss_raw, int L,
                                   int bs, int nq, int groups, int ncls, int G, int reg_kind, float cls_loss_weight,
                                   float bbox_loss_weight, float alpha, float gamma, float beta, void *stream);

/*
 * Gradient of bevf_det_loss_forward's slot scalars: grad_loss (S, 2) f32 is the upstream gradient of loss; a slot
 * whose loss_raw is not finite passes none (nan_to_num).  grad_cls (P, nq, ncls) in cls_dtype (mmcv's analytic
 * focal backward), grad_box (P, nq, 10) in box_dtype (sign(d), or d / beta inside smooth-L1's quadratic zone, times
 * code_weights; zero on rows the forward dropped).  Every element is written once: no atomics.
 */
BEVF_API int bevf_det_loss_backward(const void *cls, int cls_dtype, const void *box, int box_dtype, const int *assign,
                                    const float *gt, const int64_t *gt_labels, const int *n_gt,
                                    const float *code_weights, const float *avg, const float *loss_raw,
                                    const float *grad_loss, void *grad_cls, void *grad_box, int L, int bs, int nq,
                                    int groups, int ncls, int G, int reg_kind, float cls_loss_weight,
                                    float bbox_loss_weight, float alpha, float gamma, float beta, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BEVFORMER_B200_H_ */
