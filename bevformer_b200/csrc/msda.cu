// Multi-scale deformable attention sampler for sm_90a: the irregular multi-camera / multi-level
// bilinear gather + attention-weighted reduce, and its backward.
//
// Replaces the reference's native op (mmcv._ext.ms_deform_attn_{forward,backward}; call sites
// projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:118-124 and
// :150-160).  Arithmetic: SURVEY.md Appendix A.  This is gather/scatter work bound by L1/L2 and
// instruction issue, not GEMM-shaped: no tensor cores.
//
// Mapping (head_dim == 32 fast path).  One (pixel, head) row of `value` is 32 contiguous channels:
// 128 B in fp32, 64 B in bf16.  A lane owns 16 B of it (4 fp32 / 8 bf16 channels), so a row is
// covered by LANES = 8 (fp32) or 4 (bf16) adjacent lanes and one warp works on G = 4 / 8 consecutive
// (query, head) pairs at once.
//   * Every corner fetch is one fully-used 16 B vector load per lane.
//   * The per-sample scalar work (pixel coordinates, range test, bilinear weights x attention weight,
//     corner addresses) is done ONCE per sample: in each round the LANES lanes of a group take LANES
//     different samples, then hand {packed corner address, weights} round with __shfl_sync.
//   * Samples that are out of view for every (query, head) pair of the warp are skipped with one
//     ballot (in SCA all 8 heads of a query share the projected anchor, so whole anchors drop out).
//   * bf16 storage: fp32 accumulation through fhfma (msda_common.cuh): the bf16 operands are
//     widened from register halves (a shift each) and fed to one fp32 FMA.
//   * backward: per sample only the four dot products <grad_out, corner> are formed per lane; they
//     are reduce-scattered over the group so that the lane that produced the sample's scalars also
//     finishes grad_loc / grad_attn.  grad_value is scattered with 16 B vector reductions
//     (REDG.E.ADD.F32x4), never scalar atomics.
#include <cuda_fp16.h>

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <type_traits>

#include "msda_common.cuh"

namespace bevf {

// ------------------------------------------------------------------------------------------------
// forward, head_dim == 32
// ------------------------------------------------------------------------------------------------
// kFused: loc / attn are derived from SCA's raw head output (ScaFuse, msda_common.cuh).  A prologue computes the row's
// softmax statistics (stored for the backward) and its 32 attention weights, which the produce phase reads back from
// shared memory; the samples of the levels the dense backward takes are also stored (ScaFuse::coarse_*)
template <typename T, typename TO, bool kFused = false>
__global__ void __launch_bounds__(kThreads)
msda_fwd_d32(const T *__restrict__ value, const int64_t *__restrict__ level_hw,
             const int64_t *__restrict__ level_start, const float *__restrict__ loc,
             const float *__restrict__ attn, TO *__restrict__ out,
             const int *__restrict__ row_map, int S, int M, int Q, int L, int P, int magic,
             int iters, long long rows, const __grid_constant__ ScaFuse fz = ScaFuse{}) {
    constexpr int VEC = Vec<T>::N, LANES = 32 / VEC, G = 32 / LANES;
    static_assert(!kFused || LANES == 4, "the fused prep needs 4 lanes per row (16-bit value rows)");
    constexpr bool kHalf = std::is_same<T, bf16>::value;   // bf16: packed bf16 weights (fhfma); fp16: fp32 weights
    __shared__ __align__(16) float s_fa[kFused ? kThreads / 32 * G : 1][kFuseLP];   // attn of each row group
    __shared__ LevelTab tab;
    load_level_tab(level_hw, level_start, L, M * 32, tab);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LANES, grp = lane / LANES;
    // a warp walks `iters` consecutive groups of G rows: a CTA then covers 8 * iters * G rows, i.e.
    // a run of neighbouring queries whose image footprints overlap in L1
    for (int it = 0; it < iters; ++it) {
    long long row = (((long long)blockIdx.x * (kThreads / 32) + warp) * iters + it) * G + grp;
    if (row - grp >= rows) break;                 // warp-uniform
    bool live = row < rows;                       // dead groups still take part in the shuffles
    if (!live) row = rows - 1;
    const int m = (int)(row % M);
    int b = value_map_of(row_map, row, M, Q);
    if (b < 0) { live = false; b = 0; }           // row_map -1: unused row of a fixed-capacity list
    const int pix = M * 32;
    const int LP = L * P;
    const T *vbase = value + ((long long)b * S * M + m) * 32 + sub * VEC;
    const float2 *locp = reinterpret_cast<const float2 *>(loc) + row * LP;
    const float *attp = attn + row * LP;
    ScaRow sr;
    const int fgrp = warp * G + grp;
    if constexpr (kFused) {
        live = live && sca_row(fz, row, sr);
        float fa[8];
        const float2 st = sca_row_stats(sr, live, sub, fa);
        if (live && sub == 0) fz.stats[row] = st;
        __syncwarp();                                 // the previous row group's reads of s_fa are done
        *reinterpret_cast<float4 *>(&s_fa[fgrp][8 * sub]) = make_float4(fa[0], fa[1], fa[2], fa[3]);
        *reinterpret_cast<float4 *>(&s_fa[fgrp][8 * sub + 4]) = make_float4(fa[4], fa[5], fa[6], fa[7]);
        __syncwarp();
    }

    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;

    for (int s0 = 0; s0 < LP; s0 += LANES) {
        // ---- produce: this lane prepares sample s0 + sub of its row
        const int sm = s0 + sub;
        int enc = 0;                              // element offset of the top-left corner | dx | dy<<1
        float w00 = 0.f, w01 = 0.f, w10 = 0.f, w11 = 0.f;
        bool valid = false;
        if (sm < LP && live) {
            const int l = level_of(sm, magic);
            float2 xy;
            float a;
            if constexpr (kFused) {
                sca_loc(sr, sm, l, P, fz.Dz, tab.h[l], tab.w[l], xy.x, xy.y);
                a = s_fa[fgrp][sm];
                if (l >= fz.coarse_from) {
                    const long long ci = row * (LP - fz.coarse_from * P) + (sm - fz.coarse_from * P);
                    fz.coarse_loc[ci] = xy;
                    fz.coarse_attn[ci] = a;
                }
            } else {
                xy = __ldg(locp + sm);
                a = __ldg(attp + sm);
            }
            const Corner c = make_corner(xy.x, xy.y, tab.h[l], tab.w[l]);
            enc = (c.pidx * pix) | c.dx | (c.dy << 1);
            valid = c.valid;
            w00 = c.w00 * a; w01 = c.w01 * a; w10 = c.w10 * a; w11 = c.w11 * a;
        }
        uint32_t wa = 0, wb = 0;
        if constexpr (kHalf) { wa = pack_bf16x2(w00, w01); wb = pack_bf16x2(w10, w11); }
        const unsigned vm = __ballot_sync(0xffffffffu, valid);
        // ---- consume: every lane of the group walks the LANES samples of this round
#pragma unroll
        for (int j = 0; j < LANES; ++j) {
            if (s0 + j >= LP) break;                                   // warp-uniform
            if (!(vm & (GroupMask<LANES>::kBits << j))) continue;      // nobody needs it (uniform)
            const int src = grp * LANES + j;
            const unsigned e = (unsigned)__shfl_sync(0xffffffffu, enc, src);
            const int l = level_of(s0 + j, magic);
            const T *vl = vbase + tab.lofs[l];                        // one 64-bit add per sample
            const unsigned o00 = e & ~3u;
            const unsigned o01 = o00 + ((e & 1u) ? (unsigned)pix : 0u);
            const unsigned oy = (e & 2u) ? (unsigned)tab.rs[l] : 0u;
            Vec<T> v00, v01, v10, v11;
            v00.load(vl + o00); v01.load(vl + o01); v10.load(vl + (o00 + oy)); v11.load(vl + (o01 + oy));
            if constexpr (kHalf) {
                const uint32_t qa = __shfl_sync(0xffffffffu, wa, src);
                const uint32_t qb = __shfl_sync(0xffffffffu, wb, src);
                unsigned short h00, h01, h10, h11;
                split16(qa, h00, h01);
                split16(qb, h10, h11);
                v00.axpy_h(h00, acc); v01.axpy_h(h01, acc); v10.axpy_h(h10, acc); v11.axpy_h(h11, acc);
            } else {
                const float q00 = __shfl_sync(0xffffffffu, w00, src);
                const float q01 = __shfl_sync(0xffffffffu, w01, src);
                const float q10 = __shfl_sync(0xffffffffu, w10, src);
                const float q11 = __shfl_sync(0xffffffffu, w11, src);
                v00.axpy(q00, acc); v01.axpy(q01, acc); v10.axpy(q10, acc); v11.axpy(q11, acc);
            }
        }
    }
    if (live) store_vec<TO, VEC>(out + row * 32 + sub * VEC, acc);
    }
}

// ------------------------------------------------------------------------------------------------
// backward, head_dim == 32
// ------------------------------------------------------------------------------------------------
// kScatter = false: the "gather" half only (grad_loc, grad_attn); grad_value then comes from
// msda_bwd_splat_d32 (msda_splat.cuh), which merges the reductions of neighbouring rows in registers.
// TV = storage type of grad_value: float (default: fp32 accumulation), or __half -- every contribution is then one
// 16-byte f16x2 vector reduction per lane into a SCALED fp16 buffer (half the L2 reduction sectors; the scale is the
// power of two that puts max|grad_out| into [8, 16), gv16_scale(*gv_amax)); meant for maps where a pixel collects
// few contributions, e.g. TemporalSelfAttention's single fine level (bf16 accumulation was measured at 1.4e-2 of
// max|grad_value| there -- above the 1e-2 bar; fp16 has three more mantissa bits).
// kFused: loc / attn are recomputed from SCA's raw head output and the forward's softmax statistics (ScaFuse), and
// the row epilogue finishes d_raw (sca_prep_bwd_m8's arithmetic) for the queries that exactly one camera sees; the
// rows of the other queries store grad_loc / grad_attn for bevf_sca_prep_backward_multi as before.
template <typename T, typename TG, bool kScatter, typename TV = float, bool kFused = false>
__global__ void __launch_bounds__(kThreads)
msda_bwd_d32(const T *__restrict__ value, const int64_t *__restrict__ level_hw,
             const int64_t *__restrict__ level_start, const float *__restrict__ loc,
             const float *__restrict__ attn, const TG *__restrict__ grad_out,
             TV *__restrict__ grad_value, float *__restrict__ grad_loc,
             float *__restrict__ grad_attn, const int *__restrict__ row_map, int S, int M, int Q,
             int L, int P, int magic, int iters, long long rows, unsigned red_skip,
             const __grid_constant__ HostLevels host_levels, const unsigned *__restrict__ gv_amax = nullptr,
             __half *__restrict__ gv16 = nullptr, unsigned gv16_mask = 0u, int side_start = 0, int S_side = 0,
             const unsigned *__restrict__ fx_bounds = nullptr, int fx_bits = 0,
             const __grid_constant__ ScaFuse fz = ScaFuse{}, int rep_start = 0, int rep_k = 1) {
    // TV = long long: grad_value in 64-bit fixed point (deterministic mode): each lane adds VEC channels of every
    // corner contribution with scalar integer reductions, scaled by 2^(fx_bits - fx_exponent(fx_bounds)) (common.cuh);
    // non-finite bounds: nothing is scattered (the conversion then writes NaN)
    // Mixed accumulation (gv16 != nullptr, TV = float): the levels of gv16_mask -- the fine ones, pixels
    // [0, side_start) of every map, where a pixel collects few contributions -- are accumulated in scaled fp16 into
    // gv16 (B, side_start, M, 32); the other levels are the pixels [side_start, S) and accumulate in fp32 into
    // grad_value, which then is the SIDE buffer (B, S_side = S - side_start, M, 32).  side_start comes from the host's
    // copy of the pyramid; the level mask is re-derived from the device pyramid (below).
    // Replicated fp16 levels (mixed mode, rep_start < side_start): the pixels [rep_start, side_start) -- levels with
    // more contributions per pixel than one fp16 running sum holds accurately -- are accumulated in scaled fp16 too,
    // into rep_k copies that follow the fine pixels in every map of gv16: (B, rep_start + rep_k * S_rep, M, 32),
    // S_rep = side_start - rep_start; pair row r adds into copy r % rep_k, so each copy sums about 1 / rep_k of
    // them (adjacent pair rows are adjacent queries, which hit the same coarse pixels).  The merge sums the copies.
    // red_skip: bit l set = the grad_value contributions of level l are NOT scattered here (hybrid mode: the
    // coarse levels go through msda_bwd_splat_d32, which merges them in registers, on a second stream)
    constexpr int VEC = Vec<T>::N, LANES = 32 / VEC, G = 32 / LANES;
    constexpr bool kHalfDot = std::is_same<T, bf16>::value && std::is_same<TG, bf16>::value;
    static_assert(!kFused || (LANES == 4 && G == kFuseHeads), "the fused prep needs 16-bit value rows");
    // fused epilogue of a one-camera row: attn, grad_attn and the packed d_offsets of its 32 samples, per row group
    __shared__ float s_fa[kFused ? kThreads / 32 * G : 1][kFuseLP];
    __shared__ float s_fg[kFused ? kThreads / 32 * G : 1][kFuseLP];
    __shared__ __align__(16) uint32_t s_fo[kFused ? kThreads / 32 * G : 1][kFuseLP];
    __shared__ LevelTab tab;
    __shared__ unsigned s_skip;
    if (threadIdx.x == 0)     // levels masked for the dense path only if that kernel saw the same pyramid
        s_skip = (red_skip && host_levels.h[0] > 0 && !host_levels_match(host_levels, level_hw, level_start, L)) ? 0u : red_skip;
    __shared__ unsigned s_mask16, s_mask_rep;
    if (gv16 != nullptr && threadIdx.x == 32) {
        // which levels lie in the fp16 part is decided from the DEVICE pyramid: a level is fine if it ends at or before
        // side_start, coarse if it starts at or after it; a level that straddles the split cannot be served by either
        // buffer (the caller planned with shapes that are not the device's) and traps.  Likewise for the replicated
        // levels among the fp16 ones: those that start at or after rep_start.
        unsigned mk = 0, mr = 0;
        for (int l = 0; l < L; ++l) {
            const long long a = level_start[l], e = a + level_hw[2 * l] * level_hw[2 * l + 1];
            if (e <= side_start) {
                mk |= 1u << l;
                if (a >= rep_start) mr |= 1u << l;
                else if (e > rep_start) __trap();
            } else if (a < side_start) {
                __trap();
            }
        }
        s_mask16 = mk;
        s_mask_rep = mr;
    }
    load_level_tab(level_hw, level_start, L, M * 32, tab);
    red_skip = s_skip;
    unsigned rep_mask = 0;
    if (gv16 != nullptr) { gv16_mask = s_mask16; rep_mask = s_mask_rep; }
    const int S_rep = side_start - rep_start;
    const int S16 = rep_start + rep_k * S_rep;                             // pixels of one map of gv16
    const float gv_sc = gv_amax ? gv16_scale(__ldg(gv_amax)) : 1.f;       // scale of the fp16 accumulators
    constexpr bool kGvFx = sizeof(TV) == 8;
    double fx_sc = 0.0;
    if constexpr (kGvFx) {
        const unsigned ba = __ldg(fx_bounds), bg = __ldg(fx_bounds + 1);
        if (fx_bounds_finite(ba, bg)) fx_sc = fx_pow2(fx_bits - fx_exponent(ba, bg));
        else red_skip = ~0u;
    }

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LANES, grp = lane / LANES;
    for (int it = 0; it < iters; ++it) {
    long long row = (((long long)blockIdx.x * (kThreads / 32) + warp) * iters + it) * G + grp;
    if (row - grp >= rows) break;                 // warp-uniform
    bool live = row < rows;
    if (!live) row = rows - 1;
    const int m = (int)(row % M);
    int b = value_map_of(row_map, row, M, Q);
    if (b < 0) { live = false; b = 0; }           // row_map -1: unused row of a fixed-capacity list
    const int pix = M * 32;
    const int LP = L * P;
    const long long rep_ofs = rep_mask ? (long long)((row / M) % rep_k) * S_rep * pix : 0;   // this pair row's copy
    const long long voff = ((long long)b * S * M + m) * 32 + sub * VEC;
    const float2 *locp = reinterpret_cast<const float2 *>(loc) + row * LP;
    const float *attp = attn + row * LP;
    ScaRow sr;
    float2 st = make_float2(0.f, 0.f);
    bool single = false;                          // fused: exactly one camera sees the row's query
    const int fgrp = (threadIdx.x >> 5) * G + grp;
    if constexpr (kFused) {
        live = live && sca_row(fz, row, sr);
        if (live) {
            st = __ldg(fz.stats + row);
            // counted in pair_of: the per-item inv_count cannot tell one camera from none, and with bs > 1 it
            // follows each item's own mask while the pair list follows item 0's
            int seen = 0;
            for (int c = 0; c < fz.ncam; ++c) seen += __ldg(fz.pair_of + (long long)c * fz.Nq + sr.q) >= 0 ? 1 : 0;
            single = seen == 1;
        }
    }

    float g[VEC];                                 // this lane's slice of the grad_out row, fp32
    load_vec<TG, VEC>(grad_out + row * 32 + sub * VEC, g);
    uint4 gh = make_uint4(0, 0, 0, 0);            // the same slice as packed bf16, for the fhfma dots
    if constexpr (kHalfDot)
        gh = __ldg(reinterpret_cast<const uint4 *>(grad_out + row * 32 + sub * VEC));
    float gx[kGvFx ? VEC : 1];                    // fixed-point scatter: channels k * LANES + sub of the row
    if constexpr (kGvFx) {
#pragma unroll
        for (int k = 0; k < VEC; ++k) gx[k] = Row<TG>::load1(grad_out + row * 32 + k * LANES + sub);
    }
    // Scatter layout.  A 16 B reduction covers 4 fp32 channels and the reduction path is fastest
    // when one warp instruction fills whole 128 B lines rather than half lines.  VEC == 4: the 8 lanes of a
    // row already write its 128 B.
    // VEC == 8 (4 lanes per row, 8 rows per warp): rows are paired (grp, grp ^ 4); instruction A
    // fills the lines of the low rows -- their own lanes write channels [4 sub, +4), the partner's
    // lanes write [16 + 4 sub, +4) -- and instruction B does the same for the high rows.  Each lane
    // therefore keeps 4 grad_out channels of its own row and 4 of its partner's, and reads the
    // partner's per-sample scalars with one extra shuffle each.
    constexpr bool kGvHalf = sizeof(TV) == 2;
    static_assert(!kGvHalf || VEC == 8, "fp16 grad_value needs bf16 value rows (8 channels per lane)");
    constexpr bool kPaired = (VEC == 8) && kScatter && !kGvHalf && !kGvFx;
    const bool hi = kPaired && (grp & 4);
    const long long vrow = voff - sub * VEC;                       // element offset of the row in its map
    long long vrow_a = vrow, vrow_b = vrow;
    float gra[4], grb[4];
    if constexpr (!kPaired) {
        gra[0] = g[0]; gra[1] = g[1]; gra[2] = g[2]; gra[3] = g[3];
        grb[0] = grb[1] = grb[2] = grb[3] = 0.f;
        (void)vrow_a; (void)vrow_b;
    } else {
        const long long row_p = __shfl_xor_sync(0xffffffffu, row, 16);
        const long long vrow_p = __shfl_xor_sync(0xffffffffu, vrow, 16);
        const int chan = (hi ? 16 : 0) + 4 * sub;
        const long long row_a = hi ? row_p : row, row_b = hi ? row : row_p;
        vrow_a = (hi ? vrow_p : vrow) + chan;
        vrow_b = (hi ? vrow : vrow_p) + chan;
        if (gv16 != nullptr) {
            // the fp32 levels live in the side buffer: map stride S_side instead of S, pixel index minus side_start
            // (the fp16 levels: map stride side_start, see the scatter below)
            const int b_p = __shfl_xor_sync(0xffffffffu, b, 16);
            const int b_a = hi ? b_p : b, b_b = hi ? b : b_p;
            vrow_a -= ((long long)b_a * (S - S_side) + side_start) * pix;
            vrow_b -= ((long long)b_b * (S - S_side) + side_start) * pix;
        }
        load_vec<TG, 4>(grad_out + row_a * 32 + chan, gra);
        load_vec<TG, 4>(grad_out + row_b * 32 + chan, grb);
    }

    for (int s0 = 0; s0 < LP; s0 += LANES) {
        // ---- produce
        const int sm = s0 + sub;
        Corner c;
        c.x0 = c.y0 = 0;
        c.pidx = 0; c.dx = c.dy = 0; c.w00 = c.w01 = c.w10 = c.w11 = 0.f; c.lx = c.ly = 0.f;
        c.f00 = c.f01 = c.f10 = c.f11 = 0.f; c.valid = false;
        float a = 0.f;
        int Hm = 1, Wm = 1;
        const bool mine = sm < LP && live;
        if (mine) {
            const int l = level_of(sm, magic);
            Hm = tab.h[l]; Wm = tab.w[l];
            float2 xy;
            if constexpr (kFused) {
                sca_loc(sr, sm, l, P, fz.Dz, Hm, Wm, xy.x, xy.y);
                a = sca_attn(sr, sm, st.x, st.y);
            } else {
                xy = __ldg(locp + sm);
                a = __ldg(attp + sm);
            }
            c = make_corner(xy.x, xy.y, Hm, Wm);
        }
        const int enc = (c.pidx * pix) | c.dx | (c.dy << 1);
        const float wa00 = c.w00 * a, wa01 = c.w01 * a, wa10 = c.w10 * a, wa11 = c.w11 * a;
        const unsigned vm = __ballot_sync(0xffffffffu, c.valid);
        // d[j][k]: this lane's partial <grad_out, corner k> for sample j of the round
        float d[LANES][4];
#pragma unroll
        for (int j = 0; j < LANES; ++j) { d[j][0] = d[j][1] = d[j][2] = d[j][3] = 0.f; }
        // ---- consume
#pragma unroll
        for (int j = 0; j < LANES; ++j) {
            if (s0 + j >= LP) break;
            if (!(vm & (GroupMask<LANES>::kBits << j))) continue;
            const int src = grp * LANES + j;
            const int e = __shfl_sync(0xffffffffu, enc, src);
            const float q00 = __shfl_sync(0xffffffffu, wa00, src);
            const float q01 = __shfl_sync(0xffffffffu, wa01, src);
            const float q10 = __shfl_sync(0xffffffffu, wa10, src);
            const float q11 = __shfl_sync(0xffffffffu, wa11, src);
            const int l = level_of(s0 + j, magic);
            const long long o00 = voff + tab.lofs[l] + (long long)((unsigned)e & ~3u);
            const int ox = (e & 1) ? pix : 0, oy = (e & 2) ? tab.rs[l] : 0;
            const T *vp = value + o00;
            Vec<T> v00, v01, v10, v11;
            v00.load(vp); v01.load(vp + ox); v10.load(vp + oy); v11.load(vp + (oy + ox));
            if constexpr (kHalfDot) {
                d[j][0] = v00.dot_h(gh); d[j][1] = v01.dot_h(gh);
                d[j][2] = v10.dot_h(gh); d[j][3] = v11.dot_h(gh);
            } else {
                d[j][0] = v00.dot(g); d[j][1] = v01.dot(g); d[j][2] = v10.dot(g); d[j][3] = v11.dot(g);
            }
            // scatter w * a * g with 16 B reductions; zero-weight corners are skipped
            if constexpr (!kScatter) {
            } else if ((red_skip >> l) & 1u) {
            } else if constexpr (kGvFx) {
                // lane `sub` adds channels k * LANES + sub (gx): in each of the VEC instructions the LANES lanes of a row
                // write adjacent 8-byte words, i.e. whole 32-byte sectors
                long long *gp = reinterpret_cast<long long *>(grad_value) + (o00 - sub * VEC) + sub;
                auto redfx = [&](long long *p, float q) {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) red_add_fx(p + k * LANES, q, gx[k], fx_sc);
                };
                if (q00 != 0.f) redfx(gp, q00);
                if (q01 != 0.f) redfx(gp + ox, q01);
                if (q10 != 0.f) redfx(gp + oy, q10);
                if (q11 != 0.f) redfx(gp + oy + ox, q11);
            } else if constexpr (kGvHalf) {
                // scaled fp16 accumulation: this lane's 8 channels of the row as one 16-byte f16x2 vector reduction
                TV *gp = grad_value + o00;
                auto red8 = [&](TV *p, float q) {
                    q *= gv_sc;
                    red_add_v4_f16x2(p, pack_f16x2(q * g[0], q * g[1]), pack_f16x2(q * g[2], q * g[3]),
                                     pack_f16x2(q * g[4], q * g[5]), pack_f16x2(q * g[6], q * g[7]));
                };
                if (q00 != 0.f) red8(gp, q00);
                if (q01 != 0.f) red8(gp + ox, q01);
                if (q10 != 0.f) red8(gp + oy, q10);
                if (q11 != 0.f) red8(gp + oy + ox, q11);
            } else if constexpr (!kPaired) {
                float *gp = grad_value + o00;
                if (q00 != 0.f) red_add_v4(gp, q00 * gra[0], q00 * gra[1], q00 * gra[2], q00 * gra[3]);
                if (q01 != 0.f) red_add_v4(gp + ox, q01 * gra[0], q01 * gra[1], q01 * gra[2], q01 * gra[3]);
                if (q10 != 0.f) red_add_v4(gp + oy, q10 * gra[0], q10 * gra[1], q10 * gra[2], q10 * gra[3]);
                if (q11 != 0.f) red_add_v4(gp + oy + ox, q11 * gra[0], q11 * gra[1], q11 * gra[2], q11 * gra[3]);
            } else if ((gv16_mask >> l) & 1u) {
                // mixed mode, a fine or replicated level: scaled fp16 accumulation into gv16 (map stride S16)
                __half *gp = gv16 + (o00 - (long long)b * (S - S16) * pix + (((rep_mask >> l) & 1u) ? rep_ofs : 0));
                auto red8 = [&](__half *p, float q) {
                    q *= gv_sc;
                    red_add_v4_f16x2(p, pack_f16x2(q * g[0], q * g[1]), pack_f16x2(q * g[2], q * g[3]),
                                     pack_f16x2(q * g[4], q * g[5]), pack_f16x2(q * g[6], q * g[7]));
                };
                if (q00 != 0.f) red8(gp, q00);
                if (q01 != 0.f) red8(gp + ox, q01);
                if (q10 != 0.f) red8(gp + oy, q10);
                if (q11 != 0.f) red8(gp + oy + ox, q11);
            } else {
                const int ep = __shfl_xor_sync(0xffffffffu, e, 16);
                const float p00 = __shfl_xor_sync(0xffffffffu, q00, 16);
                const float p01 = __shfl_xor_sync(0xffffffffu, q01, 16);
                const float p10 = __shfl_xor_sync(0xffffffffu, q10, 16);
                const float p11 = __shfl_xor_sync(0xffffffffu, q11, 16);
                const int oxp = (ep & 1) ? pix : 0, oyp = (ep & 2) ? tab.rs[l] : 0;
                {   // instruction A: lines of the low rows (own scalars on low lanes, partner's on high)
                    const int ea = hi ? ep : e;
                    const int xa = hi ? oxp : ox, ya = hi ? oyp : oy;
                    const float a00 = hi ? p00 : q00, a01 = hi ? p01 : q01, a10 = hi ? p10 : q10,
                                a11 = hi ? p11 : q11;
                    float *gp = grad_value + vrow_a + tab.lofs[l] + (long long)((unsigned)ea & ~3u);
                    if (a00 != 0.f) red_add_v4(gp, a00 * gra[0], a00 * gra[1], a00 * gra[2], a00 * gra[3]);
                    if (a01 != 0.f) red_add_v4(gp + xa, a01 * gra[0], a01 * gra[1], a01 * gra[2], a01 * gra[3]);
                    if (a10 != 0.f) red_add_v4(gp + ya, a10 * gra[0], a10 * gra[1], a10 * gra[2], a10 * gra[3]);
                    if (a11 != 0.f) red_add_v4(gp + ya + xa, a11 * gra[0], a11 * gra[1], a11 * gra[2], a11 * gra[3]);
                }
                {   // instruction B: lines of the high rows
                    const int eb = hi ? e : ep;
                    const int xb = hi ? ox : oxp, yb = hi ? oy : oyp;
                    const float b00 = hi ? q00 : p00, b01 = hi ? q01 : p01, b10 = hi ? q10 : p10,
                                b11 = hi ? q11 : p11;
                    float *gp = grad_value + vrow_b + tab.lofs[l] + (long long)((unsigned)eb & ~3u);
                    if (b00 != 0.f) red_add_v4(gp, b00 * grb[0], b00 * grb[1], b00 * grb[2], b00 * grb[3]);
                    if (b01 != 0.f) red_add_v4(gp + xb, b01 * grb[0], b01 * grb[1], b01 * grb[2], b01 * grb[3]);
                    if (b10 != 0.f) red_add_v4(gp + yb, b10 * grb[0], b10 * grb[1], b10 * grb[2], b10 * grb[3]);
                    if (b11 != 0.f) red_add_v4(gp + yb + xb, b11 * grb[0], b11 * grb[1], b11 * grb[2], b11 * grb[3]);
                }
            }
        }
        // ---- reduce-scatter the dots over the group: lane `sub` ends with the totals of sample
        //      s0 + sub (the one whose scalars it holds).  log2(LANES) halving steps.
#pragma unroll
        for (int step = LANES / 2; step > 0; step >>= 1) {
            const bool upper = (sub & step) != 0;
#pragma unroll
            for (int j = 0; j < step; ++j) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    // keep the half of the samples whose index has this bit equal to mine
                    const float keep = upper ? d[j + step][k] : d[j][k];
                    const float send = upper ? d[j][k] : d[j + step][k];
                    d[j][k] = keep + __shfl_xor_sync(0xffffffffu, send, step);
                }
            }
        }
        if (mine) {
            const float hx = 1.f - c.lx, hy = 1.f - c.ly;
            const float d00 = c.f00 * d[0][0], d01 = c.f01 * d[0][1], d10 = c.f10 * d[0][2],
                        d11 = c.f11 * d[0][3];
            const float ga = hy * (hx * d00 + c.lx * d01) + c.ly * (hx * d10 + c.lx * d11);
            const float gx = a * (hy * (d01 - d00) + c.ly * (d11 - d10));
            const float gy = a * (hx * (d10 - d00) + c.lx * (d11 - d01));
            const long long si = row * LP + sm;
            const float glx = (float)Wm * gx, gly = (float)Hm * gy;
            if (!kFused || !single) {
                grad_attn[si] = ga;
                reinterpret_cast<float2 *>(grad_loc)[si] = make_float2(glx, gly);
            } else {
                // sca_prep_bwd_m8 with one camera: its sums start at 0 (0 + x only differs from x for x = -0)
                s_fa[fgrp][sm] = a;
                s_fg[fgrp][sm] = 0.f + ga;
                s_fo[fgrp][sm] = pack_bf16x2(__fdiv_rn(0.f + glx, (float)Wm), __fdiv_rn(0.f + gly, (float)Hm));
            }
        }
    }
    if constexpr (kFused) {
        // d_raw of a one-camera row, in the prep kernel's partition: lane `sub` owns samples [8 sub, 8 sub + 8)
        __syncwarp();
        float fa[8], fg[8], dot = 0.f;
        const bool fin = live && single;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            fa[i] = fin ? s_fa[fgrp][8 * sub + i] : 0.f;
            fg[i] = fin ? s_fg[fgrp][8 * sub + i] : 0.f;
            dot += fa[i] * fg[i];
        }
        dot = quad_sum(dot);
        if (fin) {
            bf16 *dr = fz.d_raw + sr.raw_row * (kFuseHeads * kFuseLP * 3);
#pragma unroll
            for (int i = 0; i < 8; ++i) fg[i] = fa[i] * (fg[i] - dot);
            *reinterpret_cast<uint4 *>(dr + kFuseHeads * kFuseLP * 2 + m * kFuseLP + 8 * sub) =
                make_uint4(pack_bf16x2(fg[0], fg[1]), pack_bf16x2(fg[2], fg[3]), pack_bf16x2(fg[4], fg[5]),
                           pack_bf16x2(fg[6], fg[7]));
            const uint4 *so = reinterpret_cast<const uint4 *>(&s_fo[fgrp][8 * sub]);
            uint4 *dof = reinterpret_cast<uint4 *>(dr + m * kFuseLP * 2 + 16 * sub);
            dof[0] = so[0];
            dof[1] = so[1];
        }
        __syncwarp();
    }
    }
}


}  // namespace bevf
#include "msda_splat.cuh"
namespace bevf {

// ------------------------------------------------------------------------------------------------
// any head_dim: one warp per (query, head) row, lanes stride over channels
// ------------------------------------------------------------------------------------------------
template <typename T, typename TO>
__global__ void __launch_bounds__(kThreads)
msda_fwd_generic(const T *__restrict__ value, const int64_t *__restrict__ level_hw,
                 const int64_t *__restrict__ level_start, const float *__restrict__ loc,
                 const float *__restrict__ attn, TO *__restrict__ out,
                 const int *__restrict__ row_map, int S, int M, int D, int Q, int L, int P,
                 long long rows) {
    __shared__ int s_h[kMaxLevels], s_w[kMaxLevels], s_start[kMaxLevels];
    load_levels(level_hw, level_start, L, s_h, s_w, s_start);
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int m = (int)(row % M);
    const int b = value_map_of(row_map, row, M, Q);
    if (b < 0) return;                            // unused row (whole warp)
    const long long pix = (long long)M * D;
    for (int c0 = lane; c0 < D; c0 += 32) {
        float acc = 0.f;
        for (int l = 0; l < L; ++l) {
            const int H = s_h[l], W = s_w[l];
            const T *vl = value + ((long long)b * S + s_start[l]) * pix + (long long)m * D + c0;
            for (int p = 0; p < P; ++p) {
                const long long si = row * L * P + l * P + p;
                const Corner c = make_corner(loc[2 * si], loc[2 * si + 1], H, W);
                const float a = attn[si];
                const T *p00 = vl + c.pidx * pix;
                const long long ox = c.dx ? pix : 0, oy = c.dy ? W * pix : 0;
                acc += a * (c.w00 * Row<T>::load1(p00) + c.w01 * Row<T>::load1(p00 + ox) +
                            c.w10 * Row<T>::load1(p00 + oy) + c.w11 * Row<T>::load1(p00 + oy + ox));
            }
        }
        Row<TO>::store1(out + row * D + c0, acc);
    }
}

// TV = long long: grad_value in 64-bit fixed point, as in msda_bwd_d32
template <typename T, typename TG, typename TV = float>
__global__ void __launch_bounds__(kThreads)
msda_bwd_generic(const T *__restrict__ value, const int64_t *__restrict__ level_hw,
                 const int64_t *__restrict__ level_start, const float *__restrict__ loc,
                 const float *__restrict__ attn, const TG *__restrict__ grad_out,
                 TV *__restrict__ grad_value, float *__restrict__ grad_loc,
                 float *__restrict__ grad_attn, const int *__restrict__ row_map, int S, int M,
                 int D, int Q, int L, int P, long long rows,
                 const unsigned *__restrict__ fx_bounds = nullptr, int fx_bits = 0) {
    __shared__ int s_h[kMaxLevels], s_w[kMaxLevels], s_start[kMaxLevels];
    load_levels(level_hw, level_start, L, s_h, s_w, s_start);
    constexpr bool kGvFx = sizeof(TV) == 8;
    double fx_sc = 0.0;
    bool scatter = true;
    if constexpr (kGvFx) {
        const unsigned ba = __ldg(fx_bounds), bg = __ldg(fx_bounds + 1);
        scatter = fx_bounds_finite(ba, bg);
        if (scatter) fx_sc = fx_pow2(fx_bits - fx_exponent(ba, bg));
    }
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    if (row >= rows) return;   // whole warp leaves together
    const int m = (int)(row % M);
    const int b = value_map_of(row_map, row, M, Q);
    if (b < 0) return;         // unused row (whole warp)
    const long long pix = (long long)M * D;
    for (int l = 0; l < L; ++l) {
        const int H = s_h[l], W = s_w[l];
        const long long lbase = ((long long)b * S + s_start[l]) * pix + (long long)m * D;
        for (int p = 0; p < P; ++p) {
            const long long si = row * L * P + l * P + p;
            const Corner c = make_corner(loc[2 * si], loc[2 * si + 1], H, W);
            const long long i00 = lbase + c.pidx * pix;
            const long long ox = c.dx ? pix : 0, oy = c.dy ? W * pix : 0;
            const long long i01 = i00 + ox, i10 = i00 + oy, i11 = i00 + oy + ox;
            const float a = attn[si];
            const float hx = 1.f - c.lx, hy = 1.f - c.ly;
            float ga = 0.f, gx = 0.f, gy = 0.f;
            for (int c0 = lane; c0 < D; c0 += 32) {
                const float gc = Row<TG>::load1(grad_out + row * D + c0), t = gc * a;
                const float v00 = c.f00 * Row<T>::load1(value + i00 + c0);
                const float v01 = c.f01 * Row<T>::load1(value + i01 + c0);
                const float v10 = c.f10 * Row<T>::load1(value + i10 + c0);
                const float v11 = c.f11 * Row<T>::load1(value + i11 + c0);
                if constexpr (kGvFx) {
                    if (scatter) {
                        if (c.w00 != 0.f) red_add_fx(grad_value + i00 + c0, c.w00 * a, gc, fx_sc);
                        if (c.w01 != 0.f) red_add_fx(grad_value + i01 + c0, c.w01 * a, gc, fx_sc);
                        if (c.w10 != 0.f) red_add_fx(grad_value + i10 + c0, c.w10 * a, gc, fx_sc);
                        if (c.w11 != 0.f) red_add_fx(grad_value + i11 + c0, c.w11 * a, gc, fx_sc);
                    }
                } else {
                    if (c.w00 != 0.f) atomicAdd(grad_value + i00 + c0, c.w00 * t);
                    if (c.w01 != 0.f) atomicAdd(grad_value + i01 + c0, c.w01 * t);
                    if (c.w10 != 0.f) atomicAdd(grad_value + i10 + c0, c.w10 * t);
                    if (c.w11 != 0.f) atomicAdd(grad_value + i11 + c0, c.w11 * t);
                }
                ga += gc * (hy * (hx * v00 + c.lx * v01) + c.ly * (hx * v10 + c.lx * v11));
                gx += t * (hy * (v01 - v00) + c.ly * (v11 - v10));
                gy += t * (hx * (v10 - v00) + c.lx * (v11 - v01));
            }
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) {
                ga += __shfl_xor_sync(0xffffffffu, ga, s);
                gx += __shfl_xor_sync(0xffffffffu, gx, s);
                gy += __shfl_xor_sync(0xffffffffu, gy, s);
            }
            if (lane == 0) {
                grad_attn[si] = ga;
                grad_loc[2 * si] = (float)W * gx;
                grad_loc[2 * si + 1] = (float)H * gy;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
// The head_dim 32 kernels take one group of G rows per warp (iters = 1): more loses parallelism for no L1 gain.
static unsigned grid_d32(long long rows, int G) {
    const long long per_block = (long long)(kThreads / 32) * G;
    return (unsigned)((rows + per_block - 1) / per_block);
}

static int check_dims(const char *who, int B, int S, int M, int D, int Q, int L, int P) {
    if (B < 0 || S < 0 || M <= 0 || D <= 0 || Q < 0 || L <= 0 || P <= 0)
        return fail("%s: negative or zero dimension", who);
    if (L > kMaxLevels) return fail("%s: at most 16 levels are supported (got %lld)", who, L);
    if ((long long)S * M * D >= (1ll << 31))
        return fail("%s: one batch item of value exceeds 2^31 elements", who);
    if ((long long)L * P * P >= 65536) return fail("%s: num_levels * num_points^2 must be < 65536", who);
    return 0;    // (level sizes are device data: H, W < 32768 is the caller's contract, see the header)
}

template <typename T, typename TO>
static int launch_fwd(const char *who, const void *value, const int64_t *hw, const int64_t *ls,
                      const float *loc, const float *attn, void *out, const int *row_map, int S,
                      int M, int D, int Q, int L, int P, long long rows, cudaStream_t st,
                      const ScaFuse *fz = nullptr) {
    if (D == 32) {
        const unsigned grid = grid_d32(rows, Vec<T>::N);
        if (fz) {
            if constexpr (std::is_same<T, bf16>::value && std::is_same<TO, bf16>::value)
                msda_fwd_d32<T, TO, true><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, nullptr, nullptr, (TO *)out,
                                                                     row_map, S, M, Q, L, P, (65536 + P - 1) / P, 1,
                                                                     rows, *fz);
            else
                return fail("%s: the fused prep needs bf16 value and output", who);
        } else {
            msda_fwd_d32<T, TO><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn, (TO *)out,
                                                           row_map, S, M, Q, L, P, (65536 + P - 1) / P, 1,
                                                           rows);
        }
    } else if (fz) {
        return fail("%s: the fused prep needs head_dim 32", who);
    } else {
        const unsigned grid = (unsigned)((rows + kThreads / 32 - 1) / (kThreads / 32));
        msda_fwd_generic<T, TO><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn,
                                                           (TO *)out, row_map, S, M, D, Q, L, P, rows);
    }
    return check_launch(who);
}

// Backward mode.  0 = one kernel (default): every corner contribution is its own 16 B-vector L2 reduction.
// 1 = split: gather half (grad_loc / grad_attn) + the register-merging splat kernel of msda_splat.cuh
// (grad_value).  The split removes 82 % of the L2 reductions but costs 2.3x the instructions; it is
// not the default and stays selectable for A/B runs -- environment
// BEVF_MSDA_BWD=split or bevf_msda_set_backward_mode(1).
static std::atomic<int> g_bwd_mode{-1};
static int bwd_split_enabled() {
    int v = g_bwd_mode.load(std::memory_order_relaxed);
    if (v < 0) {
        const char *e = getenv("BEVF_MSDA_BWD");
        v = (e && e[0] == 's') ? 1 : 0;               // (mode 2 needs its stream: only through the setter)
        g_bwd_mode.store(v, std::memory_order_relaxed);
    }
    return v;
}
static unsigned splat_direct_mask() {
    static long v = -1;
    if (v < 0) {
        const char *e = getenv("BEVF_SPLAT_DIRECT");
        v = e ? strtol(e, nullptr, 0) : 0;
    }
    return (unsigned)v;
}

int dense_coarse_backward(const char *who, const int64_t *hw_dev, const int64_t *ls_dev, const int32_t *hw_host,
                          const float *loc, const float *attn, const void *grad_out, float *grad_value,
                          const int32_t *map_range, int NB, int S, int M, int L, int P, cudaStream_t st,
                          unsigned *handled, HostLevels *host_levels, int first_level, unsigned need_mask,
                          int gv_S, int gv_base, int loc_level0);                      // msda_dense.cu

// second stream + events for the hybrid backward (created by bevf_msda_set_backward_mode(2), i.e. outside any
// stream capture; the fork / join below is capturable)
static cudaStream_t g_side_stream = nullptr;
constexpr int kSideEvents = 64;
static cudaEvent_t g_side_events[kSideEvents];
static std::atomic<unsigned> g_side_ev_next{0};

template <typename TG, int kM>
static int launch_splat_km(const char *who, const float *loc, const float *attn, const void *go, float *gv,
                           const int *row_map, const int *order, const int64_t *hw, const int64_t *ls,
                           int S, int M, int Q, int L, int P, long long pairs, unsigned level_mask,
                           cudaStream_t st) {
    static bool attr_done = false;                     // per instantiation
    if (!attr_done) {
        if (cudaFuncSetAttribute(msda_bwd_splat_d32<TG, kM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)splat_smem_bytes(kSplatMaxHeads, sizeof(TG))) != cudaSuccess) {
            cudaGetLastError();
            return fail("%s: cannot reserve shared memory for the splat kernel", who);
        }
        attr_done = true;
    }
    const unsigned grid = (unsigned)((pairs + kSplatG - 1) / kSplatG);
    msda_bwd_splat_d32<TG, kM><<<grid, 32 * M, splat_smem_bytes(M, sizeof(TG)), st>>>(
        loc, attn, (const TG *)go, gv, row_map, order, hw, ls, S, M, Q, L, P, pairs, splat_direct_mask(),
        level_mask);
    return check_launch(who);
}

template <typename TG>
static int launch_splat(const char *who, const float *loc, const float *attn, const void *go, float *gv,
                        const int *row_map, const int *order, const int64_t *hw, const int64_t *ls,
                        int S, int M, int Q, int L, int P, long long pairs, unsigned level_mask,
                        cudaStream_t st) {
    if constexpr (std::is_same<TG, __half>::value) {
        return fail("%s: the splat kernel takes fp32 or bf16 grad_out", who);
    } else {
        // the head count of every BEVFormer config is 8: that instance addresses the window with immediates
        if (M == 8)
            return launch_splat_km<TG, 8>(who, loc, attn, go, gv, row_map, order, hw, ls, S, M, Q, L, P, pairs,
                                          level_mask, st);
        return launch_splat_km<TG, 0>(who, loc, attn, go, gv, row_map, order, hw, ls, S, M, Q, L, P, pairs,
                                      level_mask, st);
    }
}

struct MixedGv {               // scaled-fp16 / mixed accumulation of grad_value (see msda_bwd_d32)
    const unsigned *amax = nullptr;          // float bits of max|grad_out| (bevf_abs_max)
    __half *gv16 = nullptr;                  // mixed mode: the fine and replicated levels' buffer
    unsigned mask = 0;
    int side_start = 0, S_side = 0;
    int rep_start = 0, rep_k = 1;            // replicated levels: pixels [rep_start, side_start), rep_k copies
};

struct FxGv {                  // 64-bit fixed-point grad_value (deterministic mode)
    const unsigned *bounds = nullptr;        // max|attn|, max|grad_out| bits (gvfx.cu: fx_bounds)
    int frac_bits = 0;
};

template <typename T, typename TG>
static int launch_bwd(const char *who, const void *value, const int64_t *hw, const int64_t *ls,
                      const float *loc, const float *attn, const void *go, float *gv, float *gl,
                      float *ga, const int *row_map, const int *order, int S, int M, int D, int Q,
                      int L, int P, long long rows, cudaStream_t st, unsigned done_levels = 0,
                      const HostLevels *host_levels = nullptr, bool gv_f16 = false,
                      const MixedGv *mixed = nullptr, const FxGv *fx = nullptr, const ScaFuse *fz = nullptr) {
    if (fz && (fx || gv_f16 || !mixed || !mixed->gv16))
        return fail("%s: the fused prep runs with mixed grad_value accumulation only", who);
    HostLevels hl;
    if (host_levels) hl = *host_levels; else memset(&hl, 0, sizeof(hl));
    if (fx) {
        // fixed-point grad_value: always the one-kernel backward (the split / hybrid / dense modes sum in fp32)
        long long *gfx = reinterpret_cast<long long *>(gv);
        if (D == 32) {
            const unsigned grid = grid_d32(rows, Vec<T>::N);
            msda_bwd_d32<T, TG, true, long long><<<grid, kThreads, 0, st>>>(
                (const T *)value, hw, ls, loc, attn, (const TG *)go, gfx, gl, ga, row_map, S, M, Q, L, P,
                (65536 + P - 1) / P, 1, rows, 0u, hl, nullptr, nullptr, 0u, 0, 0, fx->bounds, fx->frac_bits);
        } else {
            const unsigned grid = (unsigned)((rows + kThreads / 32 - 1) / (kThreads / 32));
            msda_bwd_generic<T, TG, long long><<<grid, kThreads, 0, st>>>(
                (const T *)value, hw, ls, loc, attn, (const TG *)go, gfx, gl, ga, row_map, S, M, D, Q, L, P, rows,
                fx->bounds, fx->frac_bits);
        }
        return check_launch(who);
    }
    if (gv_f16) {
        // grad_value stored and accumulated in scaled fp16: bf16 value rows, head_dim 32, the one-kernel backward only
        if constexpr (std::is_same<T, bf16>::value) {
            if (D != 32) return fail("%s: fp16 grad_value needs head_dim 32", who);
            const unsigned grid = grid_d32(rows, Vec<T>::N);
            msda_bwd_d32<T, TG, true, __half><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn, (const TG *)go,
                                                                       reinterpret_cast<__half *>(gv), gl, ga, row_map, S, M,
                                                                       Q, L, P, (65536 + P - 1) / P, 1, rows, 0u, hl,
                                                                       mixed ? mixed->amax : nullptr);
            return check_launch(who);
        } else {
            return fail("%s: fp16 grad_value needs a bf16 value tensor", who);
        }
    }
    if (mixed && mixed->gv16) {
        if constexpr (std::is_same<T, bf16>::value) {
            if (D != 32) return fail("%s: mixed accumulation needs head_dim 32", who);
            const unsigned grid = grid_d32(rows, Vec<T>::N);
            if (fz) {
                if constexpr (std::is_same<TG, bf16>::value)
                    msda_bwd_d32<T, TG, true, float, true><<<grid, kThreads, 0, st>>>(
                        (const T *)value, hw, ls, nullptr, nullptr, (const TG *)go, gv, gl, ga, row_map, S, M, Q, L, P,
                        (65536 + P - 1) / P, 1, rows, done_levels, hl, mixed->amax, mixed->gv16, mixed->mask,
                        mixed->side_start, mixed->S_side, nullptr, 0, *fz, mixed->rep_start, mixed->rep_k);
                else
                    return fail("%s: the fused prep needs a bf16 grad_out", who);
                return check_launch(who);
            }
            msda_bwd_d32<T, TG, true><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn, (const TG *)go, gv, gl, ga,
                                                               row_map, S, M, Q, L, P, (65536 + P - 1) / P, 1, rows,
                                                               done_levels, hl, mixed->amax, mixed->gv16, mixed->mask, mixed->side_start,
                                                               mixed->S_side, nullptr, 0, ScaFuse{}, mixed->rep_start,
                                                               mixed->rep_k);
            return check_launch(who);
        } else {
            return fail("%s: mixed accumulation needs a bf16 value tensor", who);
        }
    }
    if (D == 32) {
        const unsigned grid = grid_d32(rows, Vec<T>::N);
        const int mode = done_levels ? 0 : bwd_split_enabled();
        if (mode != 0 && std::is_same<T, __half>::value)
            return fail("%s: the split / hybrid backward modes take fp32 or bf16 only (fp16 needs mode 0)", who);
        const bool can_split = M <= kSplatMaxHeads && S * (long long)M * 32 < (1ll << 31);
        if (mode == 1 && can_split) {
            if (int e = launch_splat<TG>(who, loc, attn, go, gv, row_map, order, hw, ls, S, M, Q, L, P,
                                         rows / M, 0xffffffffu, st))
                return e;
            msda_bwd_d32<T, TG, false><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn,
                                                                  (const TG *)go, gv, gl, ga, row_map, S, M,
                                                                  Q, L, P, (65536 + P - 1) / P, 1, rows, 0u, hl);
        } else if (mode == 2 && can_split && L >= 2 && g_side_stream) {
            // hybrid: the coarse half of the pyramid (most collisions, 47 % of the reduction bytes at base)
            // through the register-merging splat on the second stream, everything else in the one-kernel
            // backward on the caller's stream; the two write disjoint levels of grad_value
            unsigned coarse = 0;
            for (int l = L / 2; l < L; ++l) coarse |= 1u << l;
            cudaEvent_t fork = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            cudaEvent_t join = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            cudaEventRecord(fork, st);
            cudaStreamWaitEvent(g_side_stream, fork, 0);
            if (int e = launch_splat<TG>(who, loc, attn, go, gv, row_map, order, hw, ls, S, M, Q, L, P,
                                         rows / M, coarse, g_side_stream))
                return e;
            cudaEventRecord(join, g_side_stream);
            msda_bwd_d32<T, TG, true><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn,
                                                                 (const TG *)go, gv, gl, ga, row_map, S, M,
                                                                 Q, L, P, (65536 + P - 1) / P, 1, rows, coarse, hl);
            cudaStreamWaitEvent(st, join, 0);
        } else {
            msda_bwd_d32<T, TG, true><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn,
                                                                 (const TG *)go, gv, gl, ga, row_map, S, M,
                                                                 Q, L, P, (65536 + P - 1) / P, 1, rows, done_levels, hl);
        }
    } else {
        const unsigned grid = (unsigned)((rows + kThreads / 32 - 1) / (kThreads / 32));
        msda_bwd_generic<T, TG><<<grid, kThreads, 0, st>>>((const T *)value, hw, ls, loc, attn,
                                                           (const TG *)go, gv, gl, ga, row_map, S, M,
                                                           D, Q, L, P, rows);
    }
    return check_launch(who);
}

static int msda_forward_impl(const char *who, const void *value, int value_dtype,
                             const int64_t *level_hw, const int64_t *level_start, const float *loc,
                             const float *attn, void *out, int out_dtype, const int *row_map, int B,
                             int S, int M, int D, int Q, int L, int P, void *stream,
                             const ScaFuse *fz = nullptr) {
    if (int e = check_dims(who, B, S, M, D, Q, L, P)) return e;
    const long long rows = (row_map ? 1ll : (long long)B) * Q * M;
    if (rows == 0) return 0;
    if (!value || !level_hw || !level_start || ((!loc || !attn) && !fz) || !out)
        return fail("%s: null pointer argument", who);
    if (!aligned16(value) || !aligned16(loc) || !aligned16(attn) || !aligned16(out))
        return fail("%s: device pointers must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (fz) {
        if (value_dtype != BEVF_DTYPE_BF16 || out_dtype != BEVF_DTYPE_BF16)
            return fail("%s: the fused prep needs bf16 value and output", who);
        return launch_fwd<bf16, bf16>(who, value, level_hw, level_start, nullptr, nullptr, out, row_map, S, M, D, Q, L, P,
                                      rows, st, fz);
    }
    if (value_dtype == BEVF_DTYPE_F16) {
        // fp16 value: fp16 or fp32 output
        if (out_dtype == BEVF_DTYPE_F16) return launch_fwd<__half, __half>(who, value, level_hw, level_start, loc, attn, out, row_map, S, M, D, Q, L, P, rows, st);
        if (out_dtype == BEVF_DTYPE_F32) return launch_fwd<__half, float>(who, value, level_hw, level_start, loc, attn, out, row_map, S, M, D, Q, L, P, rows, st);
        return fail("%s: fp16 value needs an fp16 or fp32 output", who);
    }
    const bool vb = value_dtype == BEVF_DTYPE_BF16, ob = out_dtype == BEVF_DTYPE_BF16;
    if ((value_dtype != BEVF_DTYPE_F32 && !vb) || (out_dtype != BEVF_DTYPE_F32 && !ob))
        return fail("%s: unsupported dtype code", who);
    if (!vb && !ob) return launch_fwd<float, float>(who, value, level_hw, level_start, loc, attn, out, row_map, S, M, D, Q, L, P, rows, st);
    if (vb && ob) return launch_fwd<bf16, bf16>(who, value, level_hw, level_start, loc, attn, out, row_map, S, M, D, Q, L, P, rows, st);
    if (vb && !ob) return launch_fwd<bf16, float>(who, value, level_hw, level_start, loc, attn, out, row_map, S, M, D, Q, L, P, rows, st);
    return fail("%s: fp32 value with bf16 output is not supported", who);
}

static int msda_backward_impl(const char *who, const void *value, int value_dtype,
                              const int64_t *level_hw, const int64_t *level_start, const float *loc,
                              const float *attn, const void *grad_out, int grad_out_dtype,
                              float *grad_value, float *grad_loc, float *grad_attn,
                              const int *row_map, const int *order, int B, int S, int M, int D, int Q,
                              int L, int P, void *stream, unsigned done_levels = 0,
                              const HostLevels *host_levels = nullptr, bool gv_f16 = false,
                              const MixedGv *mixed = nullptr, const FxGv *fx = nullptr,
                              const ScaFuse *fz = nullptr) {
    if (int e = check_dims(who, B, S, M, D, Q, L, P)) return e;
    const long long rows = (row_map ? 1ll : (long long)B) * Q * M;
    if (rows == 0) return 0;
    if (!value || !level_hw || !level_start || ((!loc || !attn) && !fz) || !grad_out || !grad_value ||
        !grad_loc || !grad_attn)
        return fail("%s: null pointer argument", who);
    if (!aligned16(value) || !aligned16(loc) || !aligned16(attn) || !aligned16(grad_out) ||
        !aligned16(grad_value) || !aligned16(grad_loc) || !aligned16(grad_attn))
        return fail("%s: device pointers must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (fz) {
        if (value_dtype != BEVF_DTYPE_BF16 || grad_out_dtype != BEVF_DTYPE_BF16)
            return fail("%s: the fused prep needs bf16 value and grad_out", who);
        return launch_bwd<bf16, bf16>(who, value, level_hw, level_start, nullptr, nullptr, grad_out, grad_value, grad_loc,
                                      grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels,
                                      gv_f16, mixed, fx, fz);
    }
    if (value_dtype == BEVF_DTYPE_F16) {
        // fp16 value: fp16 or fp32 grad_out; grad_value stays fp32 (or fixed point)
        if (grad_out_dtype == BEVF_DTYPE_F16) return launch_bwd<__half, __half>(who, value, level_hw, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels, gv_f16, mixed, fx);
        if (grad_out_dtype == BEVF_DTYPE_F32) return launch_bwd<__half, float>(who, value, level_hw, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels, gv_f16, mixed, fx);
        return fail("%s: fp16 value needs an fp16 or fp32 grad_out", who);
    }
    const bool vb = value_dtype == BEVF_DTYPE_BF16, gb = grad_out_dtype == BEVF_DTYPE_BF16;
    if ((value_dtype != BEVF_DTYPE_F32 && !vb) || (grad_out_dtype != BEVF_DTYPE_F32 && !gb))
        return fail("%s: unsupported dtype code", who);
    if (!vb && !gb) return launch_bwd<float, float>(who, value, level_hw, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels, gv_f16, mixed, fx);
    if (vb && gb) return launch_bwd<bf16, bf16>(who, value, level_hw, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels, gv_f16, mixed, fx);
    if (vb && !gb) return launch_bwd<bf16, float>(who, value, level_hw, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn, row_map, order, S, M, D, Q, L, P, rows, st, done_levels, host_levels, gv_f16, mixed, fx);
    return fail("%s: fp32 value with bf16 grad_out is not supported", who);
}

}  // namespace bevf

using namespace bevf;

extern "C" int bevf_msda_forward(const void *value, int value_dtype, const int64_t *level_hw,
                                 const int64_t *level_start, const float *loc, const float *attn,
                                 void *out, int out_dtype, int B, int S, int M, int D, int Q, int L,
                                 int P, void *stream) {
    return msda_forward_impl("bevf_msda_forward", value, value_dtype, level_hw, level_start, loc,
                             attn, out, out_dtype, nullptr, B, S, M, D, Q, L, P, stream);
}

extern "C" int bevf_msda_backward(const void *value, int value_dtype, const int64_t *level_hw,
                                  const int64_t *level_start, const float *loc, const float *attn,
                                  const void *grad_out, int grad_out_dtype, float *grad_value,
                                  float *grad_loc, float *grad_attn, int B, int S, int M, int D,
                                  int Q, int L, int P, void *stream) {
    return msda_backward_impl("bevf_msda_backward", value, value_dtype, level_hw, level_start, loc,
                              attn, grad_out, grad_out_dtype, grad_value, grad_loc, grad_attn,
                              nullptr, nullptr, B, S, M, D, Q, L, P, stream);
}

extern "C" int bevf_msda_rows_forward(const void *value, int value_dtype, const int64_t *level_hw,
                                      const int64_t *level_start, const float *loc,
                                      const float *attn, void *out, int out_dtype,
                                      const int32_t *row_map, int B, int S, int M, int D, int R,
                                      int L, int P, void *stream) {
    if (!row_map && R > 0) return fail("%s: row_map is null", "bevf_msda_rows_forward");
    return msda_forward_impl("bevf_msda_rows_forward", value, value_dtype, level_hw, level_start,
                             loc, attn, out, out_dtype, row_map, B, S, M, D, R, L, P, stream);
}

extern "C" int bevf_msda_rows_backward(const void *value, int value_dtype, const int64_t *level_hw,
                                       const int64_t *level_start, const float *loc,
                                       const float *attn, const void *grad_out, int grad_out_dtype,
                                       float *grad_value, float *grad_loc, float *grad_attn,
                                       const int32_t *row_map, int B, int S, int M, int D, int R,
                                       int L, int P, void *stream) {
    if (!row_map && R > 0) return fail("%s: row_map is null", "bevf_msda_rows_backward");
    return msda_backward_impl("bevf_msda_rows_backward", value, value_dtype, level_hw, level_start,
                              loc, attn, grad_out, grad_out_dtype, grad_value, grad_loc, grad_attn,
                              row_map, nullptr, B, S, M, D, R, L, P, stream);
}

// grad_value of the coarse levels through the dense tensor-core kernel (msda_dense.cu), everything else
// (grad_loc, grad_attn, grad_value of the fine levels) through the one-kernel backward with those levels masked.
// mode 1: both on the caller's stream; mode 2: the dense kernel on the library's second stream (fork / join
// with events, capturable) -- it works out of shared memory and registers while the other is bound by L2 reductions.
// Setting -1 = the library default: kDenseDefault for the mixed-accumulation backward (its coarse levels have
// hundreds of contributions per pixel, see bevf_msda_rows_backward_mixed_dense), off for
// bevf_msda_rows_backward_dense (fp32 reductions on every other level; opt-in).
constexpr int kDenseDefault = 2;
static std::atomic<int> g_dense_mode{-2};                   // -2: not read from the environment yet
static int dense_setting() {
    int v = g_dense_mode.load(std::memory_order_relaxed);
    if (v == -2) {
        const char *e = getenv("BEVF_MSDA_DENSE");
        v = -1;
        if (e && e[0]) {
            v = atoi(e);
            if (v < 0 || v > 1) v = 1;                  // (mode 2 needs its stream: only through the setter)
        }
        g_dense_mode.store(v, std::memory_order_relaxed);
    }
    return v;
}
static int mixed_dense_mode() {
    const int v = dense_setting();
    return v < 0 ? kDenseDefault : v;
}
static int ensure_side_stream(const char *who) {
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (g_side_stream) return 0;
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) {
        cudaGetLastError();
        return fail("%s: cannot create the second stream", who);
    }
    for (int i = 0; i < kSideEvents; ++i) cudaEventCreateWithFlags(&g_side_events[i], cudaEventDisableTiming);
    g_side_stream = s;
    return 0;
}

extern "C" int bevf_msda_set_dense_backward(int mode) {
    if (mode < -1 || mode > 2)
        return fail("%s: mode must be -1 (library default), 0 (off), 1 (same stream) or 2 (second stream)",
                    "bevf_msda_set_dense_backward");
    if (mode == 2)
        if (int e = ensure_side_stream("bevf_msda_set_dense_backward")) return e;
    g_dense_mode.store(mode, std::memory_order_relaxed);
    return 0;
}

extern "C" int bevf_msda_get_dense_backward(void) { return mixed_dense_mode(); }

extern "C" int bevf_msda_rows_backward_dense(const void *value, int value_dtype, const int64_t *level_hw,
                                             const int64_t *level_start, const int32_t *level_hw_host,
                                             const float *loc, const float *attn, const void *grad_out,
                                             int grad_out_dtype, float *grad_value, float *grad_loc,
                                             float *grad_attn, const int32_t *row_map, const int32_t *map_range,
                                             int B, int S, int M, int D, int R, int L, int P, void *stream) {
    const char *who = "bevf_msda_rows_backward_dense";
    if (!row_map && R > 0) return fail("%s: row_map is null", who);
    if (int e = check_dims(who, B, S, M, D, R, L, P)) return e;
    if (R == 0) return 0;
    if (!level_hw_host || !map_range || !level_hw || !level_start || !loc || !attn || !grad_out || !grad_value)
        return fail("%s: null pointer argument", who);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned handled = 0;
    HostLevels hl;
    memset(&hl, 0, sizeof(hl));
    const int mode = dense_setting() < 0 ? 0 : dense_setting();
    cudaEvent_t join = nullptr;
    if (value_dtype == BEVF_DTYPE_F16 || grad_out_dtype == BEVF_DTYPE_F16)
        return fail("%s: fp32 or bf16 only (fp16 runs on bevf_msda_rows_backward)", who);
    if (mode != 0 && D == 32 && grad_out_dtype == BEVF_DTYPE_BF16 && aligned16(loc) && aligned16(attn) &&
        aligned16(grad_out) && aligned16(grad_value)) {
        cudaStream_t ds = st;
        if (mode == 2 && g_side_stream) {
            cudaEvent_t fork = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            join = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            cudaEventRecord(fork, st);
            cudaStreamWaitEvent(g_side_stream, fork, 0);
            ds = g_side_stream;
        }
        const int e = dense_coarse_backward(who, level_hw, level_start, level_hw_host, loc, attn, grad_out, grad_value,
                                            map_range, B, S, M, L, P, ds, &handled, &hl, 0, 0u, S, 0, 0);
        if (join) cudaEventRecord(join, g_side_stream);
        if (e) {
            if (join) cudaStreamWaitEvent(st, join, 0);
            return e;
        }
    }
    const int e = msda_backward_impl(who, value, value_dtype, level_hw, level_start, loc, attn, grad_out,
                                     grad_out_dtype, grad_value, grad_loc, grad_attn, row_map, nullptr, B, S, M, D,
                                     R, L, P, stream, handled, &hl);
    if (join) cudaStreamWaitEvent(st, join, 0);
    return e;
}

extern "C" int bevf_msda_rows_backward_f16acc(const void *value, int value_dtype, const int64_t *level_hw,
                                              const int64_t *level_start, const float *loc, const float *attn,
                                              const void *grad_out, int grad_out_dtype, void *grad_value_f16,
                                              const uint32_t *amax_bits, float *grad_loc, float *grad_attn,
                                              const int32_t *row_map, const int32_t *group_order, int B, int S,
                                              int M, int D, int R, int L, int P, void *stream) {
    const char *who = "bevf_msda_rows_backward_f16acc";
    if (!row_map && R > 0) return fail("%s: row_map is null", who);
    if (!grad_value_f16 || !amax_bits) return fail("%s: null pointer argument", who);
    MixedGv mx;
    mx.amax = amax_bits;
    return msda_backward_impl(who, value, value_dtype, level_hw, level_start, loc, attn, grad_out, grad_out_dtype,
                              reinterpret_cast<float *>(grad_value_f16), grad_loc, grad_attn, row_map, group_order, B, S,
                              M, D, R, L, P, stream, 0u, nullptr, true, &mx);
}

static int rows_backward_mixed_impl(const char *who, const void *value, int value_dtype, const int64_t *level_hw,
                                    const int64_t *level_start, const int32_t *level_hw_host, const float *loc,
                                    const float *attn, const void *grad_out, int grad_out_dtype,
                                    void *grad_value_fine_f16, float *grad_value_side, const uint32_t *amax_bits,
                                    int num_f16_levels, int num_rep_levels, int replicas, int first_dense_level,
                                    float *grad_loc, float *grad_attn, const int32_t *row_map,
                                    const int32_t *group_order, const int32_t *map_range, int B, int S, int M, int D,
                                    int R, int L, int P, void *stream, const ScaFuse *fz = nullptr) {
    if (!row_map && R > 0) return fail("%s: row_map is null", who);
    if (L <= 1 || L > kMaxLevels || num_f16_levels < 1 || num_f16_levels >= L)
        return fail("%s: num_f16_levels must be in [1, L - 1]", who);
    if (num_rep_levels < 0 || num_rep_levels > L - num_f16_levels || replicas < 1 || replicas > 64)
        return fail("%s: num_rep_levels must be in [0, L - num_f16_levels] and replicas in [1, 64]", who);
    const int num_side_from = num_f16_levels + num_rep_levels;       // first level of the fp32 side buffer
    // (no side levels: grad_value_side is never touched and may be NULL)
    if (!level_hw_host || !grad_value_fine_f16 || (!grad_value_side && num_side_from < L) || !amax_bits)
        return fail("%s: null pointer argument", who);
    if (map_range && (first_dense_level < num_side_from || first_dense_level >= L))
        return fail("%s: first_dense_level must be in [num_f16_levels + num_rep_levels, L - 1]", who);
    if (value_dtype != BEVF_DTYPE_BF16 || D != 32) return fail("%s: needs a bf16 value tensor and head_dim 32", who);
    if (!aligned16(grad_value_fine_f16) || !aligned16(grad_value_side))
        return fail("%s: device pointers must be 16-byte aligned", who);
    HostLevels hl;
    memset(&hl, 0, sizeof(hl));
    long long start = 0;
    for (int l = 0; l < L; ++l) {
        const int h = level_hw_host[2 * l], w = level_hw_host[2 * l + 1];
        if (h <= 0 || w <= 0 || h >= 32768 || w >= 32768) return fail("%s: bad host level shape", who);
        hl.h[l] = h; hl.w[l] = w; hl.start[l] = (int)start;
        start += (long long)h * w;
    }
    if (start != S) return fail("%s: host level shapes do not add up to S (%lld vs %lld)", who, start, S);
    MixedGv mx;
    mx.amax = amax_bits;
    mx.gv16 = reinterpret_cast<__half *>(grad_value_fine_f16);
    mx.mask = (1u << num_f16_levels) - 1u;
    mx.rep_start = hl.start[num_f16_levels];
    mx.side_start = num_side_from < L ? hl.start[num_side_from] : S;
    // no side levels: nothing is written to the side buffer, the launch below only needs a non-null pointer
    if (!grad_value_side) grad_value_side = reinterpret_cast<float *>(grad_value_fine_f16);
    mx.S_side = S - mx.side_start;
    mx.rep_k = replicas;
    if ((long long)(mx.rep_start + (long long)replicas * (mx.side_start - mx.rep_start)) * M * D >= (1ll << 31))
        return fail("%s: one map of grad_value_fine_f16 exceeds 2^31 elements", who);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned dense_levels = 0;                       // levels whose grad_value the dense kernel produced
    cudaEvent_t join = nullptr;
    const int mode = map_range ? mixed_dense_mode() : 0;
    // fused prep: the dense kernel reads the coarse samples the forward stored (levels [coarse_from, L))
    const float *dloc = fz ? reinterpret_cast<const float *>(fz->coarse_loc) : loc;
    const float *dattn = fz ? fz->coarse_attn : attn;
    const int loc_level0 = fz ? fz->coarse_from : 0;
    if (mode != 0 && R > 0 && grad_out_dtype == BEVF_DTYPE_BF16 && aligned16(dloc) && aligned16(dattn) &&
        aligned16(grad_out) && dloc && dattn && loc_level0 <= first_dense_level) {
        cudaStream_t ds = st;
        if (mode == 2 && !g_side_stream) {
            // the library default creates its stream lazily, never inside a stream capture (a captured call without
            // the stream runs both kernels on the caller's stream)
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusActive;
            if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) cudaGetLastError();
            else if (cs == cudaStreamCaptureStatusNone && ensure_side_stream(who) != 0) cudaGetLastError();
        }
        if (mode == 2 && g_side_stream) {
            cudaEvent_t fork = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            join = g_side_events[g_side_ev_next.fetch_add(1) % kSideEvents];
            cudaEventRecord(fork, st);
            cudaStreamWaitEvent(g_side_stream, fork, 0);
            ds = g_side_stream;
        }
        // the dense kernel takes exactly the levels [first_dense_level, L) or nothing: a level that it cannot take
        // leaves them all to the reduction path (no level is split between the two)
        const unsigned suffix = ((1u << L) - 1u) & ~((1u << first_dense_level) - 1u);
        HostLevels dhl;
        const int e = dense_coarse_backward(who, level_hw, level_start, level_hw_host, dloc, dattn, grad_out,
                                            grad_value_side, map_range, B, S, M, L, P, ds, &dense_levels, &dhl,
                                            first_dense_level, suffix, mx.S_side, mx.side_start, loc_level0);
        if (join) cudaEventRecord(join, g_side_stream);
        if (e) {
            if (join) cudaStreamWaitEvent(st, join, 0);
            return e;
        }
    }
    const int e = msda_backward_impl(who, value, value_dtype, level_hw, level_start, loc, attn, grad_out, grad_out_dtype,
                                     grad_value_side, grad_loc, grad_attn, row_map, group_order, B, S, M, D, R, L, P,
                                     stream, dense_levels, &hl, false, &mx, nullptr, fz);
    if (join) cudaStreamWaitEvent(st, join, 0);
    return e;
}

extern "C" int bevf_msda_rows_backward_mixed(const void *value, int value_dtype, const int64_t *level_hw,
                                             const int64_t *level_start, const int32_t *level_hw_host,
                                             const float *loc, const float *attn, const void *grad_out,
                                             int grad_out_dtype, void *grad_value_fine_f16, float *grad_value_side,
                                             const uint32_t *amax_bits, int num_f16_levels, float *grad_loc,
                                             float *grad_attn, const int32_t *row_map, const int32_t *group_order,
                                             int B, int S, int M, int D, int R, int L, int P, void *stream) {
    return rows_backward_mixed_impl("bevf_msda_rows_backward_mixed", value, value_dtype, level_hw, level_start,
                                    level_hw_host, loc, attn, grad_out, grad_out_dtype, grad_value_fine_f16,
                                    grad_value_side, amax_bits, num_f16_levels, 0, 1, L, grad_loc, grad_attn, row_map,
                                    group_order, nullptr, B, S, M, D, R, L, P, stream);
}

extern "C" int bevf_msda_rows_backward_mixed_dense(const void *value, int value_dtype, const int64_t *level_hw,
                                                   const int64_t *level_start, const int32_t *level_hw_host,
                                                   const float *loc, const float *attn, const void *grad_out,
                                                   int grad_out_dtype, void *grad_value_fine_f16,
                                                   float *grad_value_side, const uint32_t *amax_bits,
                                                   int num_f16_levels, int first_dense_level, float *grad_loc,
                                                   float *grad_attn, const int32_t *row_map, const int32_t *map_range,
                                                   int B, int S, int M, int D, int R, int L, int P, void *stream) {
    const char *who = "bevf_msda_rows_backward_mixed_dense";
    if (!map_range) return fail("%s: null pointer argument", who);
    return rows_backward_mixed_impl(who, value, value_dtype, level_hw, level_start, level_hw_host, loc, attn, grad_out,
                                    grad_out_dtype, grad_value_fine_f16, grad_value_side, amax_bits, num_f16_levels, 0,
                                    1, first_dense_level, grad_loc, grad_attn, row_map, nullptr, map_range, B, S, M, D,
                                    R, L, P, stream);
}

extern "C" int bevf_msda_rows_backward_replicated(const void *value, int value_dtype, const int64_t *level_hw,
                                                  const int64_t *level_start, const int32_t *level_hw_host,
                                                  const float *loc, const float *attn, const void *grad_out,
                                                  int grad_out_dtype, void *grad_value_f16, float *grad_value_side,
                                                  const uint32_t *amax_bits, int num_f16_levels, int num_rep_levels,
                                                  int replicas, int first_dense_level, float *grad_loc,
                                                  float *grad_attn, const int32_t *row_map,
                                                  const int32_t *group_order, const int32_t *map_range, int B, int S,
                                                  int M, int D, int R, int L, int P, void *stream) {
    const char *who = "bevf_msda_rows_backward_replicated";
    if (group_order && map_range) return fail("%s: group_order and map_range exclude each other", who);
    return rows_backward_mixed_impl(who, value, value_dtype, level_hw, level_start, level_hw_host, loc, attn, grad_out,
                                    grad_out_dtype, grad_value_f16, grad_value_side, amax_bits, num_f16_levels,
                                    num_rep_levels, replicas, map_range ? first_dense_level : L, grad_loc, grad_attn,
                                    row_map, group_order, map_range, B, S, M, D, R, L, P, stream);
}

// ---- SpatialCrossAttention's sampler with the sampling-point prep fused in (ScaFuse, msda_common.cuh) ----------
static int sca_fuse_args(const char *who, const float *raw, const float *ref_cam, const int32_t *pair_q,
                         const int32_t *pair_cam, const int32_t *pair_of, const float *stats, const float *coarse_loc,
                         const float *coarse_attn, int coarse_from, int M, int D, int R, int L, int P, int bs, int Nq,
                         int pairs, int Dz, int ncam, ScaFuse &fz) {
    if (M != kFuseHeads || D != 32 || L * P != kFuseLP)
        return fail("%s: 8 heads, head_dim 32 and num_levels * num_points == 32 only", who);
    if (bs <= 0 || Nq <= 0 || pairs < 0 || (long long)bs * pairs != R || Dz <= 0 || P % Dz != 0 || ncam <= 0 ||
        ncam > 16)
        return fail("%s: bad dimension (rows = bs * pairs, num_points a multiple of the Z anchors, ncam <= 16)", who);
    if (!raw || !ref_cam || !pair_q || !pair_cam || !stats) return fail("%s: null pointer argument", who);
    if (!aligned16(raw) || !aligned16(stats) || (reinterpret_cast<uintptr_t>(ref_cam) & 7u))
        return fail("%s: raw and stats must be 16-byte aligned, ref_cam 8-byte aligned", who);
    if (coarse_from < 0 || coarse_from > L || (coarse_from < L && (!coarse_loc || !coarse_attn)))
        return fail("%s: coarse_from must be in [0, L], with coarse_loc / coarse_attn when below L", who);
    if (!aligned16(coarse_loc) || !aligned16(coarse_attn))
        return fail("%s: coarse_loc / coarse_attn must be 16-byte aligned", who);
    fz.coarse_loc = const_cast<float2 *>(reinterpret_cast<const float2 *>(coarse_from < L ? coarse_loc : nullptr));
    fz.coarse_attn = const_cast<float *>(coarse_from < L ? coarse_attn : nullptr);
    fz.coarse_from = coarse_from;
    fz.raw = raw;
    fz.ref_cam = ref_cam;
    fz.pair_q = pair_q;
    fz.pair_cam = pair_cam;
    fz.pair_of = pair_of;
    fz.stats = const_cast<float2 *>(reinterpret_cast<const float2 *>(stats));
    fz.d_raw = nullptr;
    fz.bs = bs; fz.Nq = Nq; fz.R = pairs; fz.Dz = Dz; fz.ncam = ncam;
    return 0;
}

extern "C" int bevf_sca_rows_forward_fused(const void *value, int value_dtype, const int64_t *level_hw,
                                           const int64_t *level_start, const float *raw, const float *ref_cam,
                                           const int32_t *pair_q, const int32_t *pair_cam, float *stats,
                                           float *coarse_loc, float *coarse_attn, int coarse_from, void *out,
                                           int out_dtype, const int32_t *row_map, int B, int S, int M, int D, int R,
                                           int L, int P, int bs, int Nq, int pairs, int Dz, int ncam, void *stream) {
    const char *who = "bevf_sca_rows_forward_fused";
    if (!row_map && R > 0) return fail("%s: row_map is null", who);
    if (R == 0) return 0;
    ScaFuse fz;
    if (int e = sca_fuse_args(who, raw, ref_cam, pair_q, pair_cam, nullptr, stats, coarse_loc, coarse_attn,
                              coarse_from, M, D, R, L, P, bs, Nq, pairs, Dz, ncam, fz))
        return e;
    return msda_forward_impl(who, value, value_dtype, level_hw, level_start, nullptr, nullptr, out, out_dtype, row_map,
                             B, S, M, D, R, L, P, stream, &fz);
}

static int sca_rows_backward_fused_impl(
    const char *who, const void *value, int value_dtype, const int64_t *level_hw, const int64_t *level_start,
    const int32_t *level_hw_host, const float *raw, const float *stats, const float *coarse_loc,
    const float *coarse_attn, int coarse_from, const float *ref_cam, const int32_t *pair_q, const int32_t *pair_cam,
    const int32_t *pair_of, const void *grad_out, int grad_out_dtype, void *grad_value_f16, float *grad_value_side,
    const uint32_t *amax_bits, int num_f16_levels, int num_rep_levels, int replicas, int first_dense_level,
    float *grad_loc, float *grad_attn, void *d_raw, const int32_t *row_map, const int32_t *map_range, int B, int S,
    int M, int D, int R, int L, int P, int bs, int Nq, int pairs, int Dz, int ncam, void *stream) {
    if (R == 0) return 0;
    ScaFuse fz;
    if (int e = sca_fuse_args(who, raw, ref_cam, pair_q, pair_cam, pair_of, stats, coarse_loc, coarse_attn,
                              coarse_from, M, D, R, L, P, bs, Nq, pairs, Dz, ncam, fz))
        return e;
    if (!pair_of) return fail("%s: null pointer argument", who);
    if (!d_raw || !aligned16(d_raw)) return fail("%s: d_raw must be a 16-byte aligned bf16 buffer", who);
    fz.d_raw = reinterpret_cast<bf16 *>(d_raw);
    return rows_backward_mixed_impl(who, value, value_dtype, level_hw, level_start, level_hw_host, nullptr, nullptr,
                                    grad_out, grad_out_dtype, grad_value_f16, grad_value_side, amax_bits,
                                    num_f16_levels, num_rep_levels, replicas, map_range ? first_dense_level : L,
                                    grad_loc, grad_attn, row_map, nullptr, map_range, B, S, M, D, R, L, P, stream, &fz);
}

extern "C" int bevf_sca_rows_backward_fused(const void *value, int value_dtype, const int64_t *level_hw,
                                            const int64_t *level_start, const int32_t *level_hw_host, const float *raw,
                                            const float *stats, const float *coarse_loc, const float *coarse_attn,
                                            int coarse_from, const float *ref_cam, const int32_t *pair_q,
                                            const int32_t *pair_cam, const int32_t *pair_of, const void *grad_out,
                                            int grad_out_dtype, void *grad_value_fine_f16, float *grad_value_side,
                                            const uint32_t *amax_bits, int num_f16_levels, int first_dense_level,
                                            float *grad_loc, float *grad_attn, void *d_raw, const int32_t *row_map,
                                            const int32_t *map_range, int B, int S, int M, int D, int R, int L, int P,
                                            int bs, int Nq, int pairs, int Dz, int ncam, void *stream) {
    return sca_rows_backward_fused_impl("bevf_sca_rows_backward_fused", value, value_dtype, level_hw, level_start,
                                        level_hw_host, raw, stats, coarse_loc, coarse_attn, coarse_from, ref_cam, pair_q,
                                        pair_cam, pair_of, grad_out, grad_out_dtype, grad_value_fine_f16,
                                        grad_value_side, amax_bits, num_f16_levels, 0, 1, first_dense_level, grad_loc,
                                        grad_attn, d_raw, row_map, map_range, B, S, M, D, R, L, P, bs, Nq, pairs, Dz,
                                        ncam, stream);
}

extern "C" int bevf_sca_rows_backward_fused_replicated(
    const void *value, int value_dtype, const int64_t *level_hw, const int64_t *level_start,
    const int32_t *level_hw_host, const float *raw, const float *stats, const float *coarse_loc,
    const float *coarse_attn, int coarse_from, const float *ref_cam, const int32_t *pair_q, const int32_t *pair_cam,
    const int32_t *pair_of, const void *grad_out, int grad_out_dtype, void *grad_value_f16, float *grad_value_side,
    const uint32_t *amax_bits, int num_f16_levels, int num_rep_levels, int replicas, int first_dense_level,
    float *grad_loc, float *grad_attn, void *d_raw, const int32_t *row_map, const int32_t *map_range, int B, int S,
    int M, int D, int R, int L, int P, int bs, int Nq, int pairs, int Dz, int ncam, void *stream) {
    return sca_rows_backward_fused_impl("bevf_sca_rows_backward_fused_replicated", value, value_dtype, level_hw,
                                        level_start, level_hw_host, raw, stats, coarse_loc, coarse_attn, coarse_from,
                                        ref_cam, pair_q, pair_cam, pair_of, grad_out, grad_out_dtype, grad_value_f16,
                                        grad_value_side, amax_bits, num_f16_levels, num_rep_levels, replicas,
                                        first_dense_level, grad_loc, grad_attn, d_raw, row_map, map_range, B, S, M, D,
                                        R, L, P, bs, Nq, pairs, Dz, ncam, stream);
}

namespace bevf {
int fx_bounds_launch(const char *who, const float *attn, const void *grad_out, int grad_out_dtype,
                     const int32_t *row_map, long long qrows, int M, int D, int L, int P, uint32_t *bounds,
                     cudaStream_t st);                                                    // gvfx.cu

// Deterministic backward: the bounds of this launch, then the fixed-point scatter.  rows_per_map (Q, or R for a row
// list) caps the contributions one element can receive; frac_bits above what that allows could overflow.
static int msda_backward_fx_impl(const char *who, const void *value, int value_dtype, const int64_t *level_hw,
                                 const int64_t *level_start, const float *loc, const float *attn, const void *grad_out,
                                 int grad_out_dtype, int64_t *grad_value_fx, uint32_t *bounds, int frac_bits,
                                 float *grad_loc, float *grad_attn, const int32_t *row_map, int B, int S, int M, int D,
                                 int Q, int L, int P, void *stream) {
    if (int e = check_dims(who, B, S, M, D, Q, L, P)) return e;
    const long long qrows = (row_map ? 1ll : (long long)B) * Q;
    if (qrows == 0) return 0;
    if (!bounds || !grad_value_fx || !attn || !grad_out) return fail("%s: null pointer argument", who);
    const int kmax = bevf_msda_fx_frac_bits(Q, L, P);
    if (frac_bits < 0 || frac_bits > kmax)
        return fail("%s: frac_bits must be in [0, %lld] for this launch (bevf_msda_fx_frac_bits)", who, kmax);
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = fx_bounds_launch(who, attn, grad_out, grad_out_dtype, row_map, qrows, M, D, L, P, bounds, st)) return e;
    FxGv fx;
    fx.bounds = bounds;
    fx.frac_bits = frac_bits;
    return msda_backward_impl(who, value, value_dtype, level_hw, level_start, loc, attn, grad_out, grad_out_dtype,
                              reinterpret_cast<float *>(grad_value_fx), grad_loc, grad_attn, row_map, nullptr, B, S, M,
                              D, Q, L, P, stream, 0u, nullptr, false, nullptr, &fx);
}
}  // namespace bevf

extern "C" int bevf_msda_backward_fx(const void *value, int value_dtype, const int64_t *level_hw,
                                     const int64_t *level_start, const float *loc, const float *attn,
                                     const void *grad_out, int grad_out_dtype, int64_t *grad_value_fx,
                                     uint32_t *bounds, int frac_bits, float *grad_loc, float *grad_attn, int B, int S,
                                     int M, int D, int Q, int L, int P, void *stream) {
    return msda_backward_fx_impl("bevf_msda_backward_fx", value, value_dtype, level_hw, level_start, loc, attn, grad_out,
                                 grad_out_dtype, grad_value_fx, bounds, frac_bits, grad_loc, grad_attn, nullptr, B, S, M,
                                 D, Q, L, P, stream);
}

extern "C" int bevf_msda_rows_backward_fx(const void *value, int value_dtype, const int64_t *level_hw,
                                          const int64_t *level_start, const float *loc, const float *attn,
                                          const void *grad_out, int grad_out_dtype, int64_t *grad_value_fx,
                                          uint32_t *bounds, int frac_bits, float *grad_loc, float *grad_attn,
                                          const int32_t *row_map, int B, int S, int M, int D, int R, int L, int P,
                                          void *stream) {
    if (!row_map && R > 0) return fail("%s: row_map is null", "bevf_msda_rows_backward_fx");
    return msda_backward_fx_impl("bevf_msda_rows_backward_fx", value, value_dtype, level_hw, level_start, loc, attn,
                                 grad_out, grad_out_dtype, grad_value_fx, bounds, frac_bits, grad_loc, grad_attn, row_map,
                                 B, S, M, D, R, L, P, stream);
}

extern "C" int bevf_msda_set_backward_mode(int mode) {
    if (mode < 0 || mode > 2)
        return fail("%s: mode must be 0 (one kernel), 1 (split) or 2 (hybrid)", "bevf_msda_set_backward_mode");
    if (mode == 2 && !g_side_stream) {
        if (cudaStreamCreateWithFlags(&g_side_stream, cudaStreamNonBlocking) != cudaSuccess) {
            cudaGetLastError();
            g_side_stream = nullptr;
            return fail("%s: cannot create the second stream", "bevf_msda_set_backward_mode");
        }
        for (int i = 0; i < kSideEvents; ++i) cudaEventCreateWithFlags(&g_side_events[i], cudaEventDisableTiming);
    }
    g_bwd_mode.store(mode, std::memory_order_relaxed);
    return 0;
}

extern "C" int bevf_msda_rows_backward_ordered(const void *value, int value_dtype, const int64_t *level_hw,
                                               const int64_t *level_start, const float *loc,
                                               const float *attn, const void *grad_out,
                                               int grad_out_dtype, float *grad_value, float *grad_loc,
                                               float *grad_attn, const int32_t *row_map,
                                               const int32_t *group_order, int B, int S, int M, int D,
                                               int R, int L, int P, void *stream) {
    if (!row_map && R > 0) return fail("%s: row_map is null", "bevf_msda_rows_backward_ordered");
    return msda_backward_impl("bevf_msda_rows_backward_ordered", value, value_dtype, level_hw,
                              level_start, loc, attn, grad_out, grad_out_dtype, grad_value, grad_loc,
                              grad_attn, row_map, group_order, B, S, M, D, R, L, P, stream);
}
