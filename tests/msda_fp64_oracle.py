"""Float64 restatement of the multi-scale deformable attention sampler (csrc/msda.cu, msda_splat.cuh, msda_dense.cu),
the yardstick of tests/test_msda_fp64_gpu.py.  Test infrastructure only: plain torch ops on whatever device the inputs
live on, no kernels of this package.  tests/test_msda_fp64_cpu.py pins it against Oracle-S in float64 and shows that
its bars reject the plausible kernel bugs.

Arithmetic: SURVEY.md Appendix A, i.e. multi_scale_deformable_attn_function.py:118-160 (mmcv's
ms_deform_attn_forward / _backward).  For sample (row r, head m, level l, point p) with loc (lx_, ly_):

    x = loc_x * W_l - 0.5,  y = loc_y * H_l - 0.5;  the sample counts iff -1 < x < W_l and -1 < y < H_l
    x0 = floor(x), lx = x - x0, hx = 1 - lx (same in y);  corners 00 = (x0, y0), 01 = (x0 + 1, y0),
    10 = (x0, y0 + 1), 11 = (x0 + 1, y0 + 1) with weights hy hx, hy lx, ly hx, ly lx; a corner outside the map
    contributes nothing
    out[r, m]            = sum_{l,p} a * sum_k w_k v_k
    grad_value[b, k-pix] += a * w_k * g[r, m]
    grad_attn[r, m, l, p] = sum_c g_c sum_k w_k v_k,c
    grad_loc             = (W * a * (hy (d01 - d00) + ly (d11 - d10)),  H * a * (hx (d10 - d00) + lx (d11 - d01)))
                           with the corner dots d_k = <g, v_k>

The coordinate x is rounded exactly as the kernels (make_corner, msda_common.cuh) and mmcv's fp32 kernel round it:
fl(fl(loc * W) - 0.5) with two float32 operations, then the range test, floor and lx = x - floor(x) (exact) in
float32.  So the restatement picks the kernels' cell for every sample, on cell borders too, and grad_loc -- a
discontinuous function of the cell -- needs no outlier allowance.  Everything after the coordinates runs in float64.

Each output comes with the magnitudes its bar is built from (``*_mag``, ``gv_count``); the ``bar_*`` functions turn
them into per-element bounds, one per arithmetic path, each deriving its own.  Rows are processed in chunks so that a
rig-sized launch stays within a few GB on the device.
"""
import torch

F64 = torch.float64
U32 = 2.0 ** -24          # unit roundoff of float32
U16 = 2.0 ** -11          # float16
UBF = 2.0 ** -8           # bfloat16
UNIT = {torch.float32: U32, torch.float16: U16, torch.bfloat16: UBF}
# half the spacing of the subnormals: the absolute rounding error of a store below the normal range
TINY = {torch.float32: 2.0 ** -150, torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134}

# corner k -> (dx, dy)
_CORNERS = ((0, 0), (1, 0), (0, 1), (1, 1))

MUTATIONS = ("swap_01_10", "drop_last_sample", "neighbour_level_offset", "grad_loc_without_wh",
             "scatter_to_partner_map", "fma_coordinates")


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u): the relative bound of n successive roundings (Higham, Accuracy and Stability of
    Numerical Algorithms, Lemma 3.1)."""
    return n * u / (1.0 - n * u)


# ------------------------------------------------------------------------------------------------
# sample geometry
# ------------------------------------------------------------------------------------------------
def _coords(loc, hw, fma=False):
    """loc (..., L, P, 2) float32, hw (L, 2) [H, W] -> x, y (float32 after the range test, 0 for invalid samples)
    and the validity mask.  fma: the single rounding of an FMA (a kernel bug the mutation checks model)."""
    hwf = hw.to(loc.device)
    H = hwf[:, 0].to(torch.float32).view(-1, 1)
    W = hwf[:, 1].to(torch.float32).view(-1, 1)
    lx_, ly_ = loc[..., 0].to(torch.float32), loc[..., 1].to(torch.float32)
    if fma:
        x = (lx_.to(F64) * W.to(F64) - 0.5).to(torch.float32)
        y = (ly_.to(F64) * H.to(F64) - 0.5).to(torch.float32)
    else:
        x = lx_ * W
        x = x - 0.5
        y = ly_ * H
        y = y - 0.5
    valid = (x > -1.0) & (y > -1.0) & (x < W) & (y < H)
    zero = torch.zeros((), dtype=torch.float32, device=loc.device)
    return torch.where(valid, x, zero), torch.where(valid, y, zero), valid


def _geometry(loc, hw, starts, S, mutate=None):
    """Per sample (..., L, P): the 4 corners' pixel indices into the map (..., L, P, 4), their float64 weights (zero
    for corners outside the map or invalid samples), lx, ly, and W, H per level (float64, broadcastable)."""
    x, y, valid = _coords(loc, hw, fma=mutate == "fma_coordinates")
    xf, yf = torch.floor(x), torch.floor(y)
    lx, ly = (x - xf).to(F64), (y - yf).to(F64)                  # exact in float32
    x0, y0 = xf.to(torch.int64), yf.to(torch.int64)
    dev = loc.device
    H = hw[:, 0].to(dev).view(-1, 1)
    W = hw[:, 1].to(dev).view(-1, 1)
    st = starts.to(dev).view(-1, 1)
    if mutate == "neighbour_level_offset":
        st = torch.roll(st, -1, 0)
    hx, hy = 1.0 - lx, 1.0 - ly
    wts = (hy * hx, hy * lx, ly * hx, ly * lx)
    pix, w = [], []
    for (dx, dy), wk in zip(_CORNERS, wts):
        xk, yk = x0 + dx, y0 + dy
        ok = valid & (xk >= 0) & (xk < W) & (yk >= 0) & (yk < H)
        p = st + yk.clamp(min=0) * W + xk.clamp(min=0)
        pix.append(torch.where(ok, p, torch.zeros_like(p)).clamp(max=S - 1))
        w.append(torch.where(ok, wk, torch.zeros_like(wk)))
    pix, w = torch.stack(pix, -1), torch.stack(w, -1)
    if mutate == "swap_01_10":
        pix = pix[..., [0, 2, 1, 3]]
    return pix, w, lx, ly, W.to(F64), H.to(F64)


# ------------------------------------------------------------------------------------------------
# layouts
# ------------------------------------------------------------------------------------------------
def as_rows(value, loc, attn, row_map=None, grad_out=None):
    """Dense (B, Q, M, L, P[, 2]) inputs -> the row-list form (B*Q, M, L, P[, 2]) with row_map = the batch index.
    Row-list inputs pass through.  Returns (loc, attn, row_map int64, grad_out as (R, M, D) or None)."""
    NB, S, M, D = value.shape
    if row_map is None:
        B, Q = loc.shape[:2]
        loc = loc.reshape(B * Q, *loc.shape[2:])
        attn = attn.reshape(B * Q, *attn.shape[2:])
        row_map = torch.arange(B, device=loc.device).repeat_interleave(Q)
    row_map = row_map.to(loc.device, torch.int64)
    if grad_out is not None:
        grad_out = grad_out.reshape(loc.shape[0], M, D)
    return loc, attn, row_map, grad_out


def _chunk_rows(R, M, LP, D, budget=2 ** 28):
    per_row = max(1, M * LP * 4 * D * 8 * 4)
    return max(1, min(R, budget // per_row))


# ------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------
def forward(value, level_hw, level_start, loc, attn, row_map=None, group_order=None, mutate=None):
    """out (R, M*D) or (B, Q, M*D) float64 and out_mag = sum |a w v| per element.  Rows with row_map -1: zeros.
    group_order (a permutation of the rows in which a kernel visits them) does not change the sums: accepted and
    ignored."""
    dense = row_map is None
    NB, S, M, D = value.shape
    shape = (loc.shape[0], loc.shape[1], M * D) if dense else (loc.shape[0], M * D)
    loc, attn, rmap, _ = as_rows(value, loc, attn, row_map)
    R, _, L, P = attn.shape
    hw, st = torch.as_tensor(level_hw).cpu().long(), torch.as_tensor(level_start).cpu().long()
    vflat = value.reshape(NB * S * M, D)
    out = torch.zeros(R, M, D, dtype=F64, device=loc.device)
    mag = torch.zeros_like(out)
    step = _chunk_rows(R, M, L * P, D)
    mvec = torch.arange(M, device=loc.device).view(1, M, 1, 1, 1)
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        pix, w, _, _, _, _ = _geometry(loc[r0:r1], hw, st, S, mutate)         # (c, M, L, P, 4)
        b = rmap[r0:r1].view(-1, 1, 1, 1, 1)
        live = b >= 0
        a = attn[r0:r1].to(F64)
        if mutate == "drop_last_sample":
            a = a.clone()
            a[..., -1, -1] = 0
        aw = (a[..., None] * w) * live
        idx = ((b.clamp(min=0) * S + pix) * M + mvec).reshape(-1)
        v = vflat[idx].to(F64).view(r1 - r0, M, L * P * 4, D)
        awf = aw.reshape(r1 - r0, M, L * P * 4, 1)
        out[r0:r1] = (awf * v).sum(2)
        mag[r0:r1] = (awf.abs() * v.abs()).sum(2)
    return out.view(shape), mag.view(shape)


# ------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------
def backward(value, level_hw, level_start, loc, attn, grad_out, row_map=None, group_order=None, mutate=None,
             dense_mult=False, gv_rows=None):
    """Gradients of out w.r.t. value, loc and attn for the upstream gradient grad_out, with their bar magnitudes.

    Returns a dict of float64 tensors in the layouts of the inputs:
      grad_value, gv_mag (sum |a w g|), gv_count (contributions with a non-zero weight, per (b, pixel, m));
      gv_dense_mag (only with ``dense_mult``): sum |a w g| * min(4, h), h = the contributions of the same row and head
        to the same pixel (the rounding count of msda_dense.cu's coefficients, see bar_gv_dense);
      grad_attn, ga_mag (sum_c sum_k |g w_k v_k|);
      grad_loc, gl_mag (W |a| (hy (D00 + D01) + ly (D10 + D11)), H |a| (hx (D00 + D10) + lx (D01 + D11)) with the
        corner magnitudes D_k = sum_c |g_c v_k,c|).
    ``gv_rows``: a (K,) int64 tensor of flat (b * S + pixel) indices; grad_value and its magnitudes are then returned
    for those pixels only, as (K, M, D) -- for launches whose full float64 grad_value would not fit."""
    dense = row_map is None
    NB, S, M, D = value.shape
    loc_shape, attn_shape = loc.shape, attn.shape
    locr, attnr, rmap, g_all = as_rows(value, loc, attn, row_map, grad_out)
    R, _, L, P = attnr.shape
    dev = locr.device
    hw, st = torch.as_tensor(level_hw).cpu().long(), torch.as_tensor(level_start).cpu().long()
    vflat = value.reshape(NB * S * M, D)
    if gv_rows is not None:
        remap = torch.full((NB * S,), -1, dtype=torch.int64, device=dev)
        remap[gv_rows.to(dev)] = torch.arange(gv_rows.numel(), device=dev)
        n_gv = gv_rows.numel()
    else:
        n_gv = NB * S
    gv = torch.zeros(n_gv * M, D, dtype=F64, device=dev)
    gv_mag = torch.zeros_like(gv)
    gv_cnt = torch.zeros(n_gv * M, dtype=F64, device=dev)
    gv_dmag = torch.zeros_like(gv) if dense_mult else None
    ga = torch.zeros(R, M, L, P, dtype=F64, device=dev)
    ga_mag = torch.zeros_like(ga)
    gl = torch.zeros(R, M, L, P, 2, dtype=F64, device=dev)
    gl_mag = torch.zeros_like(gl)
    step = _chunk_rows(R, M, L * P, D)
    mvec = torch.arange(M, device=dev).view(1, M, 1, 1, 1)
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        c = r1 - r0
        pix, w, lx, ly, Wl, Hl = _geometry(locr[r0:r1], hw, st, S, mutate)
        b = rmap[r0:r1].view(-1, 1, 1, 1, 1)
        live = b >= 0
        w = w * live
        a = attnr[r0:r1].to(F64)
        if mutate == "drop_last_sample":
            a = a.clone()
            a[..., -1, -1] = 0
        g = g_all[r0:r1].to(F64)                                               # (c, M, D)
        idx = ((b.clamp(min=0) * S + pix) * M + mvec)                          # (c, M, L, P, 4)
        v = vflat[idx.reshape(-1)].to(F64).view(c, M, L, P, 4, D)
        gb = g.view(c, M, 1, 1, 1, D)
        d = (v * gb).sum(-1)                                                   # corner dots (c, M, L, P, 4)
        dm = (v.abs() * gb.abs()).sum(-1)
        ga[r0:r1] = (w * d).sum(-1)
        ga_mag[r0:r1] = (w.abs() * dm).sum(-1)
        inmap = _inmap(locr[r0:r1], hw, mutate) & live                         # the f_k flags: d_k counts
        d = d * inmap
        dm = dm * inmap
        hx, hy = 1.0 - lx, 1.0 - ly
        sx = 1.0 if mutate == "grad_loc_without_wh" else Wl
        sy = 1.0 if mutate == "grad_loc_without_wh" else Hl
        gl[r0:r1, ..., 0] = sx * a * (hy * (d[..., 1] - d[..., 0]) + ly * (d[..., 3] - d[..., 2]))
        gl[r0:r1, ..., 1] = sy * a * (hx * (d[..., 2] - d[..., 0]) + lx * (d[..., 3] - d[..., 1]))
        gl_mag[r0:r1, ..., 0] = Wl * a.abs() * (hy * (dm[..., 0] + dm[..., 1]) + ly * (dm[..., 2] + dm[..., 3]))
        gl_mag[r0:r1, ..., 1] = Hl * a.abs() * (hx * (dm[..., 0] + dm[..., 2]) + lx * (dm[..., 1] + dm[..., 3]))
        # grad_value: a * w_k * g into (b, pixel, m)
        aw = a[..., None] * w                                                  # (c, M, L, P, 4)
        tgt_b = b
        if mutate == "scatter_to_partner_map":
            # the paired scatter of msda_bwd_d32 with the partner's map: row group grp ^ 4 of the same warp
            flat = (torch.arange(r0, r1, device=dev).view(-1, 1) * M + torch.arange(M, device=dev)).view(c, M)
            partner = (flat ^ 4).clamp(max=R * M - 1) // M
            tgt_b = rmap[partner].view(c, M, 1, 1, 1)
            tgt_b = torch.where(tgt_b >= 0, tgt_b, b)
        pidx = tgt_b.clamp(min=0) * S + pix                                    # (c, M, L, P, 4)
        if gv_rows is not None:
            pidx = remap[pidx]
            keep = (pidx >= 0) & (aw != 0)
        else:
            keep = aw != 0
        tgt = (pidx.clamp(min=0) * M + mvec)[keep]
        contrib = aw[keep].view(-1, 1) * g.view(c, M, 1, 1, 1, D).expand(c, M, L, P, 4, D)[keep]
        gv.index_add_(0, tgt, contrib)
        gv_mag.index_add_(0, tgt, contrib.abs())
        gv_cnt.index_add_(0, tgt, torch.ones_like(tgt, dtype=F64))
        if dense_mult:
            key = (torch.arange(c, device=dev).view(c, 1, 1, 1, 1) * M + mvec) * (NB * S) + pidx
            kk = key[keep]
            _, inv, cnt = torch.unique(kk, return_inverse=True, return_counts=True)
            mult = cnt[inv].clamp(max=4).to(F64).view(-1, 1)
            gv_dmag.index_add_(0, tgt, contrib.abs() * mult)
        del v, contrib
    out = dict(grad_attn=ga.view(attn_shape), ga_mag=ga_mag.view(attn_shape),
               grad_loc=gl.view(loc_shape), gl_mag=gl_mag.view(loc_shape))
    gshape = (n_gv, M, D) if gv_rows is not None else value.shape
    out.update(grad_value=gv.view(gshape), gv_mag=gv_mag.view(gshape),
               gv_count=gv_cnt.view(*gshape[:-1], 1).expand(gshape))
    if dense_mult:
        out["gv_dense_mag"] = gv_dmag.view(gshape)
    return out


def _inmap(loc, hw, mutate):
    """(..., L, P, 4): which corners of each sample lie inside the map (the kernels' f_k flags)."""
    x, y, valid = _coords(loc, hw, fma=mutate == "fma_coordinates")
    x0, y0 = torch.floor(x).to(torch.int64), torch.floor(y).to(torch.int64)
    H = hw[:, 0].to(loc.device).view(-1, 1)
    W = hw[:, 1].to(loc.device).view(-1, 1)
    fl = []
    for dx, dy in _CORNERS:
        xk, yk = x0 + dx, y0 + dy
        fl.append(valid & (xk >= 0) & (xk < W) & (yk >= 0) & (yk < H))
    return torch.stack(fl, -1)


# ------------------------------------------------------------------------------------------------
# bars
# ------------------------------------------------------------------------------------------------
def bar_forward(mag, ref, LP, out_dtype=torch.float32, packed_bf16_weights=False):
    """Forward output.

    fp32 arithmetic: every term a * w_k * v_k carries the roundings of hx = 1 - lx, hy * hx and (w * a) (3) and
    the product with v (1, inside the FMA); the sum over the 4 L P terms rounds once per addition (4 L P, in any
    order; the generic kernel's 4-term inner sum and its product by a add 2).  So |err| <= gamma_{4 L P + 8} * sum
    |a w v|.
    bf16 value rows through msda_fwd_d32 (``packed_bf16_weights``): the kernel packs a * w into bf16
    (pack_bf16x2) before the exact bf16 x bf16 products -- one bf16 rounding of every weight, 2^-8 |a w| -- whatever
    the output type: + 2^-8 sum |a w v|.
    16-bit output: one rounding of the stored value, u_out * (|ref| + the bound above), or below the normal range
    (fp16: 2^-14) half the subnormal spacing, 2^-25 for fp16."""
    bar = gamma(4 * LP + 8) * mag
    if packed_bf16_weights:
        bar = bar + UBF * mag
    if out_dtype != torch.float32:
        bar = bar + UNIT[out_dtype] * (ref.abs() + bar) + TINY[out_dtype]
    return bar


def bar_grad_value_f32(mag, count):
    """fp32 grad_value (one-kernel, generic, split / splat and hybrid backwards).  A contribution
    a * w_k * g is formed with 5 roundings (1 - lx, the weight product, * a, * g; the splat kernel's FMA into its
    register window counts as the product's), and the element's sum of ``count`` contributions rounds once per
    addition in any order (L2 vector reductions, the splat's per-lane windows and flushes): gamma_{count + 6}."""
    return gamma(count + 6) * mag


def bar_grad_attn(mag, D):
    """grad_attn = sum_k w_k <g, v_k>.  The corner dot over D channels rounds at most D + 5 times along any path of
    the kernels' sums (a lane's FMA chain plus the log2(LANES) reduce-scatter steps in msda_bwd_d32, the per-channel
    accumulation and the 5 butterfly steps in msda_bwd_generic); the weights (3) and the 4-corner combination (3) add
    6: gamma_{D + 11} * sum_c sum_k |g w_k v_k|."""
    return gamma(D + 11) * mag


def bar_grad_loc(mag, D):
    """grad_loc = W a (hy (d01 - d00) + ly (d11 - d10)) (and the y twin).  The dots carry gamma_{D + 5} |D_k| each;
    differences, products by hy / ly / a / W and the sum add 6 more: gamma_{D + 11} * W |a| (hy (D00 + D01) +
    ly (D10 + D11)).  Cancellation in d01 - d00 is why the bar is built on the corner magnitudes, not on |ref|."""
    return gamma(D + 11) * mag


def bar_gv_f16(mag, count, ref, scale):
    """Scaled-fp16 grad_value (msda_bwd_d32<bf16, TG, true, __half>, and the fine levels of the mixed backward),
    returned as bf16.  Each contribution (a w * scale) * g is formed in fp32 (gamma_6), packed to fp16 (one rounding,
    2^-11 of the term) and added by an f16x2 vector reduction (one fp16 rounding per addition, 2^-11 of the running
    sum <= sum of the terms).  count + 1 fp16 roundings relative to the magnitude: (count + 1) 2^-11 sum |a w g|.
    Below 2^-14 fp16 is subnormal with a fixed spacing 2^-24 (scaled units): every one of the 2 count roundings may
    also lose half of it, 2 count 2^-25 / scale.  Unscaling divides by a power of two (exact) and rounds to bf16:
    2^-8 (|ref| + the accumulation bound)."""
    acc = (count + 1) * U16 * mag + gamma(6) * mag + 2 * count * 2.0 ** -25 / scale
    return acc + UBF * (ref.abs() + acc)


def bar_gv_f32_to_bf16(mag, count, ref):
    """fp32-accumulated grad_value stored as bf16 (the side levels of the mixed backward after bevf_gv_merge)."""
    acc = bar_grad_value_f32(mag, count)
    return acc + UBF * (ref.abs() + acc)


def bar_gv_dense(mag, dense_mag, count):
    """grad_value of the levels msda_dense.cu takes.  The coefficient C[pixel, row] = sum of the row's a * w_k on that
    pixel is written into a bf16 slab in up to four corner rounds, each a bf16 read-add-write: one bf16 rounding
    (2^-8 of the partial coefficient, <= the sum of its terms' magnitudes) per round that touches it, i.e. at most
    min(4, h) of them for the h contributions the row makes to the pixel -- the ``dense_mag`` weighting.  grad_out is
    bf16, the tensor-core products are exact and accumulate in fp32; the per-unit results are added into grad_value by
    vector reductions: one fp32 rounding per contribution and per flush, gamma_{2 count + 6} sum |a w g| (the
    same-pixel lanes' fp32 pre-sum included)."""
    return UBF * dense_mag + gamma(2 * count + 6) * mag


def fx_exponent(amax, gmax):
    """E of the fixed-point scale (common.cuh: fx_exponent): max|attn| < 2^ea, max|grad_out| < 2^eg, E = ea + eg
    (a zero or denormal maximum counts as exponent field 1)."""
    def e(x):
        bits = int(torch.tensor([float(x)], dtype=torch.float32).view(torch.int32).item()) & 0x7fffffff
        return max(bits >> 23, 1) - 126
    return e(amax) + e(gmax)


def bar_gv_fx(mag, count, ref, E, K, out_dtype=torch.float32):
    """64-bit fixed-point grad_value (deterministic mode).  The factor q = a * w_k is an fp32 product (gamma_4 with the
    weight's own roundings); q * g is exact in double and rounded to the nearest multiple of 2^(E - K): half a unit
    per contribution, count 2^(E - K - 1) (test_deterministic_gpu._fx_bound states the same with count's maximum
    n_max); the integer sum is exact.  bevf_msda_fx_convert rounds the result once to the output type."""
    acc = gamma(4) * mag + count * 2.0 ** (E - K - 1)
    return acc + UNIT[out_dtype] * (ref.abs() + acc)


# ------------------------------------------------------------------------------------------------
# inputs shared by the CPU and GPU files
# ------------------------------------------------------------------------------------------------
def border_locs(hw, n, gen, kinds=("integer", "inside_edge", "outside_edge", "nonfinite", "uniform")):
    """n sampling locations per level (n, L, 2) float32 mixing the places where the cell choice is delicate:
    x / y exactly on integers after fl(fl(loc * W) - 0.5) (cell borders), -1 + ulp and W - ulp (just inside),
    exactly -1 and W (just outside), NaN, +-inf, +-1e9, and uniform positions in (-0.1, 1.1)."""
    hw = torch.as_tensor(hw).long()
    L = hw.shape[0]
    out = torch.empty(n, L, 2, dtype=torch.float32)
    nonfinite = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e9, -1e9], dtype=torch.float32)
    for l in range(L):
        for j, S_ in ((0, int(hw[l, 1])), (1, int(hw[l, 0]))):
            kind = torch.randint(0, len(kinds), (n,), generator=gen)
            u = torch.rand(n, generator=gen, dtype=F64)
            k = torch.randint(0, S_, (n,), generator=gen).to(F64)
            low = u < 0.5
            cand = {
                "integer": ((k + 0.5) / S_).to(torch.float32),
                "inside_edge": torch.where(low, _step_inside(-0.5 / S_, S_, +1), _step_inside((S_ + 0.5) / S_, S_, -1)),
                "outside_edge": torch.where(low, torch.tensor(-0.5 / S_, dtype=torch.float32),
                                            torch.tensor((S_ + 0.5) / S_, dtype=torch.float32)),
                "nonfinite": nonfinite[(u * 5).long().clamp(max=4)],
                "uniform": (-0.1 + 1.2 * u).to(torch.float32),
            }
            vals = torch.empty(n, dtype=torch.float32)
            for i, kd in enumerate(kinds):
                sel = kind == i
                vals[sel] = torch.broadcast_to(cand[kd], (n,))[sel]
            out[:, l, j] = vals
    return out


def _step_inside(v, S_, direction):
    """The float32 loc next to v (stepping by ulps) whose fl(fl(loc * S) - 0.5) is strictly inside (-1, S)."""
    v = torch.tensor(v, dtype=torch.float32)
    toward = torch.tensor(float("inf") if direction > 0 else -float("inf"), dtype=torch.float32)
    for _ in range(64):
        x = (v * S_) - 0.5
        if -1.0 < float(x) < S_:
            return v
        v = torch.nextafter(v, toward)
    return v


def pyramid(level_hw):
    hw = torch.tensor(level_hw, dtype=torch.int64)
    n = hw[:, 0] * hw[:, 1]
    starts = torch.cat([torch.zeros(1, dtype=torch.int64), n.cumsum(0)[:-1]])
    return hw, starts, int(n.sum())


def make_inputs(levels, M, P, D=32, NB=2, Q=None, R=None, unused=(), seed=0, gscale=1.0, border_frac=0.25,
                cluster=None, attn_sign=False):
    """Seeded inputs of one case, on the CPU, in float32: value (NB, S, M, D), loc and attn in the dense layout
    (NB, Q, M, L, P[, 2]) when Q is given, or the row-list layout (R, M, L, P[, 2]) with a row_map when R is given
    (rows cycling over the maps, ``unused`` rows set to -1).  A ``border_frac`` share of the samples take
    border_locs' delicate positions.  ``cluster`` = (centre spread, radius): locations gathered around a few centres,
    to steer the splat kernel into its window passes.  grad_out is scaled by ``gscale``."""
    gen = torch.Generator().manual_seed(seed)
    hw, starts, S = pyramid(levels)
    L = len(levels)
    value = torch.randn(NB, S, M, D, generator=gen)
    nrows = (NB * Q if Q is not None else R)
    if cluster is None:
        loc = torch.rand(nrows, M, L, P, 2, generator=gen) * 1.2 - 0.1
    else:
        spread, radius = cluster
        centres = torch.rand(max(1, nrows // 64 + 1), 1, 1, 1, 2, generator=gen) * spread + (0.5 - spread / 2)
        loc = centres.repeat_interleave(64, 0)[:nrows] + (torch.rand(nrows, M, L, P, 2, generator=gen) - 0.5) * radius
    if border_frac > 0:
        nb = max(1, int(nrows * M * P * border_frac))
        bl = border_locs(hw, nb, gen)                                          # (nb, L, 2)
        sel = torch.randperm(nrows * M * P, generator=gen)[:nb]
        flat = loc.permute(0, 1, 3, 2, 4).reshape(nrows * M * P, L, 2)
        flat[sel] = bl
        loc = flat.view(nrows, M, P, L, 2).permute(0, 1, 3, 2, 4).contiguous()
    attn = torch.rand(nrows, M, L, P, generator=gen) + 0.05
    attn = attn / attn.sum((-1, -2), keepdim=True)
    if attn_sign:
        attn = attn * (torch.randint(0, 2, attn.shape, generator=gen) * 2 - 1)
    grad_out = torch.randn(nrows, M * D, generator=gen) * gscale
    if Q is not None:
        loc = loc.view(NB, Q, M, L, P, 2)
        attn = attn.view(NB, Q, M, L, P)
        grad_out = grad_out.view(NB, Q, M * D)
        row_map = None
    else:
        row_map = (torch.arange(R) % NB).to(torch.int32)
        for u in unused:
            row_map[u] = -1
    return dict(value=value, level_hw=hw, level_start=starts, loc=loc.contiguous(), attn=attn.contiguous(),
                grad_out=grad_out.contiguous(), row_map=row_map)


# shapes of the GPU cases (tests/test_msda_fp64_gpu.py); the CPU mutation checks run on "rows_m5"
SHAPES = {
    # L P = 9: not a multiple of LANES (4 for 16-bit rows, 8 for fp32); M = 5: a warp's row groups span several
    # queries and maps, and the paired scatter's partner row (grp ^ 4) is another query's, some of them unused
    "rows_m5": dict(levels=[(9, 13), (5, 6), (2, 3)], M=5, P=3, NB=3, R=61, unused=(6, 13, 40)),
    # dense (B, Q, ...) layout; 1 x 1, 1 x W and H x 1 levels; L P = 8
    "dense_edges": dict(levels=[(1, 1), (1, 7), (6, 1), (4, 5)], M=3, P=2, NB=2, Q=11),
    # 16 levels (the maximum), L P = 16
    "rows_l16": dict(levels=[(2, 3), (1, 1), (3, 1), (1, 4), (4, 2), (2, 2), (5, 1), (1, 5), (3, 3), (2, 1), (1, 2),
                             (6, 2), (2, 6), (1, 3), (3, 2), (4, 4)], M=9, P=1, NB=2, R=29, unused=(0, 28)),
    # L P = 3 < LANES, one head
    "rows_m1": dict(levels=[(7, 5)], M=1, P=3, NB=2, R=40, unused=tuple(range(1, 8))),
    # 16 heads, L P = 4 = LANES of 16-bit rows
    "rows_m16": dict(levels=[(8, 12), (4, 6)], M=16, P=2, NB=2, R=21, unused=(3,)),
    # L P^2 = 65025, just under 65536: level_of's magic division must stay exact
    "magic_max": dict(levels=[(5, 7)], M=1, P=255, NB=1, Q=3),
    # 8 heads (the BEVFormer configs), P = 4
    "rows_m8": dict(levels=[(12, 20), (6, 10), (3, 5)], M=8, P=4, NB=3, R=200, unused=tuple(range(17, 23))),
}
