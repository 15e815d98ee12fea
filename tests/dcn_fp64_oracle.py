"""Float64 restatement of modulated_deform_conv2d (SURVEY.md Appendix B) in im2col form, and the per-element error
bars of the library's kernels (csrc/dcn.cu around the wgmma GEMMs of csrc/gemm.cu).

Inputs are the storage-typed tensors the op sees (offset, mask and weight already cast to the input's dtype); they are
widened exactly.  The one rounding the restatement shares with the kernels is the sampling position: the exact
integer base plus the widened offset, added once in fp32, so floor() picks the same cell on both sides.  Everything
else is float64.  Works on CPU or CUDA tensors.

Bars (gamma, bar_16, UNIT, TINY of tests/gemm_fp64_oracle.py; u = 2^-24):
  * columns: fp32 weights (two products, one multiply by the mask) and a 4-term fused sum: gamma_8 of
    cabs = |mask| sum_corners w |x|, then the store to a 16-bit type: u16 |col| + TINY.
  * forward: the GEMM over the restated columns, mag = |Wp| cabs + |b|, plus |Wp| times the columns' error; 16-bit
    outputs add their own store (bar_16, one rounding per k16 step of the reduction), fp32 (torch matmul, any order)
    gamma_{K + 2} mag.
  * dcols = dy Wp: the same GEMM bars over |dy| |Wp|.
  * grad_input: an unordered fp32 sum of n contributions mask * w * dcol (n per element, counted): gamma_{n + 3}
    times sum |mask| w (|dcol| + bar_dcol), plus the dcols' error; in 64-bit fixed point each contribution rounds by at
    most 2^(E - K - 1) instead, then one conversion to fp32; then the store to the input's dtype.
  * grad_mask / grad_offset: a Cg-term fp32 dot product of dcol with the sample (or its derivative, times the mask):
    gamma_{Cg + 8} over the absolute terms, plus the dcols' error times the absolute sample, then the store.
  * grad_weight / grad_bias: sums over the R rows in any split order: gamma_{R + 16} of |dy|^T cabs (of sum |dy|),
    plus |dy|^T times the columns' error, then the conversion to the parameter's dtype.
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

from tests.gemm_fp64_oracle import TINY, U32, UNIT, bar_16, check_exact_bound, gamma  # noqa: F401

F64 = torch.float64


def out_size(H, W, kh, kw, stride, padding, dilation):
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    return ((H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1)


def geometry(x, weight, stride, padding, dilation, dg):
    """(N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg), the tuple the C entry points take."""
    N, C, H, W = x.shape
    kh, kw = weight.shape[2:]
    Ho, Wo = out_size(H, W, kh, kw, stride, padding, dilation)
    return (N, H, W, C, Ho, Wo, kh, kw, *stride, *padding, *dilation, dg)


def positions(offset, geom):
    """Sampling positions (y, x), each (N, dg, kk, Ho*Wo) float64: the fp32 sum of the integer base and the offset."""
    N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg = geom
    kk, dev = kh * kw, offset.device
    off = offset.to(torch.float32).reshape(N, dg, kk, 2, Ho * Wo)
    ho = torch.arange(Ho, device=dev).repeat_interleave(Wo)
    wo = torch.arange(Wo, device=dev).repeat(Ho)
    i = torch.arange(kk, device=dev) // kw
    j = torch.arange(kk, device=dev) % kw
    by = (ho[None, :] * sh - ph + i[:, None] * dh).to(torch.float32)
    bx = (wo[None, :] * sw - pw + j[:, None] * dw).to(torch.float32)
    return (by + off[:, :, :, 0]).to(F64), (bx + off[:, :, :, 1]).to(F64)


def corners(y, x, H, W):
    """The bilinear corners of every sample (SURVEY.md Appendix A): [(flat pixel index, weight, inside)] for the
    corners 00, 01 (x + 1), 10 (y + 1), 11, and (lx, ly, hx, hy).  Outside -1 < y < H, -1 < x < W nothing counts."""
    valid = (y > -1) & (x > -1) & (y < H) & (x < W)
    y = torch.where(valid, y, torch.zeros_like(y))
    x = torch.where(valid, x, torch.zeros_like(x))
    y0, x0 = y.floor(), x.floor()
    ly, lx = y - y0, x - x0
    hy, hx = 1 - ly, 1 - lx
    out = []
    for (cy, wy), (cx, wx) in itertools.product(((y0, hy), (y0 + 1, ly)), ((x0, hx), (x0 + 1, lx))):
        inside = valid & (cy >= 0) & (cy <= H - 1) & (cx >= 0) & (cx <= W - 1)
        idx = (cy.clamp(0, H - 1) * W + cx.clamp(0, W - 1)).long()
        out.append((idx, torch.where(inside, wy * wx, torch.zeros_like(wy)), inside))
    return out, (lx, ly, hx, hy)


def _gather(xg, idx):
    """xg (N, dg, HW, Cg), idx (N, dg, kk, P) -> (N, dg, kk, P, Cg)."""
    N, dg, kk, P = idx.shape
    Cg = xg.shape[-1]
    flat = idx.reshape(N, dg, kk * P, 1).expand(N, dg, kk * P, Cg)
    return torch.gather(xg, 2, flat).reshape(N, dg, kk, P, Cg)


class Sampled:
    """Per (image, group, tap, pixel) samples of the pixels ``pix`` (indices into Ho*Wo; None: all)."""

    def __init__(self, x, offset, mask, geom, pix=None):
        N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg = geom
        self.geom, kk, Cg = geom, kh * kw, C // dg
        y, xx = positions(offset, geom)
        m = mask.to(F64).reshape(N, dg, kk, Ho * Wo)
        if pix is not None:
            y, xx, m = y[..., pix], xx[..., pix], m[..., pix]
        self.m = m
        self.cs, (self.lx, self.ly, self.hx, self.hy) = corners(y, xx, H, W)
        xg = x.to(F64).reshape(N, dg, Cg, H * W).transpose(2, 3)
        # corner values, zero where the corner is outside the map: (N, dg, kk, P, Cg)
        self.v = [torch.where(ins[..., None], _gather(xg, idx), torch.zeros((), dtype=F64, device=x.device))
                  for idx, _, ins in self.cs]
        self.s = sum(w[..., None] * v for (_, w, _), v in zip(self.cs, self.v))
        self.sabs = sum(w[..., None] * v.abs() for (_, w, _), v in zip(self.cs, self.v))

    def cols(self, absval=False):
        """(N * P, kk * C): column tap * C + g * Cg + c."""
        s = self.sabs if absval else self.s
        c = (self.m.abs() if absval else self.m)[..., None] * s
        N, dg, kk, P, Cg = c.shape
        return c.permute(0, 3, 2, 1, 4).reshape(N * P, kk * dg * Cg)


def weight_rows(weight):
    """Wp = weight.permute(0, 2, 3, 1) as (Cout, kk * C) float64."""
    return weight.to(F64).permute(0, 2, 3, 1).reshape(weight.shape[0], -1)


def _st(dtype):
    """The storage type whose bars apply (float64 inputs, as in the CPU comparison, get fp32's)."""
    return dtype if dtype in UNIT else torch.float32


def _store(v, e, dtype):
    """Bar of a value computed with error e and stored once in ``dtype``."""
    dtype = _st(dtype)
    if dtype == torch.float32:
        return U32 * v.abs() + (1 + U32) * e + TINY[torch.float32]
    return UNIT[dtype] * v.abs() + (1 + UNIT[dtype]) * e + TINY[dtype]


def col_error(smp, dtype):
    cabs = smp.cols(absval=True)
    e = gamma(8) * cabs
    if dtype != torch.float32:
        e = UNIT[dtype] * cabs + (1 + UNIT[dtype]) * e + TINY[dtype]
    return e


def forward(x, offset, mask, weight, bias, geom, pix=None):
    """(y64 (N * P, Cout), bar) of the output rows of pixels ``pix``; rows are image-major."""
    dtype = _st(x.dtype)
    smp = Sampled(x, offset, mask, geom, pix)
    wp = weight_rows(weight)
    y = smp.cols() @ wp.t()
    b = torch.zeros(wp.shape[0], dtype=F64, device=x.device) if bias is None else bias.to(F64)
    y = y + b
    K = wp.shape[1]
    mag = smp.cols(absval=True) @ wp.abs().t() + b.abs()
    ecol = col_error(smp, dtype) @ wp.abs().t()
    if dtype == torch.float32:
        bar = gamma(K + 2) * mag + ecol
    else:
        bar = bar_16(mag, y, K // 16, dtype) + (1 + UNIT[dtype]) * ecol
    return y, bar


def fx_frac_bits(rows_per_map, L, P):
    """bevf_msda_fx_frac_bits: the fraction bits no sum of that many contributions can overflow."""
    count = max(rows_per_map, 1) * L * P * 4
    lg = 0
    while lg < 63 and (1 << lg) < count:
        lg += 1
    return min(62 - lg, 40)


def fx_exponent(a, b):
    """fx_exponent (common.cuh) of two non-negative fp32 bounds: every product a' b' with a' <= a, b' <= b is below
    2^E."""
    bits = np.array([a, b], dtype=np.float32).view(np.uint32).astype(np.int64) >> 23
    return int(np.maximum(bits, 1).sum() - 252)


def backward(x, offset, mask, weight, bias, dy, geom, deterministic=False):
    """Float64 gradients and bars: dict name -> (want, bar) for input (N, C, H, W), offset, mask, weight, bias."""
    N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg = geom
    dtype, dev, kk, Cg, P = _st(x.dtype), x.device, kh * kw, C // dg, Ho * Wo
    smp = Sampled(x, offset, mask, geom)
    wp = weight_rows(weight)
    Cout = wp.shape[0]
    dyr = dy.to(F64).permute(0, 2, 3, 1).reshape(N * P, Cout)
    res = {}
    # dcols and their bar, as (N, dg, kk, P, Cg)
    dc = dyr @ wp
    dmag = dyr.abs() @ wp.abs()
    edc = gamma(Cout + 2) * dmag if dtype == torch.float32 else bar_16(dmag, dc, Cout // 16, dtype, adds=0)

    def groups(t):
        return t.reshape(N, P, kk, dg, Cg).permute(0, 3, 2, 1, 4)
    dc, edc = groups(dc), groups(edc)
    m = smp.m[..., None]
    v00, v01, v10, v11 = smp.v
    lx, ly, hx, hy = (t[..., None] for t in (smp.lx, smp.ly, smp.hx, smp.hy))
    # grad_mask
    gm = (dc * smp.s).sum(-1)
    egm = gamma(Cg + 8) * (dc.abs() * smp.sabs).sum(-1) + (edc * smp.sabs).sum(-1)
    res["mask"] = (gm.reshape(N, dg * kk, Ho, Wo), _store(gm, egm, dtype).reshape(N, dg * kk, Ho, Wo))
    # grad_offset: (y, x) per tap
    dy_ = hx * (v10 - v00) + lx * (v11 - v01)
    dx_ = hy * (v01 - v00) + ly * (v11 - v10)
    ay = hx * (v10.abs() + v00.abs()) + lx * (v11.abs() + v01.abs())
    ax = hy * (v01.abs() + v00.abs()) + ly * (v11.abs() + v10.abs())
    go, ego = [], []
    for d, a in ((dy_, ay), (dx_, ax)):
        g = smp.m * (dc * d).sum(-1)
        e = smp.m.abs() * (gamma(Cg + 8) * (dc.abs() * a).sum(-1) + (edc * a).sum(-1))
        go.append(g)
        ego.append(_store(g, e, dtype))
    res["offset"] = tuple(torch.stack(t, 3).reshape(N, dg * 2 * kk, Ho, Wo) for t in (go, ego))
    # grad_input: scatter of mask * w * dcol onto the corners
    gi = torch.zeros(N, dg, H * W, Cg, dtype=F64, device=dev)
    mag = torch.zeros_like(gi)
    errd = torch.zeros_like(gi)
    cnt = torch.zeros(N, dg, H * W, 1, dtype=F64, device=dev)
    for idx, w, _ in smp.cs:
        q = (smp.m * w)[..., None]
        ix = idx.reshape(N, dg, kk * P, 1)
        gi.scatter_add_(2, ix.expand(-1, -1, -1, Cg), (q * dc).reshape(N, dg, kk * P, Cg))
        mag.scatter_add_(2, ix.expand(-1, -1, -1, Cg), (q.abs() * dc.abs()).reshape(N, dg, kk * P, Cg))
        errd.scatter_add_(2, ix.expand(-1, -1, -1, Cg), (q.abs() * edc).reshape(N, dg, kk * P, Cg))
        cnt.scatter_add_(2, ix, (q != 0).to(F64).reshape(N, dg, kk * P, 1))
    if deterministic:
        K = fx_frac_bits(P, 1, kk)
        dmax = float((dc.abs() + edc).max()) if dc.numel() else 0.0
        E = fx_exponent(float(mask.to(torch.float32).abs().max()), dmax)
        e = cnt * 2.0 ** (E - K - 1) + errd
        e = U32 * gi.abs() + (1 + U32) * e          # the conversion to fp32
    else:
        e = gamma_n(cnt + 3) * (mag + errd) + errd
    def nchw(t):
        return t.transpose(2, 3).reshape(N, C, H, W)
    res["input"] = (nchw(gi), nchw(e if dtype == torch.float32 and not deterministic else _store(gi, e, dtype)))
    # weight / bias
    cols, cabs, ecol = smp.cols(), smp.cols(absval=True), col_error(smp, dtype)
    R = N * P
    gw = dyr.t() @ cols
    egw = gamma(R + 16) * (dyr.abs().t() @ cabs) + dyr.abs().t() @ ecol

    def wshape(t):
        return t.reshape(Cout, kh, kw, C).permute(0, 3, 1, 2)
    res["weight"] = (wshape(gw), wshape(_store(gw, egw, weight.dtype)))
    if bias is not None:
        gb = dyr.sum(0)
        egb = gamma(R + 16) * dyr.abs().sum(0)
        res["bias"] = (gb, _store(gb, egb, bias.dtype))
    return res


def gamma_n(n, u=U32):
    """gamma of a per-element count tensor."""
    return n * u / (1.0 - n * u)


def rn(v64, dtype):
    """Round to nearest even of float64 values to ``dtype`` (via fp32: exact whenever the value is), as float64."""
    return v64.to(torch.float32).to(dtype).to(F64)


def exact_inputs(N, C, H, W, Cout, kh, kw, stride, padding, dilation, dg, dtype, seed, device="cpu", bias=True):
    """The exact regime: integer inputs in [-4, 4], weights and dy in {-1, 0, 1}, offsets in quarter pixels, mask in
    {0, 1/2, 1}.  Every product and partial sum of the op is then a small multiple of 2^-5, and every value the op
    stores between its stages (columns, dcols) is representable in ``dtype``; check_exact_bound asserts the GEMMs'
    headroom.  Outputs and gradients then equal the float64 value rounded once."""
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = out_size(H, W, kh, kw, stride, padding, dilation)
    kk = kh * kw
    x = torch.randint(-4, 5, (N, C, H, W), generator=g).to(dtype)
    wt = torch.randint(-1, 2, (Cout, C, kh, kw), generator=g).to(dtype)
    b = torch.randint(-8, 9, (Cout,), generator=g).to(dtype) if bias else None
    off = (torch.randint(-12, 13, (N, 2 * dg * kk, Ho, Wo), generator=g) / 4.0).to(dtype)
    mask = (torch.randint(0, 3, (N, dg * kk, Ho, Wo), generator=g) / 2.0).to(dtype)
    dy = torch.randint(-1, 2, (N, Cout, Ho, Wo), generator=g).to(dtype)
    assert Cout <= 256, "|dcol| <= Cout must stay an integer every storage type holds"
    check_exact_bound(torch.full((1, C * kk), 4.0 * 32), torch.ones(1, 1))     # |col| <= 4 in 2^-5 quanta, |w| <= 1
    return [t.to(device) if t is not None else None for t in (x, off, mask, wt, b, dy)]


def normal_inputs(N, C, H, W, Cout, kh, kw, stride, padding, dilation, dg, dtype, seed, device="cpu", bias=True,
                  off_scale=2.0):
    """The rounding regime: normal inputs, weights at the module's initialiser scale, offsets of a few pixels."""
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = out_size(H, W, kh, kw, stride, padding, dilation)
    kk = kh * kw
    x = torch.randn(N, C, H, W, generator=g).to(dtype)
    wt = ((torch.rand(Cout, C, kh, kw, generator=g) * 2 - 1) / math.sqrt(C * kk)).to(dtype)
    b = (torch.randn(Cout, generator=g) * 0.1).to(dtype) if bias else None
    off = (torch.randn(N, 2 * dg * kk, Ho, Wo, generator=g) * off_scale).to(dtype)
    mask = torch.rand(N, dg * kk, Ho, Wo, generator=g).to(dtype)
    dy = torch.randn(N, Cout, Ho, Wo, generator=g).to(dtype)
    return [t.to(device) if t is not None else None for t in (x, off, mask, wt, b, dy)]
