"""The fused glue kernels of csrc/encoder_ops.cu against the float64 restatements of tests/encoder_ops_oracle.py, at
the shapes, types and edges of every template instantiation and dispatch branch.

Which kernel each dispatch branch runs is asserted through torch.profiler kernel names in a child process
(test_every_case_runs_its_instantiation reruns this file there with ENV_PROFILE set; the first case of each branch
launches its kernels under the profiler, and every case stops before its numeric checks).  Hundreds of profiler sessions leave CUPTI in a state where later sessions of
the same process drop GPU activity records, which would break the kernel-inventory tests of other files; the numeric
checks in this process run without the profiler.

Bars are derived from the rounding involved (u = 2^-24, the fp32 unit roundoff); each test states its derivation.
No bar is normalised by max|ref|: every element is held to its own bound.  Outputs are prefilled with NaN where the
test owns the buffer, so that "fully overwritten" and "left untouched" are both checked."""
import contextlib
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from bevformer_b200 import _lib, ops
from tests import encoder_ops_oracle as eo
from tests.test_encoder_ops_cpu import ln_inputs

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F64 = torch.float64
U = eo.U32
DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
CNAME = {"float32": "float", "bfloat16": "__nv_bfloat16", "float16": "__half"}
NAN = float("nan")
ENV_PROFILE = "BEVF_ENCODER_OPS_PROFILE"
PROFILING = os.environ.get(ENV_PROFILE) == "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def kernels(fn, attempts=6):
    """Run fn under the profiler; returns (fn's result, set of CUDA kernel names that ran).

    Short back-to-back profiler sessions occasionally come back with some or all GPU activity records missing.  An
    exp kernel before fn and a sqrt kernel after it bracket the window: a trace without both is incomplete, and fn
    (which every caller makes repeatable) runs again under a new session."""
    import time
    from torch.profiler import ProfilerActivity, profile
    for i in range(attempts):
        time.sleep(0.05 * i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=DEV).exp_()
            out = fn()
            torch.ones(1, device=DEV).sqrt_()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if any("exp" in n for n in names) and any("sqrt" in n for n in names):
            return out, names
    raise AssertionError(f"the profiler lost GPU activity records {attempts} times in a row: {sorted(names)}")


def assert_ran(names, *subs):
    for s in subs:
        assert any(s in n for n in names), (s, sorted(n[:120] for n in names))


_VERIFIED = set()


def ran(fn, *expected, last=True):
    """fn().  In the profiling child process: fn() under the profiler, asserting that the kernels named in
    ``expected`` (name substrings) are among those it launched -- once per dispatch branch (distinct ``expected``),
    by the first case that expects it, which keeps the child to about sixty profiler sessions.  After the case's
    ``last`` launch the case ends there; its numeric checks run in the parent process."""
    if not PROFILING:
        return fn()
    if expected in _VERIFIED:
        out = None if last else fn()
    else:
        out, names = kernels(fn)
        assert_ran(names, *expected)
        _VERIFIED.add(expected)
    if last:
        pytest.skip("dispatch checked")
    return out


def test_every_case_runs_its_instantiation():
    """Every dispatch branch of this file's cases, rerun in a child process, launches the template instantiation it is
    meant for (see the module docstring for why a child process)."""
    if PROFILING:
        pytest.skip("this is the profiling run")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider",
                        "-k", "not test_every_case_runs_its_instantiation and not refuses"],
                       cwd=ROOT, env=dict(os.environ, **{ENV_PROFILE: "1"}), capture_output=True, text=True,
                       timeout=900)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    last = [ln for ln in r.stdout.splitlines() if ln.strip()][-1]
    assert "skipped" in last and "passed" not in last and "failed" not in last, tail


def assert_within(got, ref, bar, what):
    """|got - ref| <= bar element by element (got in its storage type, ref / bar float64); NaN in got fails."""
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= bar)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        ratio = (err / bar.clamp(min=1e-300)).flatten()
        ratio = ratio[~torch.isnan(ratio)]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bar; first at {i}: got "
                             f"{got.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r} bar "
                             f"{bar.flatten()[i].item():.3g}; worst err/bar {ratio.max().item() if ratio.numel() else 'nan'}")


def _st():
    return torch.cuda.current_stream(DEV).cuda_stream


def _check(st):
    _lib.check(st, _lib.load())


@contextlib.contextmanager
def deterministic_mode():
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def _ln_run(c, t, det, spy):
    """One forward + backward through ops.LayerNormResidual; returns (y, y2, grads) with grads of x, res, gamma, beta."""
    x = t["x"].detach().clone().requires_grad_(True)
    res = None if t["res"] is None else t["res"].detach().clone().requires_grad_(True)
    gamma = t["gamma"].detach().clone().requires_grad_(True)
    beta = t["beta"].detach().clone().requires_grad_(True)
    out = ops.LayerNormResidual.apply(x, res, gamma, beta, c["eps"], c["p"], t["pos"], c["twin"])
    y, y2 = (out if isinstance(out, tuple) else (out, None))
    outs, grads = [y], [t["dy"]]
    if c["pos"] and c["strided"]:
        # y + pos feeds a cat, as the next TSA's query does: its gradient is a column slice (row stride 2C)
        big = torch.cat([torch.zeros_like(y2), y2], -1)
        outs.append(big)
        grads.append(torch.cat([torch.zeros_like(t["dy2"]), t["dy2"]], -1))
    elif y2 is not None:
        outs.append(y2)
        grads.append(t["dy2"])
    ctx = deterministic_mode() if det else contextlib.nullcontext()
    with ctx:
        torch.autograd.backward(outs, grads, retain_graph=c["p"] > 0)
        # with dropout, a second backward of the same forward (same mask) under an unrelated gradient: an element
        # is dropped iff dx is exactly zero in both (one 16-bit dx can underflow to zero where the element was kept)
        dx2 = torch.autograd.grad(outs, x, [g.roll(1, -1) for g in grads])[0] if c["p"] > 0 else None
    torch.cuda.synchronize()
    return y.detach(), None if (y2 is None or c["twin"]) else y2.detach(), (
        x.grad, None if res is None else res.grad, gamma.grad, beta.grad), dx2


class _Spy:
    """Records the dy_plus_pos row stride ops passes to the backward entry points."""

    def __init__(self, monkeypatch):
        lib = _lib.load()
        self.ld2 = []
        for name, idx in (("bevf_layernorm_backward", 8), ("bevf_layernorm_backward_det", 8)):
            orig = getattr(lib, name)

            def wrap(*a, _orig=orig, _idx=idx):
                self.ld2.append(int(a[_idx]))
                return _orig(*a)
            monkeypatch.setattr(lib, name, wrap)


def ln_plan(rows):
    """(rows per CTA, CTAs) of the LayerNorm backward: ceil(rows / (4 SMs)) rounded up to 8."""
    per = -(-rows // (4 * sms()))
    rpc = max(8, -(-per // 8) * 8)
    return rpc, -(-rows // rpc)


@pytest.mark.parametrize("c", eo.ln_cases(), ids=eo.ln_case_id)
def test_layernorm(c, monkeypatch):
    """Forward y (and y + pos) and backward dx, d_res, dgamma, dbeta against the float64 LayerNorm.

    Bars, with u = 2^-24 and K = C/32 + 12 (a lane's C/32 sequential adds, 5 butterfly levels, and the few
    subtract / multiply / rsqrt / fma steps after them):
      x-hat:   E = K u (|x-hat| + |mean| rstd + 1): the mean is off by K u mean|xin| <= K u (|mean| + std), and
               rstd by K u relative; dropout's scale and the residual add round xin by 2u more.
      y:       2 (|gamma| E + u |beta|) in fp32 (the factor 2 covers the products not counted term by term);
               16-bit storage adds one ulp of the float64 value (round to nearest, <= half an ulp of the computed
               value, which can sit in the binade above).
      y + pos: the bar of y, plus u |y + pos| for the add, plus one storage ulp.
      d_in:    rstd (g gamma - s1 - x-hat s2) cancels, so its bound is in the operands' scale:
               2 [rstd (2u |g gamma| + K u mean|g gamma| + |x-hat| (K u mean|g gamma x-hat| + mean(|g gamma| E))
               + |s2| E) + K u |d_in|], plus one storage ulp in 16-bit; dx adds u |dx| for the dropout scale.
      dgamma, dbeta: sums over rows; one lane sums rpc/8 rows, 8 warps meet in shared memory, the CTAs in global
               memory (atomics, or in CTA order in deterministic mode): 2 [(rpc/8 + 8 + CTAs + 2) u sum|g x-hat|
               + sum |g| E], plus one storage ulp when the parameter is 16-bit.
    Dropout: the keep-mask is read off the exact zeros of dx (under two unrelated upstream gradients); the drop count is within 6 sigma of the binomial
    mean, forward y is checked against that mask, and d_res (when present) against the unmasked gradient.
    The deterministic backward runs twice: bitwise equal, and within the same bars as the atomic one."""
    torch.manual_seed(1234)
    C, p = c["C"], c["p"]
    rows = eo.ln_rows(c["rows"], sms())
    t = ln_inputs(c, rows, torch.Generator().manual_seed(13), device=DEV)
    spy = _Spy(monkeypatch)
    T, TP = CNAME[c["adt"]], CNAME[c["pdt"]]
    y, y2, grads, dx2 = ran(lambda: _ln_run(c, t, False, spy), f"bevf::layernorm_fwd<{T}, {TP}, {C}>",
                            f"bevf::layernorm_bwd<{T}, {TP}, {C}, false>", last=p > 0)
    if PROFILING:                      # p = 0: the deterministic backward's instantiation, then stop
        ran(lambda: _ln_run(c, t, True, spy), f"bevf::layernorm_bwd<{T}, {TP}, {C}, true>",
            "bevf::partials_add_kernel")
    if c["strided"]:
        # read in place at row stride 2C (a single row is contiguous whatever its stride)
        assert set(spy.ld2) == {2 * C if rows > 1 else C}, spy.ld2
    dx, dres, dgamma, dbeta = grads
    keep = None
    if p > 0:
        keep = (dx != 0) | (dx2 != 0)
        dropped = int((~keep).sum())
        n = keep.numel()
        assert abs(dropped - n * p) <= eo.binomial_bound(n, p), (dropped, n * p)
    adt = DT[c["adt"]]
    f = eo.layernorm_forward(t["x"], t["res"], t["gamma"], t["beta"], c["eps"], keep, p, t["pos"])
    K = C / 32 + 12
    gam, bet = t["gamma"].to(F64), t["beta"].to(F64)
    E = K * U * (f["xhat"].abs() + (f["mean"].abs() * f["rstd"])[:, None] + 1)
    bar_y32 = 2 * (gam.abs() * E + U * bet.abs())
    st_ulp = (lambda r: eo.ulp(r, adt)) if adt != torch.float32 else (lambda r: torch.zeros_like(r))
    assert_within(y, f["y"], bar_y32 + st_ulp(f["y"]), "y")
    if y2 is not None:
        assert_within(y2, f["y2"], bar_y32 + U * f["y2"].abs() + st_ulp(f["y2"]), "y + pos")
    b = eo.layernorm_backward(t["x"], t["res"], t["gamma"], c["eps"], t["dy"], t["dy2"], keep, p)
    gg, xh, rstd = b["gg"], b["xhat"], b["rstd"][:, None]
    s2 = (gg * xh).mean(-1, keepdim=True)
    bar_d = 2 * (rstd * (2 * U * gg.abs() + K * U * gg.abs().mean(-1, keepdim=True)
                         + xh.abs() * (K * U * (gg * xh).abs().mean(-1, keepdim=True)
                                       + (gg.abs() * E).mean(-1, keepdim=True))
                         + s2.abs() * E) + K * U * b["dres"].abs())
    scale = 1.0 / (1.0 - p)
    assert_within(dx, b["dx"], (bar_d * (scale if p > 0 else 1.0)) + U * b["dx"].abs() + st_ulp(b["dx"]), "dx")
    if dres is not None:
        want = b["dres"] if p > 0 else b["dx"]
        assert_within(dres, want, bar_d + st_ulp(want), "d_res")
    g = t["dy"].to(F64) if t["dy2"] is None else t["dy"].to(F64) + t["dy2"].to(F64)
    rpc, grid = ln_plan(rows)
    depth = rpc / 8 + 8 + grid + 2
    pdt = DT[c["pdt"]]
    p_ulp = (lambda r: eo.ulp(r, pdt)) if pdt != torch.float32 else (lambda r: torch.zeros_like(r))
    bar_dg = 2 * (depth * U * (g * xh).abs().sum(0) + (g.abs() * E).sum(0))
    bar_db = 2 * depth * U * g.abs().sum(0)
    assert_within(dgamma, b["dgamma"], bar_dg + p_ulp(b["dgamma"]), "dgamma")
    assert_within(dbeta, b["dbeta"], bar_db + p_ulp(b["dbeta"]), "dbeta")
    if p > 0:
        return          # each run draws a new mask: the deterministic comparison needs p = 0
    _, _, g1, _ = ran(lambda: _ln_run(c, t, True, spy), f"bevf::layernorm_bwd<{T}, {TP}, {C}, true>",
                      "bevf::partials_add_kernel")
    _, _, g2, _ = _ln_run(c, t, True, spy)
    for a, b_, n in zip(g1, g2, ("dx", "d_res", "dgamma", "dbeta")):
        if a is not None:
            assert torch.equal(a, b_), n
    assert_within(g1[2], b["dgamma"], bar_dg + p_ulp(b["dgamma"]), "dgamma (deterministic)")
    assert_within(g1[3], b["dbeta"], bar_db + p_ulp(b["dbeta"]), "dbeta (deterministic)")
    assert torch.equal(g1[0], dx), "dx does not depend on the reduction mode"


# ------------------------------------------------------------------------------------------------
# sampling-point prep
# ------------------------------------------------------------------------------------------------
def _softmax_bar(raw_logits, LP):
    """Per-weight bar of a softmax over groups of LP fp32 logits, relative to the weight: exp correctly rounded
    (u/2) of an argument l - max rounded by u |l - max|; the LP-term positive sum by (LP - 1) u; the reciprocal and
    the product by u each.  (LP + 4 + |l - max| + max_group |l - max|) u, times 2 for the products not counted."""
    lg = raw_logits.to(F64).reshape(-1, LP)
    dev = lg.max(-1, keepdim=True).values - lg
    return 2 * (LP + 4 + dev + dev.max(-1, keepdim=True).values) * U


def _prep_loc_bar(off_over_wh, loc):
    """loc = ref + offset / (W or H): a correctly rounded division (u) and one add (u of the sum)."""
    return 2 * U * (off_over_wh.abs() + loc.abs())


def _drawbar(d_ref, out_dtype, scale):
    """d_raw: the offsets part is g / (W or H), one rounding; the logits part a (ga - sum a ga) cancels, so its bound
    is in the scale of the operands (``scale``, per element); one storage ulp when d_raw is 16-bit."""
    b = scale
    if out_dtype != torch.float32:
        b = b + eo.ulp(d_ref, out_dtype)
    return b


def _tsa_inputs(c, seed):
    M, L, P, B, Nq = c["M"], c["L"], c["P"], c["B"], c["Nq"]
    g = torch.Generator().manual_seed(seed)
    raw = (torch.randn(B * Nq, M * 2 * L * P * 3, generator=g) * 2).to(DEV)
    ref2d = torch.rand(B * 2, Nq, L, 2, generator=g).to(DEV)
    hw = torch.tensor(eo.LEVEL_HW[:L], dtype=torch.int64, device=DEV)
    return raw, ref2d, hw


@pytest.mark.parametrize("c", eo.tsa_cases(), ids=eo.tsa_case_id)
def test_tsa_prep(c):
    """bevf_tsa_prep_forward / _backward against the TSA restatement (temporal_self_attention.py:206-229).

    loc: 2u (|offset / W| + |loc|); attn: the softmax bar of _softmax_bar.  d_raw: offsets g / (W or H) are one
    correctly rounded division (u, doubled); the logits' a (ga - sum a ga) is bounded by
    (3 LP + 12 + 4 max|l - max|) u a (|ga| + sum a |ga|) (a's own bar, the dot's LP-term sum and the subtract), plus
    one storage ulp in 16-bit.  Outputs are NaN-prefilled and must be fully written."""
    M, L, P, B, Nq, il = c["M"], c["L"], c["P"], c["B"], c["Nq"], c["interleave"]
    LP = L * P
    out_dt = DT[c["dt"]]
    raw, ref2d, hw = _tsa_inputs(c, 31)
    shape = (B * Nq * 2, M, L, P) if il else (B * 2, Nq, M, L, P)
    loc = torch.full(shape + (2,), NAN, device=DEV)
    attn = torch.full(shape, NAN, device=DEV)
    lib = _lib.load()
    m8 = M == 8 and LP in (2, 4, 8, 16, 32)

    def fwd():
        _check(lib.bevf_tsa_prep_forward(raw.data_ptr(), ref2d.data_ptr(), hw.data_ptr(), loc.data_ptr(),
                                         attn.data_ptr(), B, Nq, M, L, P, il, _st()))
    g = torch.Generator().manual_seed(37)
    gl = torch.randn(loc.shape, generator=g).to(DEV)
    ga = torch.randn(attn.shape, generator=g).to(DEV)
    d_raw = torch.full(raw.shape, NAN, device=DEV, dtype=out_dt)

    def bwd():
        _check(lib.bevf_tsa_prep_backward(raw.data_ptr(), gl.data_ptr(), ga.data_ptr(), hw.data_ptr(),
                                          d_raw.data_ptr(), ops._DT[out_dt], B, Nq, M, L, P, il, _st()))
    ran(lambda: (fwd(), bwd()), f"bevf::tsa_prep_m8<{LP // 2}, false, float>" if m8 else "bevf::tsa_prep_fwd(",
        f"bevf::tsa_prep_m8<{LP // 2}, true, {CNAME[c['dt']]}>" if m8 else f"bevf::tsa_prep_bwd<{CNAME[c['dt']]}>")
    wl, wa = eo.tsa_prep_forward(raw, ref2d, hw, B, Nq, M, L, P, interleave=bool(il))
    ow = eo.tsa_prep_forward(raw, ref2d * 0, hw, B, Nq, M, L, P, interleave=bool(il))[0]      # offset / (W, H) alone
    assert_within(loc, wl, _prep_loc_bar(ow, wl), "loc")
    abar = _softmax_bar(raw[:, M * 2 * LP * 2:], LP)          # (B*Nq*M*2, LP) in raw's (b, q, m, j) order
    abar = abar.reshape(B, Nq, M, 2, L, P)
    abar = abar.permute(0, 1, 3, 2, 4, 5) if il else abar.permute(0, 3, 1, 2, 4, 5)
    assert_within(attn, wa, abar.reshape(wa.shape) * wa, "attn")
    want = eo.tsa_prep_backward(raw, ref2d, hw, gl, ga, B, Nq, M, L, P, interleave=bool(il))
    n_off = M * 2 * LP * 2
    # logits part: per (b, q, m, j) group in raw's order; gather ga into that order
    ga_r = ga.to(F64).reshape(B, Nq, 2, M, LP) if il else ga.to(F64).reshape(B, 2, Nq, M, LP).transpose(1, 2)
    ga_r = ga_r.transpose(2, 3).reshape(-1, LP)                       # (b, q, m, j) rows
    a_r = wa.reshape(B, Nq, 2, M, LP) if il else wa.reshape(B, 2, Nq, M, LP).transpose(1, 2)
    a_r = a_r.transpose(2, 3).reshape(-1, LP)
    lg = raw[:, n_off:].to(F64).reshape(-1, LP)
    dev = (lg.max(-1, keepdim=True).values - lg).max(-1, keepdim=True).values
    bar_lg = (3 * LP + 12 + 4 * dev) * U * a_r * (ga_r.abs() + (a_r * ga_r.abs()).sum(-1, keepdim=True))
    bar = torch.empty_like(want)
    bar[:, n_off:] = bar_lg.reshape(B * Nq, -1)
    bar[:, :n_off] = 2 * U * want[:, :n_off].abs()
    assert_within(d_raw, want, _drawbar(want, out_dt, bar), "d_raw")


def _sca_setup(c, seed):
    M, L, P, D, ncam, B, Nq = c["M"], c["L"], c["P"], c["D"], c["ncam"], c["B"], c["Nq"]
    g = torch.Generator().manual_seed(seed)
    pq, pc, pair_of = eo.make_pairs(Nq, ncam, seed=seed)
    raw = (torch.randn(B * Nq, M * L * P * 3, generator=g) * 2).to(DEV)
    ref_cam = torch.rand(ncam, B, Nq, D, 2, generator=g).to(DEV)
    hw = torch.tensor(eo.LEVEL_HW[:L], dtype=torch.int64, device=DEV)
    return raw, ref_cam, hw, pq.to(DEV), pc.to(DEV), pair_of.to(DEV)


def _sca_logit_bar(raw, ga_rows, pq, B, Nq, M, LP):
    """Bar of the logits part of the SCA d_raw: the per-camera gradients are summed first (n - 1 adds, n <= 16: 16 u
    of the magnitude sum), then the TSA bound of test_tsa_prep applies to the summed gradient."""
    R = pq.numel()
    valid = pq.long() >= 0
    n_off = M * LP * 2
    gsum_abs = torch.zeros(B, Nq, M, LP, dtype=F64, device=DEV)
    gsum_abs.index_add_(1, pq.long()[valid], ga_rows.to(F64).abs().reshape(B, R, M, LP)[:, valid])
    lg = raw[:, n_off:].to(F64).reshape(B, Nq, M, LP)
    a = torch.softmax(lg, -1)
    dev = (lg.max(-1, keepdim=True).values - lg).max(-1, keepdim=True).values
    return ((3 * LP + 28 + 4 * dev) * U * a * (gsum_abs + (a * gsum_abs).sum(-1, keepdim=True))).reshape(B * Nq, -1)


def _sca_off_abs_bar(gl, pq, B, Nq, M, L, P, hw):
    """Offsets part of the SCA d_raw: sum over cameras of g (16 u of sum |g|), then one division."""
    R = pq.numel()
    valid = pq.long() >= 0
    s = torch.zeros(B, Nq, M, L, P, 2, dtype=F64, device=DEV)
    s.index_add_(1, pq.long()[valid], gl.to(F64).abs().reshape(B, R, M, L, P, 2)[:, valid])
    wh = torch.stack([hw[:, 1], hw[:, 0]], -1).to(F64)
    return (2 * 17 * U * s / wh[:, None, :]).reshape(B * Nq, -1)


@pytest.mark.parametrize("c", eo.sca_cases(), ids=eo.sca_case_id)
def test_sca_prep(c):
    """bevf_sca_prep_forward / _backward against the SCA restatement (spatial_cross_attention.py:338-372) on a
    hand-built pair list: queries seen by 0, 1, 2, 3 and all cameras, padding rows at the end.

    loc / attn: the bars of test_tsa_prep.  Padding rows of loc / attn stay NaN; every other row is written.
    d_raw: the per-camera gradients are summed (at most 16 terms: 16 u of the magnitude sum) before the TSA bound
    applies; queries no camera sees get exact zeros."""
    M, L, P, D, ncam, B, Nq = c["M"], c["L"], c["P"], c["D"], c["ncam"], c["B"], c["Nq"]
    LP = L * P
    out_dt = DT[c["dt"]]
    raw, ref_cam, hw, pq, pc, pair_of = _sca_setup(c, 41)
    R = pq.numel()
    loc = torch.full((B * R, M, L, P, 2), NAN, device=DEV)
    attn = torch.full((B * R, M, L, P), NAN, device=DEV)
    lib = _lib.load()
    m8 = M == 8 and LP in (4, 8, 16, 32, 64)

    def fwd():
        _check(lib.bevf_sca_prep_forward(raw.data_ptr(), ref_cam.data_ptr(), pq.data_ptr(), pc.data_ptr(),
                                         hw.data_ptr(), loc.data_ptr(), attn.data_ptr(), B, Nq, R, M, L, P, D, ncam,
                                         _st()))
    g = torch.Generator().manual_seed(43)
    gl = torch.randn(loc.shape, generator=g).to(DEV)
    ga = torch.randn(attn.shape, generator=g).to(DEV)
    d_raw = torch.full(raw.shape, NAN, device=DEV, dtype=out_dt)

    def bwd():
        _check(lib.bevf_sca_prep_backward(raw.data_ptr(), gl.data_ptr(), ga.data_ptr(), pair_of.data_ptr(),
                                          hw.data_ptr(), d_raw.data_ptr(), ops._DT[out_dt], B, Nq, R, M, L, P, ncam,
                                          _st()))
    ran(lambda: (fwd(), bwd()), f"bevf::sca_prep_fwd_m8<{LP // 4}>" if m8 else "bevf::sca_prep_fwd(",
        f"bevf::sca_prep_bwd_m8<{LP // 4}, {CNAME[c['dt']]}, false>" if m8 else f"bevf::sca_prep_bwd<{CNAME[c['dt']]}>")
    wl, wa, valid = eo.sca_prep_forward(raw, ref_cam, pq, pc, hw, B, Nq, M, L, P)
    v = valid.repeat(B)
    assert torch.isnan(loc[~v]).all() and torch.isnan(attn[~v]).all(), "padding rows were written"
    wl0 = eo.sca_prep_forward(raw, ref_cam * 0, pq, pc, hw, B, Nq, M, L, P)[0]       # offset / (W, H) alone
    assert_within(loc[v], wl[v], _prep_loc_bar(wl0[v], wl[v]), "loc")
    q = pq.long().clamp(min=0)
    lg_rows = raw.reshape(B, Nq, -1)[:, q, M * LP * 2:].reshape(B * R, M * LP)[v]
    assert_within(attn[v], wa[v], _softmax_bar(lg_rows, LP).reshape(wa[v].shape) * wa[v], "attn")
    want = eo.sca_prep_backward(raw, ref_cam, pq, pc, hw, gl, ga, B, Nq, M, L, P)
    bar = torch.cat([_sca_off_abs_bar(gl, pq, B, Nq, M, L, P, hw), _sca_logit_bar(raw, ga, pq, B, Nq, M, LP)], -1)
    assert_within(d_raw, want, _drawbar(want, out_dt, bar), "d_raw")
    unseen = (pair_of < 0).all(0)
    assert unseen.any() and (d_raw.reshape(B, Nq, -1)[:, unseen] == 0).all()


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("L,P", [(4, 8), (1, 32)])
def test_sca_prep_backward_multi(dt, L, P):
    """bevf_sca_prep_backward_multi (the finish kernel of the fused sampler's backward) leaves the d_raw rows of
    queries seen by exactly one camera untouched and writes every other row bit for bit like bevf_sca_prep_backward."""
    c = dict(M=8, L=L, P=P, D=4, ncam=16, B=3, Nq=45, dt=dt)
    M, B, Nq, ncam = 8, 3, 45, 16
    out_dt = DT[dt]
    raw, ref_cam, hw, pq, pc, pair_of = _sca_setup(c, 47)
    R = pq.numel()
    g = torch.Generator().manual_seed(53)
    gl = torch.randn(B * R, M, L, P, 2, generator=g).to(DEV)
    ga = torch.randn(B * R, M, L, P, generator=g).to(DEV)
    lib = _lib.load()
    full = torch.full(raw.shape, NAN, device=DEV, dtype=out_dt)
    multi = torch.full(raw.shape, NAN, device=DEV, dtype=out_dt)
    _check(lib.bevf_sca_prep_backward(raw.data_ptr(), gl.data_ptr(), ga.data_ptr(), pair_of.data_ptr(), hw.data_ptr(),
                                      full.data_ptr(), ops._DT[out_dt], B, Nq, R, M, L, P, ncam, _st()))

    def run():
        _check(lib.bevf_sca_prep_backward_multi(raw.data_ptr(), gl.data_ptr(), ga.data_ptr(), pair_of.data_ptr(),
                                                hw.data_ptr(), multi.data_ptr(), ops._DT[out_dt], B, Nq, R, M, L, P,
                                                ncam, _st()))
    ran(run, f"bevf::sca_prep_bwd_m8<8, {CNAME[dt]}, true>")
    one = ((pair_of >= 0).sum(0) == 1)
    m = multi.reshape(B, Nq, -1)
    assert one.any() and (~one).any()
    assert torch.isnan(m[:, one]).all(), "rows of one-camera queries were written"
    f = full.reshape(B, Nq, -1)
    assert torch.equal(m[:, ~one].view(torch.int16), f[:, ~one].view(torch.int16))


# ------------------------------------------------------------------------------------------------
# SCA combine
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", eo.combine_cases(), ids=eo.combine_case_id)
def test_sca_combine(c):
    """ops.ScaCombine forward and backward against spatial_cross_attention.py:165-172.

    Forward: at most 16 adds of the camera rows and one multiply by the fp32 1/count (itself within u/2):
    (ncam + 2) u sum|rows| / count, plus one storage ulp in 16-bit.  Backward: one multiply, u |g| / count, plus
    one storage ulp; padding rows are left as they were (NaN prefill, through the C entry point)."""
    dt, C, ncam, B, Nq = DT[c["dt"]], c["C"], c["ncam"], c["B"], c["Nq"]
    pq, pc, pair_of = (t.to(DEV) for t in eo.make_pairs(Nq, ncam, seed=59))
    R = pq.numel()
    cnt = eo.camera_count(pq, Nq).clamp(min=1)
    inv = (1.0 / cnt).to(torch.float32)[None].expand(B, Nq).contiguous()
    g = torch.Generator().manual_seed(61)
    out = torch.randn(B * R, C, generator=g).to(DEV, dt).requires_grad_(True)
    gs = torch.randn(B, Nq, C, generator=g).to(DEV, dt)

    def run():
        slots = ops.ScaCombine.apply(out, pair_of, pq, inv, B, Nq)
        return slots, torch.autograd.grad(slots, out, gs)[0]
    slots, got = ran(run, f"bevf::sca_combine_fwd<{CNAME[c['dt']]}>", f"bevf::sca_combine_bwd<{CNAME[c['dt']]}>")
    want = eo.sca_combine_forward(out.detach(), pq, B, Nq)
    mag = eo.sca_combine_forward(out.detach().abs(), pq, B, Nq)
    ul = (lambda r: eo.ulp(r, dt)) if dt != torch.float32 else (lambda r: torch.zeros_like(r))
    assert_within(slots.detach(), want, (ncam + 2) * U * mag + ul(want), "slots")
    wg = eo.sca_combine_backward(gs, pq, B, Nq)
    valid = (pq.long() >= 0).repeat(B)
    assert_within(got[valid], wg[valid], 2 * U * wg[valid].abs() + ul(wg[valid]), "g_out")
    # the padding rows of a caller-owned buffer are not written
    g_out = torch.full((B * R, C), NAN, device=DEV, dtype=dt)
    _check(_lib.load().bevf_sca_combine_backward(gs.data_ptr(), pq.data_ptr(), inv.data_ptr(), g_out.data_ptr(), B,
                                                 Nq, R, C, ops._DT[dt], _st()))
    assert torch.isnan(g_out[~valid]).all() and torch.equal(g_out[valid], got[valid])


# ------------------------------------------------------------------------------------------------
# colsum, sum_tensors, dropout
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", eo.colsum_cases(), ids=eo.colsum_case_id)
def test_colsum(c):
    """bevf_colsum / bevf_colsum_det into a caller buffer (zero or, with -acc, non-zero).

    A thread sums its rows of a CTA (rpc / rstep, in groups of 4), rstep row lanes meet in shared memory, the CTAs
    meet through atomics or, deterministic, in CTA order: (rpc + rstep + CTAs + 4) u (sum|x| + |out|) per column,
    rstep = 256 / (C / vec) row lanes.  The deterministic form is also bitwise repeatable."""
    C, dt = c["C"], DT[c["dt"]]
    rows = eo.colsum_rows(c["rows"], sms())
    g = torch.Generator().manual_seed(67)
    x = torch.randn(rows, C, generator=g).to(DEV, dt)
    out0 = torch.randn(C, generator=g).to(DEV) if c["acc"] else torch.zeros(C, device=DEV)
    lib = _lib.load()

    def run():
        out = out0.clone()
        if c["det"]:
            need = int(lib.bevf_colsum_workspace_bytes(rows, C))
            ws = torch.full((need // 4,), NAN, device=DEV)
            _check(lib.bevf_colsum_det(x.data_ptr(), out.data_ptr(), ws.data_ptr(), need, rows, C, ops._DT[dt], _st()))
        else:
            _check(lib.bevf_colsum(x.data_ptr(), out.data_ptr(), rows, C, ops._DT[dt], _st()))
        return out
    out = ran(run, f"bevf::colsum_kernel<{CNAME[c['dt']]}>", *(["bevf::partials_add_kernel"] if c["det"] else []))
    want, mag = eo.colsum(x, out0)
    rpc, grid = eo.colsum_plan(rows, sms())
    if c["rows"] == "cta+1":
        assert rows == (grid - 1) * rpc + 1
    vec = 4 if dt == torch.float32 else 8
    rstep = 256 // (C // vec)
    assert_within(out, want, (rpc / rstep + rstep + grid + 4) * U * mag, "colsum")
    if c["det"]:
        assert torch.equal(run(), out)


@pytest.mark.parametrize("c", eo.sum_cases(), ids=eo.sum_case_id)
def test_sum_tensors(c):
    """bevf_sum_tensors (n = 1 through the C entry point: the ops wrapper returns its input unchanged).
    n - 1 fp32 adds: (n - 1) u sum|x_k|, plus one storage ulp in 16-bit; n = 1 is an exact copy."""
    n, dt, numel = c["n"], DT[c["dt"]], c["numel"]
    g = torch.Generator().manual_seed(71)
    ts = [torch.randn(numel, generator=g).to(DEV, dt) for _ in range(n)]
    out = torch.full((numel,), NAN, device=DEV, dtype=dt)
    arr = (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts])

    def run():
        _check(_lib.load().bevf_sum_tensors(ctypes.addressof(arr), n, out.data_ptr(), numel, ops._DT[dt], _st()))
    ran(run, f"sum_n_kernel<{CNAME[c['dt']]}>(")
    want, mag = eo.sum_tensors(ts)
    if n == 1:
        assert torch.equal(out, ts[0])
        return
    ul = eo.ulp(want, dt) if dt != torch.float32 else torch.zeros_like(want)
    assert_within(out, want, (n - 1) * U * mag + ul, "sum")
    if n > 1:
        assert torch.equal(ops.sum_tensors(ts), out)


@pytest.mark.parametrize("c", eo.dropout_cases(), ids=eo.dropout_case_id)
def test_dropout_and_relu_dropout_backward(c):
    """ops.dropout_inplace_: the drop count within 6 sigma of the binomial mean, dropped values exact zeros, kept
    values exactly x * fl32(1 / (1 - p)) rounded to storage.  ops.relu_dropout_backward on that h: exactly
    dy * fl32(1 / (1 - p)) where h != 0 and 0 elsewhere, i.e. the same mask and the same scale as the forward."""
    dt, p, numel = DT[c["dt"]], c["p"], c["numel"]
    g = torch.Generator().manual_seed(73)
    x = torch.randn(numel, generator=g).to(DEV, dt)
    x[x == 0] = 1.0                                   # a zero input would hide the mask
    dy = torch.randn(numel, generator=g).to(DEV, dt)

    def run():
        h = ops.dropout_inplace_(x.clone(), p)
        return h, ops.relu_dropout_backward(dy, h, p)
    h, dz = ran(run, f"bevf::dropout_inplace_kernel<{CNAME[c['dt']]}>", f"bevf::relu_dropout_bwd_kernel<{CNAME[c['dt']]}>")
    keep = h != 0
    dropped = int((~keep).sum())
    assert abs(dropped - numel * p) <= eo.binomial_bound(numel, p), (dropped, numel * p)
    s32 = eo.dropout_scale32(p)
    assert torch.equal(h[keep], eo.dropout_kept(x[keep], s32))
    assert torch.equal(dz, eo.relu_dropout_backward(dy, h, s32))
    assert torch.equal(dz != 0, keep & (dy != 0))


def test_relu_dropout_backward_refuses_noncontiguous_h():
    """h's pointer is read as a dense tensor of dy's size: a strided h, or one of another size, is refused."""
    dy = torch.randn(64, 256, device=DEV)
    h = torch.randn(256, 64, device=DEV).t()
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.relu_dropout_backward(dy, h, 0.3)
    with pytest.raises(RuntimeError, match="size"):
        ops.relu_dropout_backward(dy, torch.randn(32, 256, device=DEV), 0.3)
