"""The sampler kernels (csrc/msda.cu, msda_splat.cuh, msda_dense.cu, gv16.cu, gvfx.cu) against the float64
restatement of tests/msda_fp64_oracle.py, on every dispatch branch, element by element.

Each case calls the C entry point through _lib with its outputs prefilled with NaN (grad_value, which the entry points
accumulate into, with zeros), so that both "every live element written" and "unused rows left untouched" are checked;
the restatement runs on the device in float64 on the same storage-rounded inputs.  Every element of every output must
lie within the bar of its arithmetic path (the ``bar_*`` functions of the oracle module derive them); no bar is
normalised by max|ref|, no element is excused.  Each case reports its worst err / bar ratio per output as a ``Slack`` warning (listed in pytest's warnings
summary) and on stdout.

Which kernel each case runs is asserted through torch.profiler kernel names in a child process
(test_every_case_runs_its_instantiation reruns this file there with ENV_PROFILE set; the first case of each
instantiation launches under the profiler and every case stops before its numeric checks).  Hundreds of profiler
sessions leave CUPTI in a state where later sessions of the same process drop GPU activity records, which would break
the kernel-inventory tests of other files; the numeric checks in this process run without the profiler."""
import ctypes
import math
import os
import subprocess
import sys
import warnings

import pytest
import torch

from bevformer_b200 import _lib, ops
from tests import msda_fp64_oracle as mo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F64 = torch.float64
NAN = float("nan")
DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
CNAME = {"f32": "float", "bf16": "__nv_bfloat16", "f16": "__half"}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")]
ENV_PROFILE = "BEVF_MSDA_FP64_PROFILE"
PROFILING = os.environ.get(ENV_PROFILE) == "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------
# profiler plumbing (see the module docstring)
# ------------------------------------------------------------------------------------------------
def kernels(fn, attempts=6):
    """Run fn under the profiler; returns (fn's result, set of CUDA kernel names that ran).  An exp kernel before fn
    and a sqrt kernel after it bracket the window: a trace without both lost records, and fn runs again."""
    import time
    from torch.profiler import ProfilerActivity, profile
    names = set()
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


_VERIFIED = set()


def ran(fn, *expected, tag=None):
    """fn().  In the profiling child: fn() under the profiler, asserting that every kernel name substring in
    ``expected`` launched, then the case ends (its numeric checks run in the parent).  Once per distinct (expected,
    tag): the tag names what else selects the dispatch (shape, layout, mode), so that every such case is confirmed on
    its own while repeats that differ only in values are not profiled again."""
    if not PROFILING:
        return fn()
    key = (expected, tag)
    if key not in _VERIFIED:
        _, names = kernels(fn)
        for s in expected:
            assert any(s in n for n in names), (s, sorted(n[:120] for n in names))
        _VERIFIED.add(key)
    pytest.skip("dispatch checked")


def test_every_case_runs_its_instantiation():
    """Every case of this file, rerun in a child process under the profiler, launches the instantiations it names."""
    if PROFILING:
        pytest.skip("this is the profiling run")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider",
                        "-k", "not test_every_case_runs_its_instantiation and not refuses and not splat_direct_env"],
                       cwd=ROOT, env=dict(os.environ, **{ENV_PROFILE: "1"}), capture_output=True, text=True,
                       timeout=1200)
    tail = r.stdout[-6000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    last = [ln for ln in r.stdout.splitlines() if ln.strip()][-1]
    assert "skipped" in last and "passed" not in last and "failed" not in last, tail


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
def _lib_():
    return _lib.load()


def _st():
    return torch.cuda.current_stream(DEV).cuda_stream


def _check(st):
    _lib.check(st, _lib_())


def within(got, ref, bar, what, report):
    """|got - ref| <= bar for every element (got in its storage type, ref / bar float64); NaN fails.  Records the
    worst err / bar in ``report``."""
    err = (got.to(F64) - ref).abs()
    ratio = torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(err), math.inf, ratio)
    worst = ratio.max().item() if ratio.numel() else 0.0
    report[what] = worst
    if not worst <= 1.0:
        bad = ~(ratio <= 1.0)
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bar; first at {i}: got "
                             f"{got.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r} bar "
                             f"{bar.flatten()[i].item():.3g}; worst err/bar {worst:.3g}")


def untouched(t, what):
    """Rows of unused entries still hold the NaN prefill, bit for bit."""
    if t.numel():
        assert torch.isnan(t).all(), f"{what}: an unused row was written"


class Slack(UserWarning):
    """The worst err / bar of a case, one per case: pytest lists them in its warnings summary."""


def show(case, report):
    msg = f"[msda_fp64] {case}: " + ", ".join(f"{k} {v:.3g}" for k, v in report.items())
    print(msg)
    warnings.warn(msg, Slack)


def case_inputs(shape, vdt, godt=None, seed=0, D=32, gscale=1.0, **kw):
    """Device tensors of one case: value / grad_out in their storage types, level tables, loc / attn in fp32."""
    s = dict(mo.SHAPES[shape]) if isinstance(shape, str) else dict(shape)
    d = mo.make_inputs(D=D, seed=seed, gscale=gscale, **s, **kw)
    c = dict(value=d["value"].to(DEV, DT[vdt]).contiguous(), hw=d["level_hw"].to(DEV), ls=d["level_start"].to(DEV),
             loc=d["loc"].to(DEV), attn=d["attn"].to(DEV),
             row_map=None if d["row_map"] is None else d["row_map"].to(DEV),
             grad_out=d["grad_out"].to(DEV, DT[godt or vdt]).contiguous())
    NB, S, M, D = c["value"].shape
    L, P = c["attn"].shape[-2:]
    rows = c["loc"].shape[0] if c["row_map"] is not None else c["loc"].shape[0] * c["loc"].shape[1]
    c.update(NB=NB, S=S, M=M, D=D, L=L, P=P, Q=c["loc"].shape[0] if c["row_map"] is not None else c["loc"].shape[1],
             rows=rows, hw_host=[tuple(int(x) for x in r) for r in d["level_hw"].tolist()])
    c["dead"] = (c["row_map"] < 0) if c["row_map"] is not None else torch.zeros(rows, dtype=torch.bool, device=DEV)
    return c


def _dims(c):
    return (c["NB"], c["S"], c["M"], c["D"], c["Q"], c["L"], c["P"])


def _hw_host(c):
    return (ctypes.c_int32 * (2 * c["L"]))(*[v for hw in c["hw_host"] for v in hw])


def _backward_bufs(c):
    gl = torch.full(c["loc"].shape, NAN, device=DEV)
    ga = torch.full(c["attn"].shape, NAN, device=DEV)
    return gl, ga


def _check_loc_attn(c, gl, ga, r, report):
    D = c["D"]
    live = ~c["dead"]
    glr, gar = gl.reshape(c["rows"], -1), ga.reshape(c["rows"], -1)
    within(glr[live], r["grad_loc"].reshape(c["rows"], -1)[live], mo.bar_grad_loc(r["gl_mag"], D).reshape(c["rows"], -1)[live],
           "grad_loc", report)
    within(gar[live], r["grad_attn"].reshape(c["rows"], -1)[live],
           mo.bar_grad_attn(r["ga_mag"], D).reshape(c["rows"], -1)[live], "grad_attn", report)
    untouched(glr[c["dead"]], "grad_loc")
    untouched(gar[c["dead"]], "grad_attn")


def _ref_backward(c, **kw):
    return mo.backward(c["value"], c["hw"], c["ls"], c["loc"], c["attn"], c["grad_out"], c["row_map"], **kw)


# ------------------------------------------------------------------------------------------------
# forward: msda_fwd_d32<T, TO, false> (head_dim 32) and msda_fwd_generic<T, TO>
# ------------------------------------------------------------------------------------------------
def _forward_case(c, vdt, odt):
    lib = _lib_()
    out = torch.full((c["rows"], c["M"] * c["D"]), NAN, device=DEV, dtype=DT[odt])
    common = (c["value"].data_ptr(), ops._DT[DT[vdt]], c["hw"].data_ptr(), c["ls"].data_ptr(), c["loc"].data_ptr(),
              c["attn"].data_ptr(), out.data_ptr(), ops._DT[DT[odt]])

    def run():
        if c["row_map"] is not None:
            _check(lib.bevf_msda_rows_forward(*common, c["row_map"].data_ptr(), *_dims(c), _st()))
        else:
            _check(lib.bevf_msda_forward(*common, *_dims(c), _st()))
    return out, run


def _forward_check(case, c, vdt, odt, out):
    ref, mag = mo.forward(c["value"], c["hw"], c["ls"], c["loc"], c["attn"], c["row_map"])
    ref, mag = ref.reshape(c["rows"], -1), mag.reshape(c["rows"], -1)
    bar = mo.bar_forward(mag, ref, c["L"] * c["P"], DT[odt], packed_bf16_weights=(vdt == "bf16" and c["D"] == 32))
    live = ~c["dead"]
    report = {}
    within(out[live], ref[live], bar[live], "out", report)
    untouched(out[c["dead"]].float(), "out")
    show(case, report)


@pytest.mark.parametrize("shape", list(mo.SHAPES))
@pytest.mark.parametrize("vdt,odt", PAIRS)
def test_forward_d32(shape, vdt, odt):
    c = case_inputs(shape, vdt, seed=1)
    out, run = _forward_case(c, vdt, odt)
    ran(run, f"msda_fwd_d32<{CNAME[vdt]}, {CNAME[odt]}, false>", tag=shape)
    torch.cuda.synchronize()
    _forward_check(f"fwd_d32 {shape} {vdt}->{odt}", c, vdt, odt, out)


GENERIC = {4: "rows_m5", 30: "dense_edges", 64: "rows_m1", 71: "dense_edges"}


@pytest.mark.parametrize("D", list(GENERIC))
@pytest.mark.parametrize("vdt,odt", PAIRS)
def test_forward_generic(D, vdt, odt):
    c = case_inputs(GENERIC[D], vdt, seed=2, D=D)
    out, run = _forward_case(c, vdt, odt)
    ran(run, f"msda_fwd_generic<{CNAME[vdt]}, {CNAME[odt]}>", tag=D)
    torch.cuda.synchronize()
    _forward_check(f"fwd_generic D={D} {vdt}->{odt}", c, vdt, odt, out)


def test_forward_refuses_magic_overflow():
    """L P^2 = 65536 is refused before any launch (level_of's magic division would no longer be exact)."""
    c = case_inputs("magic_max", "f32", seed=3)
    lib = _lib_()
    out = torch.full((c["rows"], 32), NAN, device=DEV)
    NB, S, M, D, Q, L, P = _dims(c)
    loc = torch.zeros(NB, Q, M, 1, 256, 2, device=DEV)
    attn = torch.zeros(NB, Q, M, 1, 256, device=DEV)
    st = lib.bevf_msda_forward(c["value"].data_ptr(), ops._DT[torch.float32], c["hw"].data_ptr(), c["ls"].data_ptr(),
                               loc.data_ptr(), attn.data_ptr(), out.data_ptr(), ops._DT[torch.float32],
                               NB, S, M, D, Q, 1, 256, _st())
    assert st != 0
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


# ------------------------------------------------------------------------------------------------
# backward with fp32 grad_value: one kernel, generic, split / hybrid
# ------------------------------------------------------------------------------------------------
def _backward_case(c, vdt, godt, order=None):
    lib = _lib_()
    gv = torch.zeros(c["value"].shape, device=DEV)
    gl, ga = _backward_bufs(c)
    common = (c["value"].data_ptr(), ops._DT[DT[vdt]], c["hw"].data_ptr(), c["ls"].data_ptr(), c["loc"].data_ptr(),
              c["attn"].data_ptr(), c["grad_out"].data_ptr(), ops._DT[DT[godt]], gv.data_ptr(), gl.data_ptr(),
              ga.data_ptr())

    def run():
        gv.zero_()
        if c["row_map"] is not None:
            _check(lib.bevf_msda_rows_backward_ordered(*common, c["row_map"].data_ptr(),
                                                       None if order is None else order.data_ptr(), *_dims(c), _st()))
        else:
            _check(lib.bevf_msda_backward(*common, *_dims(c), _st()))
    return gv, gl, ga, run


def _backward_check(case, c, gv, gl, ga):
    r = _ref_backward(c)
    report = {}
    within(gv, r["grad_value"], mo.bar_grad_value_f32(r["gv_mag"], r["gv_count"]), "grad_value", report)
    _check_loc_attn(c, gl, ga, r, report)
    show(case, report)


@pytest.mark.parametrize("shape", list(mo.SHAPES))
@pytest.mark.parametrize("vdt,godt", PAIRS)
def test_backward_one_kernel(shape, vdt, godt):
    c = case_inputs(shape, vdt, godt, seed=4)
    gv, gl, ga, run = _backward_case(c, vdt, godt)
    ran(run, f"msda_bwd_d32<{CNAME[vdt]}, {CNAME[godt]}, true, float", tag=shape)
    torch.cuda.synchronize()
    _backward_check(f"bwd_d32 {shape} {vdt}/{godt}", c, gv, gl, ga)


@pytest.mark.parametrize("D", list(GENERIC))
@pytest.mark.parametrize("vdt,godt", PAIRS)
def test_backward_generic(D, vdt, godt):
    c = case_inputs(GENERIC[D], vdt, godt, seed=5, D=D)
    gv, gl, ga, run = _backward_case(c, vdt, godt)
    ran(run, f"msda_bwd_generic<{CNAME[vdt]}, {CNAME[godt]}, float>", tag=D)
    torch.cuda.synchronize()
    _backward_check(f"bwd_generic D={D} {vdt}/{godt}", c, gv, gl, ga)


@pytest.fixture
def bwd_mode():
    lib = _lib_()
    yield lambda m: _check(lib.bevf_msda_set_backward_mode(m))
    _check(lib.bevf_msda_set_backward_mode(0))


@pytest.mark.parametrize("shape", ["rows_m8", "rows_m5", "rows_m16", "dense_edges"])
@pytest.mark.parametrize("vdt,godt", [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32")])
@pytest.mark.parametrize("mode", [1, 2])
def test_backward_split_hybrid(shape, vdt, godt, mode, bwd_mode):
    """Mode 1 (split): msda_bwd_splat_d32 takes every level's grad_value, msda_bwd_d32<..., false> the rest.  Mode 2
    (hybrid): the splat kernel takes the coarse half on the second stream.  M > 8 (rows_m16) falls back to mode 0;
    the row list runs with a group_order permutation."""
    c = case_inputs(shape, vdt, godt, seed=6)
    order = None
    if c["row_map"] is not None:
        order = torch.randperm(c["Q"], generator=torch.Generator().manual_seed(6)).to(DEV, torch.int32)
    gv, gl, ga, run = _backward_case(c, vdt, godt, order)
    bwd_mode(mode)
    M, L = c["M"], c["L"]
    tg = CNAME[godt]
    if M > 8:
        names = (f"msda_bwd_d32<{CNAME[vdt]}, {tg}, true, float",)
    else:
        names = (f"msda_bwd_splat_d32<{tg}, {8 if M == 8 else 0}>",)
        names += (f"msda_bwd_d32<{CNAME[vdt]}, {tg}, {'false' if mode == 1 else 'true'}, float",)
        if mode == 2 and L < 2:
            names = (f"msda_bwd_d32<{CNAME[vdt]}, {tg}, true, float",)
    ran(run, *names, tag=(shape, mode))
    torch.cuda.synchronize()
    _backward_check(f"bwd mode {mode} {shape} {vdt}/{godt}", c, gv, gl, ga)


SPLAT = {
    "clustered": dict(cluster=(0.3, 0.08), border_frac=0.0),      # every slice fits one window pass
    "wide": dict(cluster=(0.3, 0.2), border_frac=0.0),            # level 0 takes several passes
    "uniform": dict(border_frac=0.05),                            # more than kSplatMaxPasses: the direct branch
}
SPLAT_G, SPLAT_WX, SPLAT_WY, SPLAT_MAX_PASSES = 64, 10, 5, 8     # msda_splat.cuh: kSplatG, kWX, kWY, kSplatMaxPasses


def splat_branches(c):
    """How many (CTA, head, level, point, value map) slices of msda_bwd_splat_d32 take one window pass, several, or
    the direct branch: the kernel sweeps the bounding box of the valid samples' top-left cells in kWX x kWY windows and
    goes direct above kSplatMaxPasses of them (the rows of a CTA are kSplatG consecutive rows: no group order)."""
    loc, rm, hw = c["loc"], c["row_map"].long(), c["hw"]
    R, M, L, P, _ = loc.shape
    x, y, valid = mo._coords(loc, hw)
    x0, y0 = torch.floor(x).long(), torch.floor(y).long()
    valid = valid & (rm >= 0).view(-1, 1, 1, 1)
    dev = loc.device
    ar = lambda n, sh: torch.arange(n, device=dev).view(sh)
    key = ((((ar(R, (-1, 1, 1, 1)) // SPLAT_G * M + ar(M, (1, -1, 1, 1))) * L + ar(L, (1, 1, -1, 1))) * P
            + ar(P, (1, 1, 1, -1))) * c["NB"] + rm.clamp(min=0).view(-1, 1, 1, 1))
    k, n, big = key[valid], int(key.max()) + 1, 1 << 30

    def red(v, op, init):
        return torch.full((n,), init, dtype=torch.long, device=dev).scatter_reduce(0, k, v[valid], op)
    mnx, mxx, mny, mxy = red(x0, "amin", big), red(x0, "amax", -big), red(y0, "amin", big), red(y0, "amax", -big)
    used = mnx < big
    npass = (((mxx - mnx) // SPLAT_WX + 1) * ((mxy - mny) // SPLAT_WY + 1))[used]
    return dict(one=int((npass == 1).sum()), several=int(((npass > 1) & (npass <= SPLAT_MAX_PASSES)).sum()),
                direct=int((npass > SPLAT_MAX_PASSES).sum()))


@pytest.mark.parametrize("which", list(SPLAT))
@pytest.mark.parametrize("godt", ["f32", "bf16"])
def test_splat_branches(which, godt, bwd_mode):
    shape = dict(levels=[(40, 60), (20, 30), (10, 15)], M=8, P=4, NB=2, R=640, unused=(5, 200))
    vdt = "bf16" if godt == "bf16" else "f32"
    c = case_inputs(shape, vdt, godt, seed=7, **SPLAT[which])
    br = splat_branches(c)
    total = sum(br.values())
    if which == "clustered":
        assert br["one"] == total, br
    elif which == "wide":
        assert br["several"] >= total // 3 and br["direct"] == 0, br
    else:
        assert br["direct"] >= total // 2, br
    gv, gl, ga, run = _backward_case(c, vdt, godt)
    bwd_mode(1)
    ran(run, f"msda_bwd_splat_d32<{CNAME[godt]}, 8>", tag=which)
    torch.cuda.synchronize()
    _backward_check(f"splat {which} {godt} direct={os.environ.get('BEVF_SPLAT_DIRECT', '')} slices {br}", c, gv, gl,
                    ga)


def test_splat_direct_env():
    """BEVF_SPLAT_DIRECT (read once per process) forces the direct branch on every level: the splat cases rerun in a
    child process with it set."""
    if PROFILING or os.environ.get("BEVF_SPLAT_DIRECT"):
        pytest.skip("child process")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-s", "-p", "no:cacheprovider",
                        "-k", "test_splat_branches"], cwd=ROOT, env=dict(os.environ, BEVF_SPLAT_DIRECT="0xffff"),
                       capture_output=True, text=True, timeout=600)
    tail = r.stdout[-4000:] + r.stderr[-2000:]
    assert r.returncode == 0 and " passed" in r.stdout, tail
    for ln in r.stdout.splitlines():
        if ln.startswith("[msda_fp64]"):
            print(ln)
            warnings.warn(ln, Slack)


# ------------------------------------------------------------------------------------------------
# scaled fp16 and mixed accumulation of grad_value
# ------------------------------------------------------------------------------------------------
def _scale(go):
    amax = go.float().abs().max().item()
    if not (0 < amax < 3.0e38):
        return 1.0
    e = max(math.frexp(amax)[1] - 1, -127) if amax >= 2.0 ** -126 else -127
    return 2.0 ** min(3 - e, 127)


@pytest.mark.parametrize("shape", ["rows_m5", "rows_m8"])
@pytest.mark.parametrize("godt", ["bf16", "f32"])
@pytest.mark.parametrize("gscale", [1.0, 1e-6, 1e3, 0.0])
def test_f16acc(shape, godt, gscale):
    c = case_inputs(shape, "bf16", godt, seed=8, gscale=gscale)
    lib = _lib_()
    gv16 = torch.zeros(c["value"].shape, device=DEV, dtype=torch.float16)
    out = torch.full(c["value"].shape, NAN, device=DEV, dtype=torch.bfloat16)
    gl, ga = _backward_bufs(c)

    def run():
        amax = ops.abs_max_bits(c["grad_out"])
        gv16.zero_()
        _check(lib.bevf_msda_rows_backward_f16acc(
            c["value"].data_ptr(), ops._DT[torch.bfloat16], c["hw"].data_ptr(), c["ls"].data_ptr(), c["loc"].data_ptr(),
            c["attn"].data_ptr(), c["grad_out"].data_ptr(), ops._DT[DT[godt]], gv16.data_ptr(), amax.data_ptr(),
            gl.data_ptr(), ga.data_ptr(), c["row_map"].data_ptr(), None, *_dims(c), _st()))
        _check(lib.bevf_gv16_unscale(gv16.data_ptr(), amax.data_ptr(), out.data_ptr(), out.numel(), _st()))
    ran(run, f"msda_bwd_d32<__nv_bfloat16, {CNAME[godt]}, true, __half", "gv16_unscale_kernel", "abs_max_kernel", tag=shape)
    torch.cuda.synchronize()
    r = _ref_backward(c)
    report = {}
    within(out, r["grad_value"], mo.bar_gv_f16(r["gv_mag"], r["gv_count"], r["grad_value"], _scale(c["grad_out"])),
           "grad_value", report)
    _check_loc_attn(c, gl, ga, r, report)
    show(f"f16acc {shape} {godt} gscale={gscale:g}", report)


def _mixed_run(c, godt, nf16, map_range=None, first_dense=None):
    lib = _lib_()
    s_fine = sum(h * w for h, w in c["hw_host"][:nf16])
    fine = torch.zeros((c["NB"], s_fine, c["M"], 32), device=DEV, dtype=torch.float16)
    side = torch.zeros((c["NB"], c["S"] - s_fine, c["M"], 32), device=DEV)
    out = torch.full(c["value"].shape, NAN, device=DEV, dtype=torch.bfloat16)
    gl, ga = _backward_bufs(c)
    hw = _hw_host(c)

    def run():
        amax = ops.abs_max_bits(c["grad_out"])
        fine.zero_()
        side.zero_()
        args = (c["value"].data_ptr(), ops._DT[torch.bfloat16], c["hw"].data_ptr(), c["ls"].data_ptr(),
                ctypes.addressof(hw), c["loc"].data_ptr(), c["attn"].data_ptr(), c["grad_out"].data_ptr(),
                ops._DT[DT[godt]], fine.data_ptr(), side.data_ptr(), amax.data_ptr(), nf16)
        if map_range is None:
            _check(lib.bevf_msda_rows_backward_mixed(*args, gl.data_ptr(), ga.data_ptr(), c["row_map"].data_ptr(), None,
                                                     *_dims(c), _st()))
        else:
            _check(lib.bevf_msda_rows_backward_mixed_dense(*args, first_dense, gl.data_ptr(), ga.data_ptr(),
                                                           c["row_map"].data_ptr(), map_range.data_ptr(), *_dims(c),
                                                           _st()))
        _check(lib.bevf_gv_merge(fine.data_ptr(), side.data_ptr(), amax.data_ptr(), out.data_ptr(), c["NB"], c["S"],
                                 s_fine, c["M"] * 32, _st()))
    return out, gl, ga, run, s_fine


def _mixed_check(case, c, out, gl, ga, s_fine, dense_from=None):
    """Fine pixels [0, s_fine): scaled-fp16 bar; side pixels: fp32 (or, from pixel ``dense_from`` on, the dense
    kernel's) bar, then bf16."""
    r = _ref_backward(c, dense_mult=dense_from is not None)
    ref, mag, cnt = r["grad_value"], r["gv_mag"], r["gv_count"]
    bar = mo.bar_gv_f32_to_bf16(mag, cnt, ref)
    bar[:, :s_fine] = mo.bar_gv_f16(mag, cnt, ref, _scale(c["grad_out"]))[:, :s_fine]
    if dense_from is not None:
        db = mo.bar_gv_dense(mag, r["gv_dense_mag"], cnt)
        db = db + mo.UBF * (ref.abs() + db)
        bar[:, dense_from:] = db[:, dense_from:]
    report = {}
    within(out, ref, bar, "grad_value", report)
    _check_loc_attn(c, gl, ga, r, report)
    show(case, report)


@pytest.mark.parametrize("shape", ["rows_m5", "rows_m8", "rows_m16"])
@pytest.mark.parametrize("godt", ["bf16", "f32"])
@pytest.mark.parametrize("nf16", [1, 2])
def test_mixed(shape, godt, nf16):
    c = case_inputs(shape, "bf16", godt, seed=9)
    if nf16 >= c["L"]:
        pytest.skip("the pyramid has fewer levels")
    out, gl, ga, run, s_fine = _mixed_run(c, godt, nf16)
    ran(run, f"msda_bwd_d32<__nv_bfloat16, {CNAME[godt]}, true, float", "gv_merge_kernel", tag=(shape, nf16))
    torch.cuda.synchronize()
    _mixed_check(f"mixed {shape} {godt} nf16={nf16}", c, out, gl, ga, s_fine)


# ------------------------------------------------------------------------------------------------
# dense tensor-core levels (msda_dense.cu)
# ------------------------------------------------------------------------------------------------
# level 0 (9000 pixels) is above BEVF_DENSE_MAXPIX (8192): reduction path; level 1 (2400) is cut into 5 bins of
# <= 512; levels 2 and 3 share a bin
DENSE_SHAPE = dict(levels=[(90, 100), (40, 60), (12, 20), (6, 10)], M=8, P=4, NB=2, R=300, unused=(7, 150, 299))


def _dense_inputs(vdt, seed):
    """Rows grouped by value map, each map's rows contiguous, the unused rows (-1) after the last range: the layout
    bevf_sca_plan_build produces and map_range describes (the dense kernel takes every row of a range as the map's)."""
    c = case_inputs(DENSE_SHAPE, vdt, "bf16", seed=seed)
    rm = c["row_map"]
    key = torch.where(rm >= 0, rm, torch.full_like(rm, c["NB"]))
    perm = torch.argsort(key, stable=True)
    for k in ("loc", "attn", "grad_out"):
        c[k] = c[k][perm].contiguous()
    c["row_map"] = rm[perm].contiguous()
    c["dead"] = c["row_map"] < 0
    rng = []
    for b in range(c["NB"]):
        idx = (c["row_map"] == b).nonzero().flatten()
        rng += [int(idx.min()), int(idx.max()) + 1]
    c["map_range"] = torch.tensor(rng, device=DEV, dtype=torch.int32)
    return c


@pytest.fixture
def dense_mode():
    lib = _lib_()
    yield lambda m: _check(lib.bevf_msda_set_dense_backward(m))
    _check(lib.bevf_msda_set_dense_backward(-1))


@pytest.mark.parametrize("vdt", ["bf16"])       # the dense kernel needs a bf16 grad_out, which needs a bf16 value
@pytest.mark.parametrize("mode", [1, 2])
def test_dense(vdt, mode, dense_mode):
    c = _dense_inputs(vdt, seed=10)
    dense_mode(mode)
    lib = _lib_()
    gv = torch.zeros(c["value"].shape, device=DEV)
    gl, ga = _backward_bufs(c)
    hw = _hw_host(c)

    def run():
        gv.zero_()
        _check(lib.bevf_msda_rows_backward_dense(
            c["value"].data_ptr(), ops._DT[DT[vdt]], c["hw"].data_ptr(), c["ls"].data_ptr(), ctypes.addressof(hw),
            c["loc"].data_ptr(), c["attn"].data_ptr(), c["grad_out"].data_ptr(), ops._DT[torch.bfloat16],
            gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), c["row_map"].data_ptr(), c["map_range"].data_ptr(),
            *_dims(c), _st()))
    ran(run, "msda_bwd_dense_tc<4, 4, 3>", f"msda_bwd_d32<{CNAME[vdt]}, __nv_bfloat16, true, float", tag=mode)
    torch.cuda.synchronize()
    r = _ref_backward(c, dense_mult=True)
    bar = mo.bar_grad_value_f32(r["gv_mag"], r["gv_count"])
    first = c["hw_host"][0][0] * c["hw_host"][0][1]                # levels 1.. go through the dense kernel
    bar[:, first:] = mo.bar_gv_dense(r["gv_mag"], r["gv_dense_mag"], r["gv_count"])[:, first:]
    report = {}
    within(gv, r["grad_value"], bar, "grad_value", report)
    _check_loc_attn(c, gl, ga, r, report)
    show(f"dense mode {mode} {vdt}", report)


@pytest.mark.parametrize("first_dense", [1, 2])
@pytest.mark.parametrize("mode", [1, 2])
def test_mixed_dense(first_dense, mode, dense_mode):
    c = _dense_inputs("bf16", seed=11)
    dense_mode(mode)
    out, gl, ga, run, s_fine = _mixed_run(c, "bf16", 1, c["map_range"], first_dense)
    ran(run, "msda_bwd_dense_tc<4, 4, 3>", "msda_bwd_d32<__nv_bfloat16, __nv_bfloat16, true, float", "gv_merge_kernel",
        tag=(mode, first_dense))
    torch.cuda.synchronize()
    dense_from = sum(h * w for h, w in c["hw_host"][:first_dense])
    _mixed_check(f"mixed_dense mode {mode} from level {first_dense}", c, out, gl, ga, s_fine, dense_from)


# ------------------------------------------------------------------------------------------------
# fixed point (deterministic mode)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["d32", "generic"])
@pytest.mark.parametrize("vdt,godt", PAIRS)
def test_fixed_point(kind, vdt, godt):
    c = case_inputs("rows_m5" if kind == "d32" else "dense_edges", vdt, godt, seed=12,
                    D=32 if kind == "d32" else 71)
    lib = _lib_()
    k = int(lib.bevf_msda_fx_frac_bits(c["Q"], c["L"], c["P"]))
    fx = torch.zeros(c["value"].shape, device=DEV, dtype=torch.int64)
    bounds = torch.empty(2, device=DEV, dtype=torch.int32)
    out = torch.full(c["value"].shape, NAN, device=DEV)
    gl, ga = _backward_bufs(c)

    def run():
        fx.zero_()
        args = (c["value"].data_ptr(), ops._DT[DT[vdt]], c["hw"].data_ptr(), c["ls"].data_ptr(), c["loc"].data_ptr(),
                c["attn"].data_ptr(), c["grad_out"].data_ptr(), ops._DT[DT[godt]], fx.data_ptr(), bounds.data_ptr(), k,
                gl.data_ptr(), ga.data_ptr())
        if c["row_map"] is not None:
            _check(lib.bevf_msda_rows_backward_fx(*args, c["row_map"].data_ptr(), *_dims(c), _st()))
        else:
            _check(lib.bevf_msda_backward_fx(*args, *_dims(c), _st()))
        _check(lib.bevf_msda_fx_convert(fx.data_ptr(), bounds.data_ptr(), k, out.data_ptr(), ops._DT[torch.float32], 0,
                                        out.numel(), _st()))
    name = "msda_bwd_d32" if kind == "d32" else "msda_bwd_generic"
    tail = ", true, long long" if kind == "d32" else ", long long>"
    ran(run, f"{name}<{CNAME[vdt]}, {CNAME[godt]}{tail}", "fx_convert_kernel", tag=kind)
    torch.cuda.synchronize()
    r = _ref_backward(c)
    amax = c["attn"].abs().max().item()               # an upper bound of the launch's own max|attn|
    E = mo.fx_exponent(amax, c["grad_out"].float().abs().max().item())
    report = {}
    within(out, r["grad_value"], mo.bar_gv_fx(r["gv_mag"], r["gv_count"], r["grad_value"], E, k), "grad_value", report)
    _check_loc_attn(c, gl, ga, r, report)
    show(f"fx {kind} {vdt}/{godt}", report)


# ------------------------------------------------------------------------------------------------
# the high bits of the packed corner offset
# ------------------------------------------------------------------------------------------------
def test_high_offset_bits():
    """One 2048 x 2100 level with 8 heads: for its lower rows the packed in-level offset pidx * M * 32 of the 32-bit
    corner word (enc = offset | dx | dy << 1 in msda_fwd_d32 / msda_bwd_d32) exceeds 2^30.  About 2.2 GB of bf16 value
    and 4.4 GB of fp32 grad_value; the restatement's grad_value covers the touched pixels only, every other pixel must
    hold an exact zero."""
    H, W, M, P, R = 2048, 2100, 8, 4, 256
    S = H * W
    gd = torch.Generator(device=DEV).manual_seed(13)
    gen = torch.Generator().manual_seed(13)
    value = torch.randn(1, S, M, 32, device=DEV, dtype=torch.bfloat16, generator=gd)
    hw, starts, _ = mo.pyramid([(H, W)])
    loc = torch.rand(R, M, 1, P, 2, generator=gen)
    loc[..., 1] = 0.96 + 0.04 * loc[..., 1]
    flat = loc.view(-1, 2)
    sel = torch.randperm(flat.shape[0], generator=gen)[:flat.shape[0] // 8]
    flat[sel] = mo.border_locs(hw, sel.numel(), gen).view(-1, 2)
    attn = torch.rand(R, M, 1, P, generator=gen) + 0.05
    attn = attn / attn.sum((-1, -2), keepdim=True)
    row_map = torch.zeros(R, dtype=torch.int32)
    row_map[[3, 100, 101]] = -1
    c = dict(value=value, hw=hw.to(DEV), ls=starts.to(DEV), loc=loc.to(DEV).contiguous(), attn=attn.to(DEV),
             row_map=row_map.to(DEV), grad_out=torch.randn(R, M * 32, generator=gen).to(DEV, torch.bfloat16),
             NB=1, S=S, M=M, D=32, Q=R, L=1, P=P, rows=R, hw_host=[(H, W)])
    c["dead"] = c["row_map"] < 0
    pix, w, _, _, _, _ = mo._geometry(c["loc"], c["hw"], c["ls"], S)
    live_w = (w != 0) & (c["row_map"] >= 0).view(-1, 1, 1, 1, 1)
    assert int(pix[live_w].max()) * M * 32 > 2 ** 30, "no sample reaches the high bits of the offset"
    touched = torch.unique(pix[live_w])
    out, run_f = _forward_case(c, "bf16", "bf16")
    gv, gl, ga, run_b = _backward_case(c, "bf16", "bf16")
    ran(lambda: (run_f(), run_b()), "msda_fwd_d32<__nv_bfloat16, __nv_bfloat16, false>",
        "msda_bwd_d32<__nv_bfloat16, __nv_bfloat16, true, float")
    torch.cuda.synchronize()
    _forward_check("high offset bits", c, "bf16", "bf16", out)
    r = _ref_backward(c, gv_rows=touched)
    gvf = gv.view(S, M, 32)
    report = {}
    within(gvf[touched], r["grad_value"], mo.bar_grad_value_f32(r["gv_mag"], r["gv_count"]), "grad_value", report)
    nz = (gvf != 0).flatten(1).any(1)
    nz[touched] = False
    assert not bool(nz.any()), f"{int(nz.sum())} untouched pixels of grad_value are not zero"
    _check_loc_attn(c, gl, ga, r, report)
    show("high offset bits (touched pixels)", report)


# ------------------------------------------------------------------------------------------------
# SpatialCrossAttention's fused sampler: msda_fwd_d32<bf16, bf16, true>, msda_bwd_d32<bf16, bf16, true, float, true>
# ------------------------------------------------------------------------------------------------
def _cam_sum(x, pq, B, Nq, tail):
    """Per-query sum over the cameras' pair rows of x (B * R, ...) -> (B, Nq, *tail) float64."""
    R = pq.numel()
    valid = pq.long() >= 0
    s = torch.zeros(B, Nq, *tail, dtype=F64, device=DEV)
    s.index_add_(1, pq.long()[valid], x.to(F64).reshape(B, R, *tail)[:, valid])
    return s


@pytest.mark.parametrize("dense", [False, True])
def test_sca_fused(dense):
    """The fused SCA sampler on the small4 rig (device-built pair list with unused rows; queries seen by 0, 1 and
    several cameras), forward through ops.sca_rows_forward_fused, backward through the C entry point with NaN-prefilled
    grad_loc / grad_attn / d_raw and bevf_sca_prep_backward_multi after it, as ops.sca_rows_backward_fused runs them.
    The restatement takes loc / attn from ops.sca_prep_forward (bit-identical to the fused samples,
    tests/test_sca_fused_prep_gpu.py).
      out, grad_value: the bars of the unfused paths (level 0 scaled fp16, the rest fp32 or, with ``dense``, level 3
        through the dense kernel);
      grad_loc / grad_attn: written for the rows whose query several cameras see, untouched for the others;
      d_raw: encoder_ops_oracle's SCA prep backward of the restated grad_loc / grad_attn.  Its bar is the prep's own
        (test_encoder_ops_gpu's _sca_off_abs_bar / _sca_logit_bar on the magnitudes |g| + bar) plus the sampler's
        error carried through the prep's linear backward: sum over cameras of bar_gl / (W, H) on the offsets,
        a (S + sum_j a_j S_j) with S = the camera sum of bar_ga on the logits."""
    from tests import encoder_ops_oracle as eo
    from tests import test_encoder_ops_gpu as eg
    from tests import test_sca_fused_prep_gpu as sf
    k = sf._case("small4", 1, True, seed=14)
    plan, raw, v, ss, lsi, levels = k["plan"], k["raw"], k["value"], k["ss"], k["lsi"], k["levels"]
    B, Nq, L, P = k["bs"], k["nq"], k["l"], k["p"]
    M, D, LP = 8, 32, k["l"] * k["p"]
    gout = k["gout"]
    lib = _lib_()
    NB, S = v.shape[:2]
    rows, pairs = plan.row_map.numel(), plan.pair_q.numel()
    ncam, Dz = plan.ref_cam.shape[0], plan.ref_cam.shape[3]
    nf16, first_dense = 1, (L - 1 if dense else L)
    s_fine = levels[0][0] * levels[0][1]
    fine = torch.zeros((NB, s_fine, M, D), device=DEV, dtype=torch.float16)
    side = torch.zeros((NB, S - s_fine, M, D), device=DEV)
    gvo = torch.full(v.shape, NAN, device=DEV, dtype=torch.bfloat16)
    gl = torch.full((rows, M, L, P, 2), NAN, device=DEV)
    ga = torch.full((rows, M, L, P), NAN, device=DEV)
    d_raw = torch.full(raw.shape, NAN, device=DEV, dtype=torch.bfloat16)
    hw = (ctypes.c_int32 * (2 * L))(*[x for h_w in levels for x in h_w])
    box = {}

    def run():
        out, stats, coarse = ops.sca_rows_forward_fused(v, ss, lsi, raw, plan.ref_cam, plan.pair_q, plan.pair_cam,
                                                        plan.row_map, B, Nq, first_dense if dense else None)
        box["out"] = out
        amax = ops.abs_max_bits(gout)
        fine.zero_()
        side.zero_()
        _check(lib.bevf_sca_rows_backward_fused(
            v.data_ptr(), ops._DT[torch.bfloat16], ss.data_ptr(), lsi.data_ptr(), ctypes.addressof(hw), raw.data_ptr(),
            stats.data_ptr(), coarse[0].data_ptr() if coarse else None, coarse[1].data_ptr() if coarse else None,
            coarse[2] if coarse else L, plan.ref_cam.data_ptr(), plan.pair_q.data_ptr(), plan.pair_cam.data_ptr(),
            plan.pair_of.data_ptr(), gout.data_ptr(), ops._DT[torch.bfloat16], fine.data_ptr(), side.data_ptr(),
            amax.data_ptr(), nf16, first_dense, gl.data_ptr(), ga.data_ptr(), d_raw.data_ptr(),
            plan.row_map.data_ptr(), plan.map_range.data_ptr() if dense else None, NB, S, M, D, rows, L, P, B, Nq,
            pairs, Dz, ncam, _st()))
        _check(lib.bevf_sca_prep_backward_multi(raw.data_ptr(), gl.data_ptr(), ga.data_ptr(), plan.pair_of.data_ptr(),
                                                ss.data_ptr(), d_raw.data_ptr(), ops._DT[torch.bfloat16], B, Nq,
                                                pairs, M, L, P, ncam, _st()))
        _check(lib.bevf_gv_merge(fine.data_ptr(), side.data_ptr(), amax.data_ptr(), gvo.data_ptr(), NB, S, s_fine,
                                 M * D, _st()))
    names = ("msda_fwd_d32<__nv_bfloat16, __nv_bfloat16, true>",
             "msda_bwd_d32<__nv_bfloat16, __nv_bfloat16, true, float, true>", "sca_prep_bwd_m8<8, __nv_bfloat16, true>")
    ran(run, *(names + (("msda_bwd_dense_tc<4, 8, 3>",) if dense else ())), tag=dense)
    torch.cuda.synchronize()
    loc, attn = ops.sca_prep_forward(raw, plan.ref_cam, plan.pair_q, plan.pair_cam, ss, B, Nq, M, L, P)
    c = dict(value=v, hw=ss, ls=lsi, loc=loc, attn=attn, row_map=plan.row_map, grad_out=gout, NB=NB, S=S, M=M, D=D,
             Q=rows, L=L, P=P, rows=rows, hw_host=levels)
    live = plan.row_map >= 0
    c["dead"] = ~live
    report = {}
    ref, mag = mo.forward(v, ss, lsi, loc, attn, plan.row_map)
    within(box["out"][live], ref[live], mo.bar_forward(mag, ref, LP, torch.bfloat16, True)[live], "out", report)
    r = _ref_backward(c, dense_mult=dense)
    g_ref, g_mag, cnt = r["grad_value"], r["gv_mag"], r["gv_count"]
    bar = mo.bar_gv_f32_to_bf16(g_mag, cnt, g_ref)
    bar[:, :s_fine] = mo.bar_gv_f16(g_mag, cnt, g_ref, _scale(gout))[:, :s_fine]
    if dense:
        db = mo.bar_gv_dense(g_mag, r["gv_dense_mag"], cnt)
        dense_from = sum(h * w for h, w in levels[:first_dense])
        bar[:, dense_from:] = (db + mo.UBF * (g_ref.abs() + db))[:, dense_from:]
    within(gvo, g_ref, bar, "grad_value", report)
    # grad_loc / grad_attn: rows of queries seen by several cameras; the others keep the prefill
    seen = (plan.pair_of >= 0).sum(0)
    q_of_row = plan.pair_q.long().repeat(B).clamp(min=0)
    multi = live & (seen[q_of_row] > 1)
    assert multi.any() and (live & ~multi).any()
    gl_bar, ga_bar = mo.bar_grad_loc(r["gl_mag"], D), mo.bar_grad_attn(r["ga_mag"], D)
    within(gl[multi], r["grad_loc"][multi], gl_bar[multi], "grad_loc (multi-camera rows)", report)
    within(ga[multi], r["grad_attn"][multi], ga_bar[multi], "grad_attn (multi-camera rows)", report)
    untouched(gl[~multi], "grad_loc")
    untouched(ga[~multi], "grad_attn")
    # d_raw
    pq, pc = plan.pair_q, plan.pair_cam
    want = eo.sca_prep_backward(raw, plan.ref_cam, pq, pc, ss, r["grad_loc"], r["grad_attn"], B, Nq, M, L, P)
    own = torch.cat([eg._sca_off_abs_bar(r["grad_loc"].abs() + gl_bar, pq, B, Nq, M, L, P, ss),
                     eg._sca_logit_bar(raw, r["grad_attn"].abs() + ga_bar, pq, B, Nq, M, LP)], -1)
    wh = torch.stack([ss[:, 1], ss[:, 0]], -1).to(F64)
    p_off = _cam_sum(gl_bar, pq, B, Nq, (M, L, P, 2)) / wh[:, None, :]
    sga = _cam_sum(ga_bar, pq, B, Nq, (M, LP))
    a = torch.softmax(raw[:, M * LP * 2:].to(F64).reshape(B, Nq, M, LP), -1)
    p_lg = a * (sga + (a * sga).sum(-1, keepdim=True))
    prop = torch.cat([p_off.reshape(B * Nq, -1), p_lg.reshape(B * Nq, -1)], -1)
    within(d_raw, want, eg._drawbar(want, torch.bfloat16, own + prop), "d_raw", report)
    show(f"sca_fused dense={dense}", report)


# ------------------------------------------------------------------------------------------------
# through the ops routing (SamplerRows: mode selection, fp16 / mixed accumulation plumbing, group order)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["fp32", "order", "f16", "mixed"])
def test_sampler_rows_routing(route):
    vdt = "f32" if route in ("fp32", "order") else "bf16"
    c = case_inputs("rows_m8", vdt, seed=15)
    gv_mode = {"f16": "f16", "mixed": ("mixed", c["hw_host"], 1)}.get(route)
    order = None
    if route == "order":
        order = torch.randperm(c["Q"], generator=torch.Generator().manual_seed(15)).to(DEV, torch.int32)
    v = c["value"].clone().requires_grad_(True)
    loc = c["loc"].clone().requires_grad_(True)
    attn = c["attn"].clone().requires_grad_(True)
    box = {}

    def run():
        v.grad = loc.grad = attn.grad = None
        out = ops.SamplerRows.apply(v, loc, attn, c["row_map"], c["hw"], c["ls"], order, None, gv_mode)
        out.backward(c["grad_out"])
        box["out"] = out.detach()
    bwd = {"fp32": "msda_bwd_d32<float, float, true, float", "order": "msda_bwd_d32<float, float, true, float",
           "f16": "msda_bwd_d32<__nv_bfloat16, __nv_bfloat16, true, __half",
           "mixed": "msda_bwd_d32<__nv_bfloat16, __nv_bfloat16, true, float"}[route]
    ran(run, f"msda_fwd_d32<{CNAME[vdt]}, {CNAME[vdt]}, false>", bwd, tag=route)
    torch.cuda.synchronize()
    live = ~c["dead"]
    report = {}
    ref, mag = mo.forward(c["value"], c["hw"], c["ls"], c["loc"], c["attn"], c["row_map"])
    within(box["out"][live], ref[live], mo.bar_forward(mag, ref, c["L"] * c["P"], DT[vdt], vdt == "bf16")[live], "out",
           report)
    r = _ref_backward(c)
    g_ref, g_mag, cnt = r["grad_value"], r["gv_mag"], r["gv_count"]
    if route in ("fp32", "order"):
        bar = mo.bar_grad_value_f32(g_mag, cnt)
    else:
        f16 = mo.bar_gv_f16(g_mag, cnt, g_ref, _scale(c["grad_out"]))
        bar = f16 if route == "f16" else mo.bar_gv_f32_to_bf16(g_mag, cnt, g_ref)
        s_fine = c["hw_host"][0][0] * c["hw_host"][0][1]
        bar[:, :s_fine] = f16[:, :s_fine]
    within(v.grad, g_ref, bar, "grad_value", report)
    within(loc.grad[live], r["grad_loc"][live], mo.bar_grad_loc(r["gl_mag"], 32)[live], "grad_loc", report)
    within(attn.grad[live], r["grad_attn"][live], mo.bar_grad_attn(r["ga_mag"], 32)[live], "grad_attn", report)
    show(f"SamplerRows {route}", report)
