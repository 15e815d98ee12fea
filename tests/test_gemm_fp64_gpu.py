"""The wgmma projection GEMMs (csrc/gemm.cu) against the float64 restatement of tests/gemm_fp64_oracle.py, on every
instantiation: weight-stationary and streamed forward / input gradient, the split-M weight gradient and the two-pass
reduce.

Every case calls the C entry point through _lib with:
- inputs that are views into larger buffers whose rows past M (and weight rows past N) are NaN;
- outputs that are views inside buffers filled with a sentinel bit pattern: the output itself is prefilled with it too
  (zeros / the old value where the entry point accumulates), so every element must be written and nothing outside
  [M, N] / [N, K] / [N] may change;
- for the two-pass weight gradient, a workspace filled with NaN, so pass 2 must read only what pass 1 wrote.
Exact-regime cases must equal RN_out(y64) bit for bit (NaN where the restatement has NaN); rounding-regime cases must
lie within the per-element bar of their arithmetic path, and report their worst err / bar as a ``Slack`` warning.

A pipeline deadlock must not hold the GPU, so the cases run in child processes under a hard timeout, one per family
and operand dtype; each child reports one JSON line per case.  Which instantiation every case launches is checked in
one more child under torch.profiler (test_every_case_runs_its_instantiation)."""
import ctypes
import json
import math
import os
import subprocess
import sys
import time
import warnings

import pytest
import torch

from bevformer_b200 import _lib, ops
from tests import gemm_fp64_oracle as go

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
NAN = float("nan")
PAD = 256                                # sentinel / NaN elements around every buffer (keeps 16-byte alignment)
SENTINEL = {torch.float32: 0x7FA5A5A5, torch.bfloat16: 0x7FA5, torch.float16: 0x7E5A}   # quiet NaN patterns
INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
DTN = {"bf16": torch.bfloat16, "f16": torch.float16}
CHILD_TIMEOUT = 900


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


CASES = go.cases(_sms())
BY_ID = {c["id"]: c for c in CASES}


# ------------------------------------------------------------------------------------------------
# the child: runs one batch of cases and prints one JSON line per case
# ------------------------------------------------------------------------------------------------
def _padded(t, pad_rows):
    """t inside a buffer whose trailing pad_rows rows (or, for a vector, PAD elements) are NaN: returns the view."""
    if t.dim() == 1:
        buf = torch.full((t.shape[0] + PAD,), NAN, device=t.device, dtype=t.dtype)
    else:
        buf = torch.full((t.shape[0] + pad_rows, t.shape[1]), NAN, device=t.device, dtype=t.dtype)
    buf[:t.shape[0]] = t
    return buf[:t.shape[0]]


class Guarded:
    """An output view inside a sentinel-filled buffer; ``init`` (or the sentinel) fills the view itself."""

    def __init__(self, shape, dtype, device, init=None):
        n = math.prod(shape)
        self.buf = torch.empty(n + 2 * PAD, device=device, dtype=dtype)
        self.pattern = SENTINEL[dtype]
        self.buf.view(INT[dtype]).fill_(self.pattern)
        self.view = self.buf[PAD:PAD + n].view(shape)
        if init is not None:
            self.view.copy_(init)

    def outside_untouched(self):
        bits = self.buf.view(INT[self.buf.dtype])
        return bool((bits[:PAD] == self.pattern).all() and (bits[PAD + self.view.numel():] == self.pattern).all())


def exact_mismatch(got, want):
    """Elements where got (storage type) differs from want (float64) as values; NaN must meet NaN."""
    g = got.to(F64)
    same = (g == want) | (torch.isnan(g) & torch.isnan(want))
    return ~same


def _describe(bad, got, want, extra=""):
    i = int(bad.flatten().nonzero()[0])
    shape = tuple(got.shape)
    idx = []
    for d in reversed(shape):
        idx.append(i % d)
        i //= d
    idx = tuple(reversed(idx))
    return (f"{int(bad.sum())} of {bad.numel()} elements wrong; first at {idx}: got {got[idx].item()!r} want "
            f"{want[idx].item()!r}{extra}")


def within(got, ref, bar):
    """Worst |got - ref| / bar (inf where got is NaN or exceeds a zero bar), and the mask of elements above 1."""
    err = (got.to(F64) - ref).abs()
    ratio = torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(err), math.inf, ratio)
    return (ratio.max().item() if ratio.numel() else 0.0), ~(ratio <= 1.0)


def _path(case, out):
    op = case["op"]
    if op == "fwd":
        return "fwd f32 out" if case.get("out") == "f32" else "fwd 16-bit out"
    if op == "dgrad":
        return "dgrad 16-bit out"
    if op == "wgrad":
        return f"wgrad {out} red.add"
    if op == "wgrad_out":
        return f"wgrad {out} two-pass {go._DTN[case['grad_dtype']]}"
    return f"wgrad {out} accumulate-into"


def launch(case, lib, a, b, bias=None, addend=None, outs=None, ws=None):
    """The C entry point of ``case`` on device tensors; returns its status."""
    op, M, N, K, dt = case["op"], case["M"], case["N"], case["K"], case["dtype"]
    st = torch.cuda.current_stream().cuda_stream
    P = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    if op == "fwd":
        bdt = ops._DT[bias.dtype] if bias is not None else ops.F32
        ydt = torch.float32 if case.get("out") == "f32" else dt
        return lib.bevf_linear_forward_dt(P(a), P(b), P(bias), bdt, P(addend), P(outs[0]), ops._DT[ydt], M, N, K,
                                          int(case.get("relu", False)), ops._DT[dt], st)
    if op == "dgrad":
        if addend is None:
            return lib.bevf_linear_dgrad_dt(P(a), P(b), P(outs[0]), M, N, K, ops._DT[dt], st)
        return lib.bevf_linear_dgrad_acc_dt(P(a), P(b), P(addend), P(outs[0]), M, N, K, ops._DT[dt], st)
    dw, db = outs
    if op == "wgrad":
        return lib.bevf_linear_wgrad_dt(P(a), P(b), P(dw), P(db), M, N, K, ops._DT[dt], st)
    if op == "wgrad_out":
        return lib.bevf_linear_wgrad_out_dt(P(a), P(b), P(dw), P(db), ops._DT[case["grad_dtype"]], P(ws), ws.numel(),
                                            M, N, K, ops._DT[dt], st)
    return lib.bevf_linear_wgrad_into_dt(P(a), P(b), P(dw), P(db), P(ws), ws.numel(), M, N, K, ops._DT[dt], st)


def _out_shapes(case):
    op, M, N, K = case["op"], case["M"], case["N"], case["K"]
    if op == "fwd":
        return [("y", (M, N), torch.float32 if case.get("out") == "f32" else case["dtype"])]
    if op == "dgrad":
        return [("y", (M, K), case["dtype"])]
    gdt = case.get("grad_dtype", torch.float32)
    outs = [("dw", (N, K), gdt)]
    if case.get("db"):
        outs.append(("db", (N,), gdt))
    return outs


def run_case(case, lib, sms, dev):
    """One case end to end on the device; returns (report {path: worst err/bar}, exact: bool)."""
    pl = go.plan(case, sms)
    if case["op"] in ("wgrad_out", "wgrad_into"):
        got_ws = int(lib.bevf_linear_wgrad_workspace_bytes(case["M"], case["N"], case["K"]))
        assert got_ws == pl["workspace"], f"workspace {got_ws} != restated plan {pl['workspace']}"
    inp = go.make_inputs(case, dev)
    a = _padded(inp["a"], 128)
    b = _padded(inp["b"], 128)
    bias = _padded(inp["bias"], 0) if "bias" in inp else None
    addend = _padded(inp["addend"], 128) if "addend" in inp else None
    outs = []
    for name, shape, odt in _out_shapes(case):
        init = None
        if case["op"] == "wgrad":
            init = torch.zeros(shape, device=dev, dtype=odt)
        elif case["op"] == "wgrad_into":
            init = inp["dw0"] if name == "dw" else inp["db0"]
        outs.append(Guarded(shape, odt, dev, init))
    ws = None
    if case["op"] in ("wgrad_out", "wgrad_into"):
        ws = torch.full((pl["workspace"] // 4,), NAN, device=dev).view(torch.uint8)
    views = [g.view for g in outs] + [None] * (2 - len(outs))
    _lib.check(launch(case, lib, a, b, bias, addend, views, ws), lib)
    torch.cuda.synchronize()
    for g, (name, _, _) in zip(outs, _out_shapes(case)):
        assert g.outside_untouched(), f"{name}: memory next to the output was written"
    # the restatement (on the storage-rounded inputs, i.e. exactly what the kernel read)
    rows = case.get("rows")
    if rows:
        r0, r1 = rows
        sub = dict(case, M=r1 - r0)
        sub_inp = dict(inp, a=inp["a"][r0:r1])
        ref = go.reference(sub, sub_inp, sms)
        got = {"y": outs[0].view[r0:r1]}
    else:
        ref = go.reference(case, inp, sms)
        got = {name: g.view for g, (name, _, _) in zip(outs, _out_shapes(case))}
    report, exact = {}, case["regime"] == "exact"
    for name, (want, y64, bar) in ref.items():
        if exact:
            bad = exact_mismatch(got[name], want)
            if bad.any():
                raise AssertionError(f"{name}: " + _describe(bad, got[name], want))
        else:
            worst, bad = within(got[name], y64, bar)
            report[_path(case, name)] = worst
            if bad.any():
                raise AssertionError(f"{name}: worst err/bar {worst:.3g}; " + _describe(bad, got[name], y64))
    special = case.get("special")
    if special:
        odt = case["dtype"]
        y64 = ref["y"][1]
        if special == "ties":
            assert go.is_tie(y64, odt).any(), "the ties case has no tie"
        elif special == "inf":
            assert (y64.abs() >= 65520).any() and torch.isinf(got["y"]).any(), "no fp16 overflow in the inf case"
        elif special == "subnormal":
            sub = (y64 != 0) & (y64.abs() < 2.0 ** -14)
            assert sub.float().mean().item() > 0.5 and (got["y"].to(F64)[sub] != 0).any(), "not subnormal"
    if case.get("poison"):
        want = ref[next(iter(ref))][0]
        assert torch.isnan(want).any(), "poisoned case without a NaN"
    return report, exact


def child_main(family, dtn):
    lib = _lib.load()
    dev = torch.device("cuda:0")
    sms = _sms()
    for case in CASES:
        if case["family"] != family or go._DTN[case["dtype"]] != dtn:
            continue
        t0 = time.time()
        try:
            report, exact = run_case(case, lib, sms, dev)
            rec = dict(id=case["id"], ok=True, report=report, exact=exact)
        except Exception as e:     # noqa: BLE001 -- reported per case; the parent fails that case
            rec = dict(id=case["id"], ok=False, msg=f"{type(e).__name__}: {e}")
        rec["seconds"] = round(time.time() - t0, 3)
        print("CASE " + json.dumps(rec), flush=True)
        torch.cuda.empty_cache()


def profile_main():
    """Every case once under the profiler (zeros as inputs: the dispatch does not depend on values), one session;
    a marker kernel before each launch splits the kernel list per case."""
    from torch.profiler import ProfilerActivity, profile
    lib = _lib.load()
    dev = torch.device("cuda:0")
    seen = {}
    order = []
    one = torch.ones(1, device=dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in CASES:
            key = (case["op"], case["dtype"], case["M"], case["N"], case["K"], case.get("out"),
                   case.get("grad_dtype"), bool(case.get("addend")))
            if key in seen:
                continue
            seen[key] = case["id"]
            M, N, K, dt = case["M"], case["N"], case["K"], case["dtype"]
            sa, sb = {"fwd": ((M, K), (N, K)), "dgrad": ((M, N), (N, K))}.get(case["op"], ((M, N), (M, K)))
            a, b = torch.zeros(sa, device=dev, dtype=dt), torch.zeros(sb, device=dev, dtype=dt)
            cols = N if case["op"] == "fwd" else K
            bias = torch.zeros(cols, device=dev) if case.get("bias") else None
            addend = torch.zeros((M, cols), device=dev, dtype=dt) if case.get("addend") else None
            outs = [torch.zeros(s, device=dev, dtype=o) for _, s, o in _out_shapes(case)] + [None]
            pl = go.plan(case, _sms())
            ws = torch.zeros(pl.get("workspace", 0), device=dev, dtype=torch.uint8)
            torch.cuda.synchronize()
            one.atan2_(one)                                    # marker
            _lib.check(launch(case, lib, a, b, bias, addend, outs[:2], ws), lib)
            torch.cuda.synchronize()
            order.append(case["id"])
            del a, b, bias, addend, outs, ws
            torch.cuda.empty_cache()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    per = []
    for e in evs:
        if "atan2" in e.name:
            per.append([])
        elif per and ("gemm_" in e.name or "wgrad_reduce" in e.name):
            per[-1].append(e.name)
    print("PROFILE " + json.dumps(dict(order=order, kernels=per)), flush=True)


# ------------------------------------------------------------------------------------------------
# the parent: one child per (family, dtype), cached; one test per case
# ------------------------------------------------------------------------------------------------
_RESULTS = {}


def batch(family, dtn):
    key = (family, dtn)
    if key not in _RESULTS:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, "-m", "tests.test_gemm_fp64_gpu", "--family", family, "--dtype", dtn],
                               cwd=ROOT, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
            out, tail, rc = r.stdout, r.stdout[-3000:] + r.stderr[-3000:], r.returncode
        except subprocess.TimeoutExpired as e:
            out = (e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")
            tail, rc = f"timed out after {CHILD_TIMEOUT} s (a pipeline deadlock?)\n" + out[-3000:], None
        recs = {}
        for ln in out.splitlines():
            if ln.startswith("CASE "):
                rec = json.loads(ln[5:])
                recs[rec["id"]] = rec
        _RESULTS[key] = (recs, tail, rc, time.time() - t0)
    return _RESULTS[key]


class Slack(UserWarning):
    """The worst err / bar of a rounding-regime case: pytest lists them in its warnings summary."""


@pytest.mark.parametrize("cid", [c["id"] for c in CASES])
def test_case(cid):
    case = BY_ID[cid]
    recs, tail, rc, _ = batch(case["family"], go._DTN[case["dtype"]])
    assert cid in recs, f"the child did not report this case (exit {rc}):\n{tail}"
    rec = recs[cid]
    assert rec["ok"], rec["msg"]
    if rec["report"]:
        msg = f"[gemm_fp64] {cid}: " + ", ".join(f"{k} {v:.3g}" for k, v in rec["report"].items())
        print(msg)
        warnings.warn(msg, Slack)


def test_summary():
    """Worst err / bar per arithmetic path over every rounding-regime case, and the count of bit-exact cases (the
    summary runs the batches it needs if the cases did not)."""
    worst, exact, seconds = {}, 0, 0.0
    for fam, dtn in sorted({(c["family"], go._DTN[c["dtype"]]) for c in CASES}):
        recs, _, _, t = batch(fam, dtn)
        seconds += t
        for rec in recs.values():
            if not rec["ok"]:
                continue
            exact += rec["exact"]
            for k, v in rec["report"].items():
                worst[k] = max(worst.get(k, 0.0), v)
    msg = (f"[gemm_fp64] {exact} bit-exact cases; children {seconds:.0f} s; worst err/bar per path: " +
           "; ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    print(msg)
    warnings.warn(msg, Slack)
    assert exact >= sum(c["regime"] == "exact" for c in CASES)


def test_every_case_runs_its_instantiation():
    """One child under torch.profiler launches every distinct case once: each must run exactly the GEMM / reduce
    instantiations its plan declares, and together they cover all 28."""
    r = subprocess.run([sys.executable, "-m", "tests.test_gemm_fp64_gpu", "--profile"], cwd=ROOT, capture_output=True,
                       text=True, timeout=CHILD_TIMEOUT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("PROFILE ")][-1]
    prof = json.loads(line[8:])
    assert len(prof["kernels"]) == len(prof["order"]), "the profiler lost marker records"
    sms = _sms()
    names = set()
    for cid, launched in zip(prof["order"], prof["kernels"]):
        want = go.plan(BY_ID[cid], sms)["kernels"]
        got = sorted(launched)
        assert len(got) == len(want) and all(any(w in n for n in got) for w in want), (cid, want, got)
        names.update(want)
    assert len(names) == 28, sorted(names)


def test_plans_reach_their_edges():
    """The case list reaches the dispatch edges it claims on this device."""
    sms = _sms()
    pls = {c["id"]: (c, go.plan(c, sms)) for c in CASES if c["dtype"] == torch.bfloat16 and c["regime"] == "exact"}
    ws = [p for c, p in pls.values() if p.get("ws")]
    assert any(p["groups"] == p["tiles_m"] and p["tiles_m"] < sms for p in ws)             # one tile per CTA
    assert any(p["tiles_m"] == p["groups"] and p["groups"] * p["tiles_n"] >= sms - 1 for p in ws)
    assert any(p["tiles_m"] == p["groups"] + 1 for p in ws)
    assert any(p["tiles_m"] > 10 * p["groups"] for p in ws)
    wg = [(c, p) for c, p in pls.values() if c["op"].startswith("wgrad")]
    assert any(p["splits"] == 1 for _, p in wg)
    assert any(p["splits"] > 1 and p["last_rows"] < p["rows"] for _, p in wg)
    assert any(p["splits"] > 1 and p["splits"] * p["rows"] == c["M"] for c, p in wg)
    assert any(c["N"] % 16 == 8 for c, _ in wg) and any(c["K"] % 128 for c, _ in wg)


# ------------------------------------------------------------------------------------------------
# M = 0, and the Python wrappers' argument contract
# ------------------------------------------------------------------------------------------------
def test_m_zero_launches_nothing():
    lib = _lib.load()
    dev = torch.device("cuda:0")
    a = torch.ones(64, 256, device=dev, dtype=torch.bfloat16)
    w = torch.ones(256, 256, device=dev, dtype=torch.bfloat16)
    y = Guarded((64, 256), torch.bfloat16, dev)
    dw = Guarded((256, 256), torch.float32, dev)
    db = Guarded((256,), torch.float32, dev)
    st = torch.cuda.current_stream().cuda_stream
    before = lib.bevf_launch_count()
    p = a.data_ptr()
    assert lib.bevf_linear_forward_dt(p, w.data_ptr(), 0, 0, 0, y.view.data_ptr(), 1, 0, 256, 256, 0, 1, st) == 0
    assert lib.bevf_linear_dgrad_dt(p, w.data_ptr(), y.view.data_ptr(), 0, 256, 256, 1, st) == 0
    assert lib.bevf_linear_dgrad_acc_dt(p, w.data_ptr(), p, y.view.data_ptr(), 0, 256, 256, 1, st) == 0
    assert lib.bevf_linear_wgrad_dt(p, p, dw.view.data_ptr(), db.view.data_ptr(), 0, 256, 256, 1, st) == 0
    # the two-pass forms have no empty workspace to size and refuse M = 0 before touching anything
    assert lib.bevf_linear_wgrad_workspace_bytes(0, 256, 256) == 0
    assert lib.bevf_linear_wgrad_out_dt(p, p, dw.view.data_ptr(), db.view.data_ptr(), 0, p, 1 << 20, 0, 256, 256, 1,
                                        st) != 0
    assert b"bad dimension" in lib.bevf_last_error()
    torch.cuda.synchronize()
    assert lib.bevf_launch_count() == before
    for g in (y, dw, db):
        assert g.outside_untouched() and (g.buf.view(INT[g.buf.dtype]) == g.pattern).all()
    # the wrappers: an empty batch gives empty / zero gradients
    e = torch.empty(0, 256, device=dev, dtype=torch.bfloat16)
    assert ops.linear_tc(e, w).shape == (0, 256)
    dwo, dbo = ops.linear_wgrad_out(e, e, torch.bfloat16, True)
    assert dwo.shape == (256, 256) and not dwo.any() and not dbo.any()


def _lin_inputs(dt, M=300, N=128, K=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 5, (M, K), generator=g).to("cuda", dt)
    w = torch.randint(-4, 5, (N, K), generator=g).to("cuda", dt)
    b = torch.randint(-4, 5, (N,), generator=g).float().cuda()
    r = torch.randint(-4, 5, (M, N), generator=g).to("cuda", dt)
    return x, w, b, r


def _want(x, w, b=None, r=None):
    y = x.double() @ w.double().t()
    if b is not None:
        y = y + b.double()
    if r is not None:
        y = y + r.double()
    return y


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_linear_tc_non_contiguous_operands(dt):
    """Transposed / sliced x, weight and residual are read as the tensors they are (exact-regime values)."""
    x, w, b, r = _lin_inputs(dt)
    xt = x.t().contiguous().t()                       # same values, column-major
    wt = w.t().contiguous().t()
    rs = torch.cat([r, torch.zeros_like(r)], 1)[:, :r.shape[1]]
    assert not xt.is_contiguous() and not wt.is_contiguous() and not rs.is_contiguous()
    y = ops.linear_tc(xt, wt, b, rs, out_dtype=torch.float32)
    assert torch.equal(y.double(), _want(x, w, b, r))
    # a 3-D activation sliced along its last dimension
    x3 = torch.cat([x, x], 1).view(3, 100, -1)[..., :x.shape[1]]
    assert not x3.is_contiguous()
    y3 = ops.linear_tc(x3, w, out_dtype=torch.float32)
    assert torch.equal(y3.reshape(300, -1).double(), _want(x, w))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_linear_tc_refuses_mismatched_arguments(dt):
    x, w, b, r = _lin_inputs(dt)
    bad = [
        dict(weight=w[:, :128].contiguous()),                         # weight.shape[1] != K
        dict(weight=w.view(1, 128, 256)),                             # not 2-D
        dict(residual=r.float()),                                     # fp32 residual next to 16-bit x
        dict(residual=r[:200]),                                       # fewer rows
        dict(residual=r.reshape(-1)),                                 # same numel, wrong shape
        dict(bias=b[:64]),                                            # bias length != N
        dict(bias=b.view(2, 64)),
    ]
    for kw in bad:
        args = dict(weight=w, bias=b, residual=r)
        args.update(kw)
        with pytest.raises(RuntimeError):
            ops.linear_tc(x, args["weight"], args["bias"], args["residual"])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_wgrad_wrappers_non_contiguous_and_shapes(dt):
    g = torch.Generator().manual_seed(1)
    M, N, K = 300, 128, 256
    dy = torch.randint(-4, 5, (M, N), generator=g).to("cuda", dt)
    x = torch.randint(-4, 5, (M, K), generator=g).to("cuda", dt)
    want = dy.double().t() @ x.double()
    wantb = dy.double().sum(0)
    dyt, xt = dy.t().contiguous().t(), torch.cat([x, x], 1)[:, K:]
    assert not dyt.is_contiguous() and not xt.is_contiguous()
    dw, db = ops.linear_wgrad_tc(dyt, xt, with_bias=True)
    assert torch.equal(dw.double(), want) and torch.equal(db.double(), wantb)
    dw2, db2 = ops.linear_wgrad_out(dyt, xt, torch.float32, True)
    assert torch.equal(dw2.double(), want) and torch.equal(db2.double(), wantb)
    acc = torch.ones(N, K, device="cuda")
    accb = torch.ones(N, device="cuda")
    ops.linear_wgrad_into(dyt, xt, acc, accb)
    assert torch.equal(acc.double(), want + 1) and torch.equal(accb.double(), wantb + 1)
    for fn in (lambda a, b: ops.linear_wgrad_tc(a, b), lambda a, b: ops.linear_wgrad_out(a, b, torch.float32, False),
               lambda a, b: ops.linear_wgrad_into(a, b, torch.zeros(N, K, device="cuda"))):
        with pytest.raises(RuntimeError):
            fn(dy.view(3, 100, N), x)                                 # 3-D dy
        with pytest.raises(RuntimeError):
            fn(dy, x.view(3, 100, K))
        with pytest.raises(RuntimeError):
            fn(dy[:299], x)                                           # unequal M
    with pytest.raises(RuntimeError):
        ops.linear_wgrad_into(dy, x, torch.zeros(N, K, device="cuda"), torch.zeros(N + 1, device="cuda"))


if __name__ == "__main__":
    if "--profile" in sys.argv:
        profile_main()
    else:
        child_main(sys.argv[sys.argv.index("--family") + 1], sys.argv[sys.argv.index("--dtype") + 1])
