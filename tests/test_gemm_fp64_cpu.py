"""tests/gemm_fp64_oracle.py pinned against integer arithmetic, its mutations shown to be caught on the inputs of the GPU
cases they target, the restated workspace plan checked against the library, and the C entry points shown to refuse bad
arguments before they touch memory (fake, never dereferenced pointers)."""
from fractions import Fraction

import pytest
import torch

from bevformer_b200 import _lib
from tests import gemm_fp64_oracle as go

F64 = torch.float64
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
BY_ID = {c["id"]: c for c in go.cases(SMS)}


def _rne(v, mant_bits, emin):
    """Round the exact rational v to a binary format with mant_bits significant bits and smallest normal exponent emin
    (round half to even, subnormals, no overflow handling): Python's round() on a Fraction is half-to-even."""
    if v == 0:
        return Fraction(0)
    e = max(abs(v).numerator.bit_length() - abs(v).denominator.bit_length(), emin)
    while abs(v) >= Fraction(2) ** (e + 1):
        e += 1
    while e > emin and abs(v) < Fraction(2) ** e:
        e -= 1
    q = Fraction(2) ** (e - mant_bits + 1)
    return round(v / q) * q


FMT = {torch.bfloat16: (8, -126), torch.float16: (11, -14)}


@pytest.mark.parametrize("cid", ["fwd-bf16-exact-1000x256x256-bf32-ties", "fwd-f16-exact-1000x256x256-bf32-ties",
                                 "fwd-f16-exact-300x256x256-subnormal", "dgrad-bf16-exact-1000x256x256-addend-ties",
                                 "fwd-bf16-exact-4099x16x512-bf32-relu-addend"])
def test_exact_regime_matches_integer_arithmetic(cid):
    """y64 of the restatement is the integer result (int64 matmul on the integer operands, times the quanta), and its
    16-bit RN equals round-half-to-even on exact rationals, ties included."""
    case = BY_ID[cid]
    inp = go.make_inputs(case)
    r = go.reference(case, inp, SMS)["y"]
    want, y64 = r[0], r[1]
    ea, eb = (-11, -14) if case.get("special") == "subnormal" else (0, 0)
    ia = (inp["a"].to(F64) * 2.0 ** -ea).to(torch.int64)
    ib = (inp["b"].to(F64) * 2.0 ** -eb).to(torch.int64)
    acc = ia @ (ib.t() if case["op"] == "fwd" else ib)
    y = acc.to(F64) * 2.0 ** (ea + eb)
    if "bias" in inp:
        y = y + inp["bias"].to(F64)
    if case.get("relu"):
        y = y.clamp(min=0)
    if "addend" in inp:
        y = y + inp["addend"].to(F64)
    assert torch.equal(y, y64)
    assert (acc.abs() < go.EXACT_LIMIT).all()
    mant, emin = FMT[case["dtype"]]
    ties = go.is_tie(y64, case["dtype"])
    idx = torch.cat([ties.flatten().nonzero()[:200, 0], torch.arange(0, y64.numel(), max(1, y64.numel() // 300))])
    assert ties.any() or case.get("special") == "subnormal"
    for i in idx.tolist():
        v = Fraction(float(y64.flatten()[i]))
        assert Fraction(float(want.flatten()[i])) == _rne(v, mant, emin), (i, v)


def test_exact_bound_is_enforced():
    a = torch.full((2, 1 << 18), 4.0)
    b = torch.full((1 << 18, 3), 4.0)
    with pytest.raises(AssertionError):
        go.check_exact_bound(a, b)                       # 16 * 2^18 = 2^22 quanta
    assert go.check_exact_bound(a[:, :-1], b[:-1]) < go.EXACT_LIMIT
    # every exact case of the GPU file satisfies it (make_inputs asserts), the largest reduction included
    big = max((c for c in BY_ID.values() if c["regime"] == "exact" and c["op"].startswith("wgrad")),
              key=lambda c: c["M"])
    assert big["M"] == 184950
    go.make_inputs(big)


def test_rounding_helpers():
    v = torch.tensor([257.0, 259.0, 258.0, -257.0, 65519.0, 65520.0, 3 * 2.0 ** -25], dtype=F64)
    assert go.is_tie(v[:4], torch.bfloat16).tolist() == [True, True, False, True]
    assert go.rn(v[:4], torch.bfloat16).tolist() == [256.0, 260.0, 258.0, -256.0]
    assert go.rz16(v[:4], torch.bfloat16).tolist() == [256.0, 258.0, 258.0, -256.0]
    h = go.rn(v[4:], torch.float16)
    assert h[0] == 65504.0 and h[1] == float("inf") and h[2] == 2 * 2.0 ** -24
    assert go.rz16(v[4:6], torch.float16).tolist() == [65504.0, 65504.0]


# ------------------------------------------------------------------------------------------------
# mutations: each plausible kernel bug, restated, fails at least one element of the GPU case it targets
# ------------------------------------------------------------------------------------------------
TARGETS = {
    "kblock_partial_16": ["fwd-bf16-round-300x272x256-bf32-relu", "fwd-f16-round-300x272x256-bf32-relu"],
    "double_rounding": ["fwd-bf16-exact-40000x256x256-addend", "dgrad-f16-round-300x256x320-addend"],
    "truncate_store": ["fwd-bf16-exact-1000x256x256-bf32-ties", "fwd-f16-exact-300x256x256-subnormal"],
    "bias_partner": ["fwd-bf16-exact-300x272x256-bf32-relu", "fwd-f16-exact-1000x272x256-b16-addend-of32"],
    "relu_after_addend": ["fwd-bf16-exact-4099x16x512-bf32-relu-addend"],
    "drop_last_row": ["wgrad-bf16-exact-184950x256x256-db", "wgrad-f16-exact-65x200x256"],
    "db_missing_split": ["wgrad-bf16-exact-10000x768x192-db", "wgrad_out-f16-exact-65x200x256-db-gf32"],
    "slabs_16bit": ["wgrad_out-bf16-exact-10000x768x192-db-gbf16", "wgrad_out-f16-exact-10000x768x192-db-gf16"],
}


def test_every_mutation_has_targets():
    assert sorted(TARGETS) == sorted(go.MUTATIONS)
    for ids in TARGETS.values():
        assert all(i in BY_ID for i in ids), [i for i in ids if i not in BY_ID]


def _caught(case, inp, mutate):
    """The mutated restatement, stored as the kernel would store it, fails the GPU test's check somewhere."""
    ref = go.reference(case, inp, SMS)
    mut = go.reference(case, inp, SMS, mutate=mutate)
    for name, (want, y64, bar) in ref.items():
        got = mut[name][0]
        if case["regime"] == "exact":
            same = (got == want) | (torch.isnan(got) & torch.isnan(want))
            if not same.all():
                return True
        elif ((got - y64).abs() > bar).any():
            return True
    return False


@pytest.mark.parametrize("mutate,cid", [(m, c) for m, ids in TARGETS.items() for c in ids])
def test_mutation_is_caught(mutate, cid):
    case = BY_ID[cid]
    assert _caught(case, go.make_inputs(case), mutate)


def test_dropped_row_hides_in_the_rounding_bar_but_not_in_the_exact_regime():
    """At M = 184950 one dropped reduction row moves dW by at most |dy_r| |x_r|, about 1 for a row of unit scale; the
    rounding regime's bar there is about gamma_385 * sum |dy x| = 2.7, so the bug passes it, while the exact regime
    catches it.  The dropped row (the last row of the last split) is scaled to max |.| = 1, a typical row."""
    rnd = BY_ID["wgrad-bf16-round-184950x256x256-db"]
    pl = go.plan(rnd, SMS)
    assert pl["splits"] > 1 and pl["steps"] > 300
    inp = go.make_inputs(rnd)
    for k in ("a", "b"):
        row = inp[k][-1].float()
        inp[k][-1] = (row / row.abs().max()).to(inp[k].dtype)
    ref = go.reference(rnd, inp, SMS)["dw"]
    mut = go.reference(rnd, inp, SMS, mutate="drop_last_row")["dw"]
    diff = (mut[0] - ref[1]).abs()
    assert diff.max() > 0.5                                          # the bug moves dW by about 1 ...
    assert (diff <= ref[2]).all()                                    # ... and every element stays within its bar
    exact = BY_ID["wgrad-bf16-exact-184950x256x256-db"]
    assert _caught(exact, go.make_inputs(exact), "drop_last_row")


# ------------------------------------------------------------------------------------------------
# the library: workspace plan and argument refusals
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(1, 8, 64), (63, 72, 320), (65, 200, 256), (10000, 768, 192), (184950, 256, 256),
                                   (44511, 768, 256), (4099, 8, 1088), (0, 256, 256), (100, 256, 96)])
def test_workspace_matches_restated_plan(M, N, K):
    lib = _lib.load()
    assert lib.bevf_linear_wgrad_workspace_bytes(M, N, K) == go.workspace_bytes(M, N, K, SMS)


A16 = 0x10000            # fake 16-byte aligned addresses: the checks must fail before any of them is used
A16b, A16c, A16d, MIS = 0x20000, 0x30000, 0x40000, 0x10008


def _refused(status, lib, text):
    assert status != 0
    assert text in lib.bevf_last_error().decode(), lib.bevf_last_error()


def test_forward_refuses_bad_arguments():
    lib = _lib.load()
    f = lib.bevf_linear_forward_dt
    ok = dict(x=A16, w=A16b, bias=0, bdt=0, res=0, y=A16c, ydt=1, M=128, N=256, K=256, relu=0, dt=1)

    def call(**kw):
        a = dict(ok, **kw)
        return f(a["x"], a["w"], a["bias"], a["bdt"], a["res"], a["y"], a["ydt"], a["M"], a["N"], a["K"], a["relu"],
                 a["dt"], None)
    _refused(call(K=96), lib, "K must be a multiple of 64")
    _refused(call(N=40), lib, "N must be a multiple of 16")
    _refused(call(x=MIS), lib, "16-byte aligned")
    _refused(call(y=MIS), lib, "16-byte aligned")
    _refused(call(bias=MIS), lib, "16-byte aligned")
    _refused(call(res=MIS), lib, "16-byte aligned")
    _refused(call(ydt=2), lib, "unsupported dtype code")               # fp16 out for bf16 operands
    _refused(call(ydt=7), lib, "unsupported dtype code")
    _refused(call(bias=A16d, bdt=2), lib, "unsupported bias dtype code")
    _refused(call(dt=0), lib, "unsupported operand dtype code")
    _refused(call(M=-1), lib, "bad dimension")
    _refused(call(M=1 << 31), lib, "M too large")
    _refused(call(w=0), lib, "null pointer")


def test_dgrad_refuses_bad_arguments():
    lib = _lib.load()
    _refused(lib.bevf_linear_dgrad_dt(A16, A16b, A16c, 128, 96, 256, 1, None), lib, "multiples of 64")
    _refused(lib.bevf_linear_dgrad_dt(A16, A16b, A16c, 128, 256, 96, 1, None), lib, "multiples of 64")
    _refused(lib.bevf_linear_dgrad_dt(MIS, A16b, A16c, 128, 256, 256, 1, None), lib, "16-byte aligned")
    _refused(lib.bevf_linear_dgrad_dt(A16, A16b, A16c, 128, 256, 256, 0, None), lib, "unsupported operand dtype")
    _refused(lib.bevf_linear_dgrad_acc_dt(A16, A16b, MIS, A16c, 128, 256, 256, 1, None), lib, "addend must be")


def test_wgrad_refuses_bad_arguments():
    lib = _lib.load()
    w = lib.bevf_linear_wgrad_dt
    _refused(w(A16, A16b, A16c, 0, 128, 256, 96, 1, None), lib, "K must be a multiple of 64 and N of 8")
    _refused(w(A16, A16b, A16c, 0, 128, 12, 256, 1, None), lib, "K must be a multiple of 64 and N of 8")
    _refused(w(A16, A16b, A16c, MIS, 128, 256, 256, 1, None), lib, "16-byte aligned")
    _refused(w(MIS, A16b, A16c, 0, 128, 256, 256, 1, None), lib, "16-byte aligned")
    _refused(w(A16, A16b, A16c, 0, 128, 256, 256, 5, None), lib, "unsupported operand dtype")
    need = go.workspace_bytes(1000, 256, 256, SMS)
    o = lib.bevf_linear_wgrad_out_dt
    _refused(o(A16, A16b, A16c, 0, 1, A16d, need - 1, 1000, 256, 256, 1, None), lib, "workspace too small")
    _refused(o(A16, A16b, A16c, 0, 9, A16d, need, 1000, 256, 256, 1, None), lib, "unsupported dtype code")
    _refused(o(A16, A16b, A16c, 0, 1, A16d, need, 1000, 12, 256, 1, None), lib, "N of 8")
    _refused(o(A16, A16b, A16c, 0, 1, MIS, need, 1000, 256, 256, 1, None), lib, "16-byte aligned")
    _refused(o(A16, A16b, A16c, 0, 1, A16d, need, 1000, 256, 256, 3, None), lib, "unsupported operand dtype")
    i = lib.bevf_linear_wgrad_into_dt
    _refused(i(A16, A16b, A16c, 0, A16d, need - 1, 1000, 256, 256, 1, None), lib, "workspace too small")
    _refused(i(A16, A16b, A16c, 0, 0, need, 1000, 256, 256, 1, None), lib, "null pointer")
