"""Pins the float64 restatements of tests/encoder_ops_oracle.py on CPU, at every case the GPU file runs: the prep
restatements against oracle/torch_ref.temporal_self_attention and msda3d (float64, with a sampler that captures
loc / attn), LayerNorm against F.layer_norm and autograd, the rest against plain loops.  Also: the C entry points
refuse misaligned vector operands before any launch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_ref
from tests import encoder_ops_oracle as eo

F64 = torch.float64
DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}


class Capture:
    """A ``sampler`` for torch_ref that records the sampling locations and weights it is given."""

    def __call__(self, value, ss, lsi, loc, att):
        self.loc, self.att = loc, att
        return torch.zeros(value.shape[0], loc.shape[1], value.shape[2] * value.shape[3], dtype=loc.dtype)


def _eye_rows(rows, width):
    """A linear layer's state whose output is input channels [rows) of a ``width``-channel input."""
    w = torch.zeros(rows.stop - rows.start, width, dtype=F64)
    w[torch.arange(w.shape[0]), torch.arange(rows.start, rows.stop)] = 1.0
    return w, torch.zeros(w.shape[0], dtype=F64)


# ------------------------------------------------------------------------------------------------
# TSA prep
# ------------------------------------------------------------------------------------------------
def _tsa_inputs(c, g):
    M, L, P, B, Nq = c["M"], c["L"], c["P"], c["B"], c["Nq"]
    raw = torch.randn(B * Nq, M * 2 * L * P * 3, generator=g, dtype=F64) * 2
    ref2d = torch.rand(B * 2, Nq, L, 2, generator=g, dtype=F64)
    hw = torch.tensor(eo.LEVEL_HW[:L], dtype=torch.int64)
    return raw, ref2d, hw


def _tsa_torch_ref(raw, ref2d, hw, c):
    """torch_ref.temporal_self_attention (one level) with identity projections, so that its sampling-offset and
    attention-weight outputs are the rows of ``raw`` itself; loc / attn captured, frame-major."""
    M, P, B, Nq = c["M"], c["P"], c["B"], c["Nq"]
    width = raw.shape[1]
    n_off = M * 2 * P * 2
    sd = {}
    sd["t.sampling_offsets.weight"], sd["t.sampling_offsets.bias"] = _eye_rows(range(width, width + n_off), 2 * width)
    sd["t.attention_weights.weight"], sd["t.attention_weights.bias"] = _eye_rows(range(width + n_off, 2 * width),
                                                                                 2 * width)
    sd["t.value_proj.weight"], sd["t.value_proj.bias"] = torch.eye(width, dtype=F64), torch.zeros(width, dtype=F64)
    sd["t.output_proj.weight"], sd["t.output_proj.bias"] = torch.eye(width, dtype=F64), torch.zeros(width, dtype=F64)
    cap = Capture()
    query = raw.reshape(B, Nq, width)
    prev = torch.zeros(B * 2, Nq, width, dtype=F64)
    h, w = int(hw[0, 0]), int(hw[0, 1])
    torch_ref.temporal_self_attention(sd, "t.", query, prev, torch.zeros_like(query), ref2d, (h, w), cap,
                                      num_heads=M, num_points=P)
    return cap.loc, cap.att


def _msda3d(raw_rows, ref_rows, hw, M, L, P):
    """torch_ref.msda3d with identity projections on query rows that are raw rows of the (M, L, P) layout."""
    width = raw_rows.shape[-1]
    n_off = M * L * P * 2
    sd = {}
    sd["m.sampling_offsets.weight"], sd["m.sampling_offsets.bias"] = _eye_rows(range(0, n_off), width)
    sd["m.attention_weights.weight"], sd["m.attention_weights.bias"] = _eye_rows(range(n_off, width), width)
    sd["m.value_proj.weight"], sd["m.value_proj.bias"] = torch.eye(M, dtype=F64), torch.zeros(M, dtype=F64)
    cap = Capture()
    n = raw_rows.shape[0]
    torch_ref.msda3d(sd, "m.", raw_rows.reshape(1, n, width), torch.zeros(1, 1, M, dtype=F64),
                     ref_rows.reshape(1, n, -1, 2), hw.tolist(), [0] * L, cap, num_heads=M, num_points=P)
    return cap.loc.reshape(n, M, L, P, 2), cap.att.reshape(n, M, L, P)


def _tsa_msda3d(raw, ref2d, hw, c):
    """The TSA prep of any level count through msda3d: queue entry j's offsets / logits are an (M, L, P) raw row,
    the reference point enters per level (msda3d's anchors are per point, TSA's per level), frame-major rows."""
    M, L, P, B, Nq = c["M"], c["L"], c["P"], c["B"], c["Nq"]
    LP = L * P
    off = raw[:, :M * 2 * LP * 2].reshape(B, Nq, M, 2, LP * 2)
    lg = raw[:, M * 2 * LP * 2:].reshape(B, Nq, M, 2, LP)
    locs, atts = [], []
    for j in range(2):
        rows = torch.cat([off[:, :, :, j].reshape(B * Nq, -1), lg[:, :, :, j].reshape(B * Nq, -1)], -1)
        loc, att = _msda3d(rows, torch.zeros(B * Nq, 1, 2, dtype=F64), hw, M, L, P)
        ref = ref2d.reshape(B, 2, Nq, L, 2)[:, j].reshape(B * Nq, 1, L, 1, 2)
        locs.append((loc + ref).reshape(B, Nq, M, L, P, 2))
        atts.append(att.reshape(B, Nq, M, L, P))
    return torch.stack(locs, 1).reshape(B * 2, Nq, M, L, P, 2), torch.stack(atts, 1).reshape(B * 2, Nq, M, L, P)


@pytest.mark.parametrize("c", eo.tsa_cases(), ids=eo.tsa_case_id)
def test_tsa_prep_restatement(c):
    """Forward and d_raw of the TSA restatement equal msda3d's (any L) and temporal_self_attention's (L = 1) to
    float64 rounding; the interleaved layout is the frame-major one with the two frames of a query adjacent."""
    M, L, P, B, Nq = c["M"], c["L"], c["P"], c["B"], c["Nq"]
    g = torch.Generator().manual_seed(7)
    raw, ref2d, hw = _tsa_inputs(c, g)
    loc, att = eo.tsa_prep_forward(raw, ref2d, hw, B, Nq, M, L, P)
    refs = [_tsa_msda3d] + ([_tsa_torch_ref] if L == 1 else [])
    gl, ga = torch.randn(loc.shape, generator=g, dtype=F64), torch.randn(att.shape, generator=g, dtype=F64)
    want = eo.tsa_prep_backward(raw, ref2d, hw, gl, ga, B, Nq, M, L, P)
    for fn in refs:
        r = raw.clone().requires_grad_(True)
        wl, wa = fn(r, ref2d, hw, c)
        torch.testing.assert_close(loc, wl.reshape(loc.shape).detach(), rtol=0, atol=1e-13)
        torch.testing.assert_close(att, wa.reshape(att.shape).detach(), rtol=0, atol=1e-15)
        ((wl.reshape(loc.shape) * gl).sum() + (wa.reshape(att.shape) * ga).sum()).backward()
        torch.testing.assert_close(want, r.grad, rtol=0, atol=1e-12)
    li, ai = eo.tsa_prep_forward(raw, ref2d, hw, B, Nq, M, L, P, interleave=True)
    assert torch.equal(li, loc.reshape(B, 2, Nq, M, L, P, 2).transpose(1, 2).reshape(li.shape))
    assert torch.equal(ai, att.reshape(B, 2, Nq, M, L, P).transpose(1, 2).reshape(ai.shape))


# ------------------------------------------------------------------------------------------------
# SCA prep
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", eo.sca_cases(), ids=eo.sca_case_id)
def test_sca_prep_restatement(c):
    """Forward and d_raw of the SCA restatement on a hand-built pair list equal msda3d's on the gathered pair rows;
    padding rows are NaN, and a query no camera sees gets a zero d_raw row."""
    M, L, P, D, ncam, B, Nq = c["M"], c["L"], c["P"], c["D"], c["ncam"], c["B"], c["Nq"]
    g = torch.Generator().manual_seed(11)
    pq, pc, pair_of = eo.make_pairs(Nq, ncam, seed=5)
    R = pq.numel()
    raw = torch.randn(B * Nq, M * L * P * 3, generator=g, dtype=F64) * 2
    ref_cam = torch.rand(ncam, B, Nq, D, 2, generator=g, dtype=F64)
    hw = torch.tensor(eo.LEVEL_HW[:L], dtype=torch.int64)
    loc, att, valid = eo.sca_prep_forward(raw, ref_cam, pq, pc, hw, B, Nq, M, L, P)
    assert loc.shape == (B * R, M, L, P, 2) and att.shape == (B * R, M, L, P)
    v = valid.repeat(B)
    assert torch.isnan(loc[~v]).all() and torch.isnan(att[~v]).all() and not torch.isnan(loc[v]).any()
    # pair_of is the inverse of the pair list
    for r in range(R):
        if pq[r] >= 0:
            assert pair_of[pc[r], pq[r]] == r
    assert int((pair_of >= 0).sum()) == int(valid.sum())
    bq = (torch.arange(B)[:, None] * Nq + pq.long().clamp(min=0)[None]).reshape(-1)[v]
    cam = pc.long().clamp(min=0).repeat(B)[v]
    bidx = torch.arange(B).repeat_interleave(R)[v]
    r = raw.clone().requires_grad_(True)
    wl, wa = _msda3d(r[bq], ref_cam[cam, bidx, pq.long().clamp(min=0).repeat(B)[v]], hw, M, L, P)
    torch.testing.assert_close(loc[v], wl.detach(), rtol=0, atol=1e-13)
    torch.testing.assert_close(att[v], wa.detach(), rtol=0, atol=1e-15)
    gl = torch.randn(loc.shape, generator=g, dtype=F64)
    ga = torch.randn(att.shape, generator=g, dtype=F64)
    ((wl * gl[v]).sum() + (wa * ga[v]).sum()).backward()
    want = eo.sca_prep_backward(raw, ref_cam, pq, pc, hw, gl, ga, B, Nq, M, L, P)
    torch.testing.assert_close(want, r.grad, rtol=0, atol=1e-12)
    unseen = (pair_of < 0).all(0)
    assert unseen.any() and (want.reshape(B, Nq, -1)[:, unseen] == 0).all()


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def ln_inputs(c, rows, g, device="cpu"):
    """Inputs of one LayerNorm case in the case's storage types (generated in fp32 on the CPU)."""
    C, adt, pdt = c["C"], DT[c["adt"]], DT[c["pdt"]]
    x = torch.randn(rows, C, generator=g)
    if c["data"] == "const":
        x[::3] = torch.randn(x[::3].shape[0], 1, generator=g)             # every third row constant
    elif c["data"] == "offset":
        x = 1000.0 + x
    res = torch.randn(rows, C, generator=g) if c["res"] else None
    if c["data"] == "const" and res is not None:
        res[::3] = 0.5
    gamma = 1 + 0.3 * torch.randn(C, generator=g)
    beta = 0.3 * torch.randn(C, generator=g)
    pos = torch.randn(rows, C, generator=g) if c["pos"] else None
    dy = torch.randn(rows, C, generator=g)
    dy2 = torch.randn(rows, C, generator=g) if (c["pos"] or c["twin"]) else None
    to = lambda t, dt: None if t is None else t.to(device=device, dtype=dt)
    return dict(x=to(x, adt), res=to(res, adt), gamma=to(gamma, pdt), beta=to(beta, pdt), pos=to(pos, adt),
                dy=to(dy, adt), dy2=to(dy2, adt))


@pytest.mark.parametrize("c", eo.ln_cases(), ids=eo.ln_case_id)
def test_layernorm_restatement(c):
    """The LayerNorm restatement equals float64 F.layer_norm of dropout(x) + res (y, and y + pos) and its autograd
    gradients (the residual's, x's through the keep-mask, gamma's and beta's)."""
    rows = eo.ln_rows(c["rows"], eo.H100_SMS)
    g = torch.Generator().manual_seed(13)
    t = ln_inputs(c, rows, g)
    p = c["p"]
    keep = (torch.rand(rows, c["C"], generator=g) >= p).to(F64) if p > 0 else None
    f = eo.layernorm_forward(t["x"], t["res"], t["gamma"], t["beta"], c["eps"], keep, p, t["pos"])
    x = t["x"].to(F64).requires_grad_(True)
    res = None if t["res"] is None else t["res"].to(F64).requires_grad_(True)
    gamma = t["gamma"].to(F64).requires_grad_(True)
    beta = t["beta"].to(F64).requires_grad_(True)
    xin = x if keep is None else x * keep / (1 - p)
    if res is not None:
        xin = xin + res
    y = F.layer_norm(xin, (c["C"],), gamma, beta, c["eps"])
    torch.testing.assert_close(f["y"], y.detach(), rtol=0, atol=1e-11)
    if t["pos"] is not None:
        torch.testing.assert_close(f["y2"], (y + t["pos"].to(F64)).detach(), rtol=0, atol=1e-11)
    dy = t["dy"].to(F64)
    up = dy if t["dy2"] is None else dy + t["dy2"].to(F64)
    y.backward(up)
    b = eo.layernorm_backward(t["x"], t["res"], t["gamma"], c["eps"], t["dy"], t["dy2"], keep, p)
    scale = up.abs().max().item() * f["rstd"].max().item()
    torch.testing.assert_close(b["dx"], x.grad, rtol=0, atol=1e-11 * scale)
    if res is not None:
        torch.testing.assert_close(b["dres"], res.grad, rtol=0, atol=1e-11 * scale)
    torch.testing.assert_close(b["dgamma"], gamma.grad, rtol=1e-11, atol=1e-9)
    torch.testing.assert_close(b["dbeta"], beta.grad, rtol=1e-11, atol=1e-9)
    if c["data"] == "const":
        assert (f["xhat"][::3] == 0).all() and (f["y"][::3] == t["beta"].to(F64)).all()


# ------------------------------------------------------------------------------------------------
# SCA combine, reductions, elementwise
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", eo.combine_cases(), ids=eo.combine_case_id)
def test_sca_combine_restatement(c):
    """slots / its backward against a per-query loop over the cameras (count clamped to 1)."""
    B, Nq, C, ncam = c["B"], c["Nq"], c["C"], c["ncam"]
    g = torch.Generator().manual_seed(17)
    pq, pc, pair_of = eo.make_pairs(Nq, ncam, seed=3)
    R = pq.numel()
    out = torch.randn(B * R, C, generator=g).to(DT[c["dt"]])
    slots = eo.sca_combine_forward(out, pq, B, Nq)
    gs = torch.randn(B, Nq, C, generator=g).to(DT[c["dt"]])
    gout = eo.sca_combine_backward(gs, pq, B, Nq)
    o = out.to(F64).reshape(B, R, C)
    for q in range(Nq):
        rows = [int(pair_of[k, q]) for k in range(ncam) if pair_of[k, q] >= 0]
        want = sum((o[:, r] for r in rows), torch.zeros(B, C, dtype=F64)) / max(1, len(rows))
        torch.testing.assert_close(slots[:, q], want, rtol=0, atol=1e-14)
    for r in range(R):
        got = gout.reshape(B, R, C)[:, r]
        if pq[r] < 0:
            assert torch.isnan(got).all()
        else:
            n = int((pair_of[:, pq[r]] >= 0).sum())
            torch.testing.assert_close(got, gs[:, pq[r]].to(F64) / n, rtol=0, atol=0)


@pytest.mark.parametrize("c", eo.colsum_cases(), ids=eo.colsum_case_id)
def test_colsum_restatement(c):
    rows = eo.colsum_rows(c["rows"], eo.H100_SMS)
    g = torch.Generator().manual_seed(19)
    x = torch.randn(rows, c["C"], generator=g).to(DT[c["dt"]])
    out0 = torch.randn(c["C"], generator=g) if c["acc"] else None
    s, a = eo.colsum(x, out0)
    xn = x.to(F64).numpy()
    want = xn.sum(0) + (0 if out0 is None else out0.double().numpy())
    np.testing.assert_allclose(s.numpy(), want, rtol=1e-12, atol=1e-9)
    assert (a.numpy() >= np.abs(want) - 1e-9).all()
    rpc, grid = eo.colsum_plan(rows, eo.H100_SMS)
    if c["rows"] == "cta+1":
        assert rows == (grid - 1) * rpc + 1 and grid == 4 * eo.H100_SMS


@pytest.mark.parametrize("c", eo.sum_cases(), ids=eo.sum_case_id)
def test_sum_tensors_restatement(c):
    g = torch.Generator().manual_seed(23)
    ts = [torch.randn(c["numel"], generator=g).to(DT[c["dt"]]) for _ in range(c["n"])]
    s, a = eo.sum_tensors(ts)
    want = np.sum(np.stack([t.to(F64).numpy() for t in ts]), 0)
    np.testing.assert_allclose(s.numpy(), want, rtol=1e-15, atol=1e-15)
    np.testing.assert_array_equal(a.numpy(), np.sum(np.abs(np.stack([t.to(F64).numpy() for t in ts])), 0))


@pytest.mark.parametrize("c", eo.dropout_cases(), ids=eo.dropout_case_id)
def test_dropout_restatements(c):
    """Kept values are x * fl32(1 / (1 - p)) rounded in fp32, then to storage; the relu-dropout backward passes dy
    times that scale where h != 0."""
    g = torch.Generator().manual_seed(29)
    dt = DT[c["dt"]]
    s32 = eo.dropout_scale32(c["p"])
    assert s32 == float(np.float32(1.0) / (np.float32(1.0) - np.float32(c["p"])))
    x = torch.randn(c["numel"], generator=g).to(dt)
    want = (x.float().numpy() * np.float32(s32)).astype(np.float32)
    np.testing.assert_array_equal(eo.dropout_kept(x, s32).float().numpy(),
                                  torch.from_numpy(want).to(dt).float().numpy())
    h = torch.where(torch.rand(c["numel"], generator=g) < 0.5, torch.zeros((), dtype=dt), x)
    dy = torch.randn(c["numel"], generator=g).to(dt)
    got = eo.relu_dropout_backward(dy, h, s32)
    want = np.where(h.float().numpy() != 0, (dy.float().numpy() * np.float32(s32)).astype(np.float32), 0)
    np.testing.assert_array_equal(got.float().numpy(), torch.from_numpy(want).to(dt).float().numpy())


def test_shared_case_lists_cover_the_dispatch_branches():
    """The case lists reach every instantiation the GPU file asserts through the profiler."""
    ppl_tsa = {c["L"] * c["P"] // 2 for c in eo.tsa_cases() if c["M"] == 8 and c["L"] * c["P"] in (2, 4, 8, 16, 32)}
    assert ppl_tsa == {1, 2, 4, 8, 16}
    assert {(c["M"], c["L"] * c["P"]) for c in eo.tsa_cases()} >= {(4, 12), (6, 12)}
    ppl_sca = {c["L"] * c["P"] // 4 for c in eo.sca_cases() if c["M"] == 8 and c["L"] * c["P"] in (4, 8, 16, 32, 64)}
    assert ppl_sca == {1, 2, 4, 8, 16}
    assert {c["D"] for c in eo.sca_cases()} == {1, 2, 4} and max(c["ncam"] for c in eo.sca_cases()) == 16
    ln = eo.ln_cases()
    assert {(c["C"], c["adt"], c["pdt"]) for c in ln} == {(C, a, p) for C in (256, 512) for a, p in eo.LN_DTYPES}
    for key in ("res", "pos", "twin", "strided"):
        assert {c[key] for c in ln} == {False, True}
    assert {c["p"] for c in ln} == {0.0, 0.3} and {c["eps"] for c in ln} == {1e-5, 1e-1}
    assert {c["rows"] for c in ln} >= set(eo.LN_ROWS)
    assert {c["C"] for c in eo.colsum_cases()} == set(eo.COLSUM_C)
    assert {c["n"] for c in eo.sum_cases()} == set(range(1, 9))


# ------------------------------------------------------------------------------------------------
# argument checks of the C entry points (no device: every call below returns before any launch, or fails its launch)
# ------------------------------------------------------------------------------------------------
A, MIS = 1 << 20, (1 << 20) + 4            # fake device addresses: 16-byte aligned / 4 bytes past


def _refuses(fn, args, bad_index, what):
    from bevformer_b200 import _lib
    lib = _lib.load()
    good = list(args)
    st = getattr(lib, fn)(*good)
    # all-aligned arguments pass the checks and reach the launch, which fails on a host without a device
    assert b"aligned" not in lib.bevf_last_error()
    for i in bad_index:
        a = list(args)
        a[i] = MIS
        assert getattr(lib, fn)(*a) != 0, (fn, i)
        msg = lib.bevf_last_error()
        assert b"16-byte aligned" in msg and what in msg, (fn, i, msg)
    return st


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers must never reach a device")
def test_entry_points_refuse_misaligned_vector_operands():
    """Every pointer that a kernel reads or writes with 16 B vectors is refused 4 bytes off alignment; the scalar and
    atomic ones (LayerNorm mean / rstd / dgamma / dbeta, colsum's out, inv_count) are not."""
    from bevformer_b200 import _lib, ops
    lib = _lib.load()
    f32, bf = ops.F32, ops.BF16
    hw = A
    # prep: raw, loc / d_raw
    _refuses("bevf_sca_prep_forward", [A, A, A, A, hw, A, A, 1, 4, 4, 8, 4, 8, 4, 6, None], [0, 5], b"raw")
    _refuses("bevf_sca_prep_backward", [A, A, A, A, hw, A, f32, 1, 4, 4, 8, 4, 8, 6, None], [0, 5], b"d_raw")
    _refuses("bevf_sca_prep_backward_multi", [A, A, A, A, hw, A, bf, 1, 4, 4, 8, 4, 8, 6, None], [0, 5], b"d_raw")
    _refuses("bevf_tsa_prep_forward", [A, A, hw, A, A, 1, 4, 8, 1, 4, 0, None], [0, 3], b"loc")
    _refuses("bevf_tsa_prep_backward", [A, A, A, hw, A, f32, 1, 4, 8, 1, 4, 0, None], [0, 4], b"d_raw")
    # LayerNorm forward: x, residual, gamma, beta, param_dtype, pos, y, y_plus_pos, mean, rstd, rows, C, eps, p, seed,
    # seed_base, dtype, stream
    fwd = [A, A, A, A, f32, A, A, A, A, A, 8, 256, 1e-5, 0.0, 0, None, f32, None]
    _refuses("bevf_layernorm_forward", fwd, [0, 1, 5, 6, 7], b"y_plus_pos")
    scalar = list(fwd)
    for i in (2, 3, 8, 9):                             # gamma, beta, mean, rstd: scalar accesses
        scalar[i] = MIS
    lib.bevf_layernorm_forward(*scalar)
    assert b"aligned" not in lib.bevf_last_error()
    # LayerNorm backward: x, residual, gamma, pd, mean, rstd, dy, dy2, ld2, dx, dres, dgamma, dbeta, rows, C, p, seed,
    # seed_base, dtype, stream
    bwd = [A, A, A, f32, A, A, A, A, 0, A, A, A, A, 8, 256, 0.0, 0, None, f32, None]
    _refuses("bevf_layernorm_backward", bwd, [0, 1, 6, 7, 9, 10], b"dres")
    scalar = list(bwd)
    for i in (2, 4, 5, 11, 12):                        # gamma, mean, rstd, dgamma, dbeta
        scalar[i] = MIS
    lib.bevf_layernorm_backward(*scalar)
    assert b"aligned" not in lib.bevf_last_error()
    det = bwd[:13] + [A, 1 << 30] + bwd[13:]
    _refuses("bevf_layernorm_backward_det", det, [0, 1, 6, 7, 9, 10], b"dres")
    # colsum: x only (out is atomic)
    _refuses("bevf_colsum", [A, A, 64, 256, f32, None], [0], b"x")
    lib.bevf_colsum(A, MIS, 64, 256, f32, None)
    assert b"aligned" not in lib.bevf_last_error()
    _refuses("bevf_colsum_det", [A, A, A, 1 << 30, 64, 256, f32, None], [0], b"x")
    # SCA combine: out, slots / g_slots, g_out (inv_count scalar)
    _refuses("bevf_sca_combine_forward", [A, A, A, A, 1, 8, 8, 256, 6, f32, None], [0, 3], b"slots")
    lib.bevf_sca_combine_forward(A, A, MIS, A, 1, 8, 8, 256, 6, f32, None)
    assert b"aligned" not in lib.bevf_last_error()
    _refuses("bevf_sca_combine_backward", [A, A, A, A, 1, 8, 8, 256, f32, None], [0, 3], b"g_out")
    _refuses("bevf_dropout_inplace", [A, 64, 0.3, 0, None, f32, None], [0], b"x")
    _refuses("bevf_relu_dropout_backward", [A, A, A, 64, 1.5, f32, None], [0, 1, 2], b"h")

