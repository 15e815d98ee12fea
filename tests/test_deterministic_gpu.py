"""Deterministic mode (torch.use_deterministic_algorithms(True)) on the GPU: every backward of the package that sums
through atomics by default -- sampler grad_value, LayerNorm dgamma / dbeta, bias column sums, weight gradients --
gives bit-identical results from run to run, and stays within the accuracy bars of the default kernels.

PyTorch's NaN fill of uninitialised memory stays ON here (its default under the flag): a workspace or output that a
kernel does not fully overwrite shows up as NaN."""
import math
import warnings

import pytest
import torch

from bevformer_b200 import _lib, ops, synthetic as syn
from oracle import msda_oracle
from tests.util import fixed_projection, golden, max_err, rel_err, stats

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float32: 1e-3, torch.bfloat16: 1e-2}


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _rig(which):
    from tools.bench_msda import rig_sca_inputs, rig_tsa_inputs, rig_tsa_rows_inputs
    if which == "sca":
        v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
        return v, ss, lsi, loc, attn, row_map, None
    if which == "tsa_rows":
        return rig_tsa_rows_inputs(DEV)
    v, ss, lsi, loc, attn = rig_tsa_inputs(DEV)
    return v, ss, lsi, loc, attn, None, None


def _backward(vd, ss, lsi, loc, attn, row_map, gout, order=None):
    if row_map is not None:
        return ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout, group_order=order)
    return ops.msda_backward(vd, ss, lsi, loc, attn, gout.view(loc.shape[0], loc.shape[1], -1))


def _oracle(vd, ss, lsi, loc, attn, row_map, gout, dtype=torch.float32):
    vr, gr = vd.to(dtype).cpu(), gout.to(dtype).cpu()
    loc_c, attn_c = loc.to(dtype).cpu(), attn.to(dtype).cpu()
    if row_map is None:
        return msda_oracle.msda_backward(vr, ss.cpu(), lsi.cpu(), loc_c, attn_c, gr.view(*loc.shape[:2], -1))
    rm = row_map.cpu().long()
    rgv = torch.zeros(vr.shape, dtype=dtype)
    rgl = torch.zeros(loc_c.shape, dtype=dtype)
    rga = torch.zeros(attn_c.shape, dtype=dtype)
    for b in range(vr.shape[0]):
        idx = (rm == b).nonzero().flatten()
        if idx.numel():
            a, g, c = msda_oracle.msda_backward(vr[b:b + 1], ss.cpu(), lsi.cpu(), loc_c[idx][None].contiguous(),
                                                attn_c[idx][None].contiguous(), gr[idx][None].contiguous())
            rgv[b] = a[0]; rgl[idx] = g[0]; rga[idx] = c[0]
    return rgv, rgl, rga


@pytest.mark.parametrize("which", ["sca", "tsa", "tsa_rows"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_base_rig_reproducible_and_accurate(which, dtype, det):
    """The base launches (geometry of test_base_rig_geometry_against_oracle): two runs give the same bits; grad_value
    holds the Oracle-S bars; grad_loc / grad_attn are those of the default path bit for bit."""
    v, ss, lsi, loc, attn, row_map, order = _rig(which)
    vd = v.to(dtype)
    nrows = loc.shape[0] if row_map is not None else loc.shape[0] * loc.shape[1]
    gout = fixed_projection((nrows, 256)).to(DEV, dtype)
    a = _backward(vd, ss, lsi, loc, attn, row_map, gout, order)
    b = _backward(vd, ss, lsi, loc, attn, row_map, gout, order)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    torch.use_deterministic_algorithms(False)
    _, gl0, ga0 = _backward(vd, ss, lsi, loc, attn, row_map, gout, order)
    torch.use_deterministic_algorithms(True)
    assert torch.equal(a[1], gl0) and torch.equal(a[2], ga0)
    rgv, _, _ = _oracle(vd.float(), ss, lsi, loc, attn, row_map, gout.float())
    e = rel_err(a[0].cpu(), rgv)
    print(which, dtype, "fixed-point grad_value vs Oracle-S", e)
    assert e < TOL[dtype]


def test_row_permutation_leaves_grad_value_unchanged(det):
    """Rows permuted together with their grad_out rows: grad_value is the same bit for bit (the fp32 reductions of the
    default path cannot promise this)."""
    v, ss, lsi, loc, attn, row_map, _ = _rig("sca")
    gout = fixed_projection((loc.shape[0], 256)).to(DEV)
    gv, gl, ga = ops.msda_rows_backward(v, ss, lsi, loc, attn, row_map, gout)
    perm = torch.randperm(loc.shape[0], generator=torch.Generator().manual_seed(0)).to(DEV)
    gv_p, gl_p, ga_p = ops.msda_rows_backward(v, ss, lsi, loc[perm].contiguous(), attn[perm].contiguous(),
                                              row_map[perm].contiguous(), gout[perm].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(gv, gv_p)
    assert torch.equal(gl[perm], gl_p) and torch.equal(ga[perm], ga_p)


@pytest.mark.parametrize("dim", [4, 30, 32, 64, 71, 1025])
def test_head_dims_against_oracle(dim, det):
    """The generic head_dim kernel's fixed-point form (and head_dim 32's): Oracle-S bars of the default path, two runs
    identical."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(6, 4), (3, 2)], 9, 2, dim, 2, seed=dim, loc_range=(-0.3, 1.3))
    gout = fixed_projection((2, 9, 2 * dim))
    args = (v.to(DEV), ss.to(DEV), lsi.to(DEV), loc.to(DEV), attn.to(DEV), gout.to(DEV))
    gv, gl, ga = ops.msda_backward(*args)
    gv2, gl2, ga2 = ops.msda_backward(*args)
    torch.cuda.synchronize()
    assert torch.equal(gv, gv2) and torch.equal(gl, gl2) and torch.equal(ga, ga2)
    rgv, rgl, rga = msda_oracle.msda_backward(v, ss, lsi, loc, attn, gout)
    assert max_err(gv.cpu(), rgv) < 1e-4 and max_err(gl.cpu(), rgl) < 1e-3 and max_err(ga.cpu(), rga) < 1e-4


def _fx_bound(attn, gout, rows_per_map, L, P):
    """Documented rounding bound of the fixed-point sum: n_max * 2^(E - K - 1)."""
    k = _lib.load().bevf_msda_fx_frac_bits(rows_per_map, L, P)
    e = math.frexp(attn.abs().max().item())[1] + math.frexp(gout.abs().max().item())[1]
    return rows_per_map * L * P * 4 * 2.0 ** (e - k - 1)


@pytest.mark.parametrize("dim", [32, 71])
def test_fp64_oracle_within_fixed_point_bound(dim, det):
    """Against Oracle-S in fp64: the difference is the fp32 rounding of the factors w * attn (2^-22 relative per
    contribution), the documented fixed-point bound and the final rounding to fp32 -- nothing else.  Locations are
    multiples of 2^-12, so loc * W - 0.5 and the bilinear fractions are exact in fp32 as in fp64."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(12, 10), (6, 5)], 300, 4, dim, 4, seed=7, loc_range=(-0.2, 1.2))
    loc = torch.round(loc * 4096) / 4096
    gout = fixed_projection((2, 300, 4 * dim)) * 3.0
    gv, _, _ = ops.msda_backward(v.to(DEV), ss.to(DEV), lsi.to(DEV), loc.to(DEV), attn.to(DEV), gout.to(DEV))
    torch.cuda.synchronize()
    ref, _, _ = msda_oracle.msda_backward(v.double(), ss, lsi, loc.double(), attn.double(), gout.double())
    mass, _, _ = msda_oracle.msda_backward(v.double(), ss, lsi, loc.double(), attn.double().abs(), gout.double().abs())
    bound = 2.0 ** -21 * mass + _fx_bound(attn, gout, 300, 2, 4) + 2.0 ** -24 * ref.abs()
    err = (gv.cpu().double() - ref).abs()
    assert torch.all(err <= bound), (err - bound).max().item()


def test_one_pixel_adversarial(det):
    """Every sample of 131072 rows on one pixel with weight 1 and attn 1: the most contributions an element can take
    at K = 40 with nothing cancelling -- no overflow, the exact sum within the bound."""
    R, P = 131072, 8
    ss = torch.tensor([[1, 1]], device=DEV); lsi = torch.tensor([0], device=DEV)
    value = torch.randn(1, 1, 1, 32, device=DEV)
    loc = torch.full((R, 1, 1, P, 2), 0.5, device=DEV)
    attn = torch.ones(R, 1, 1, P, device=DEV)
    g = 1.999755859375                                    # just below 2: contributions just below 2^E / 2
    gout = torch.full((R, 32), g, device=DEV)
    row_map = torch.zeros(R, dtype=torch.int32, device=DEV)
    gv, _, _ = ops.msda_rows_backward(value, ss, lsi, loc, attn, row_map, gout)
    torch.cuda.synchronize()
    exact = R * P * g
    assert _lib.load().bevf_msda_fx_frac_bits(R, 1, P) == 40
    assert torch.all((gv.double() - exact).abs() <= _fx_bound(attn, gout, R, 1, P) + 2.0 ** -24 * exact)


def test_zero_and_non_finite_inputs(det):
    """All-zero grad_out: zero gradients.  inf / NaN in attn or grad_out of a LIVE row: grad_value is NaN everywhere
    (documented in the header); NaN in an unused row (row_map -1) does not count."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(3, [(9, 16)], 200, 8, 32, 4, seed=5, device=DEV)
    loc, attn = loc.flatten(0, 1).contiguous(), attn.flatten(0, 1).contiguous()
    row_map = torch.arange(3, device=DEV, dtype=torch.int32).repeat_interleave(200).contiguous()
    row_map[17:23] = -1
    gout = fixed_projection((600, 256)).to(DEV)
    gv, gl, ga = ops.msda_rows_backward(v, ss, lsi, loc, attn, row_map, torch.zeros_like(gout))
    used = row_map >= 0                     # (grad_loc / grad_attn of unused rows are not written, as by default)
    assert gv.abs().max().item() == 0 and gl[used].abs().max().item() == 0 and ga[used].abs().max().item() == 0
    base, _, _ = ops.msda_rows_backward(v, ss, lsi, loc, attn, row_map, gout)
    assert torch.isfinite(base).all()
    g_unused = gout.clone(); g_unused[18] = float("nan")
    a_unused = attn.clone(); a_unused[19] = float("inf")
    gv, _, _ = ops.msda_rows_backward(v, ss, lsi, loc, a_unused, row_map, g_unused)
    assert torch.equal(gv, base)
    for bad in ("nan_grad", "inf_grad", "nan_attn", "inf_attn"):
        g2, a2 = gout.clone(), attn.clone()
        x = float("nan") if bad.startswith("nan") else float("inf")
        if bad.endswith("grad"):
            g2[5, 7] = x
        else:
            a2[5, 0, 0, 1] = x
        gv, _, _ = ops.msda_rows_backward(v, ss, lsi, loc, a2, row_map, g2)
        assert torch.isnan(gv).all(), bad
    g2 = gout.to(torch.bfloat16)
    g2[5, 7] = float("nan")
    gv, _, _ = ops.msda_rows_backward(v.to(torch.bfloat16), ss, lsi, loc, attn, row_map, g2)
    assert torch.isnan(gv).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum_layernorm_wgrad(dtype, det):
    """The ordered reductions: bit-identical twice, and within the default kernels' bars of an fp64 reference."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(40000, 256, generator=g).to(DEV, dtype)
    c1, c2 = ops.colsum(x), ops.colsum(x)
    assert torch.equal(c1, c2) and rel_err(c1, x.double().sum(0)) < 1e-5

    xs = torch.randn(2, 2500, 256, generator=g).to(DEV, dtype)
    res = torch.randn(2, 2500, 256, generator=g).to(DEV, dtype)
    gamma = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV, dtype).requires_grad_(True)
    beta = (0.1 * torch.randn(256, generator=g)).to(DEV, dtype).requires_grad_(True)
    dy = torch.randn(2, 2500, 256, generator=g).to(DEV, dtype)

    def ln_grads():
        gamma.grad = beta.grad = None
        xi = xs.clone().requires_grad_(True)
        ops.LayerNormResidual.apply(xi, res, gamma, beta, 1e-5, 0.0).backward(dy)
        return gamma.grad.clone(), beta.grad.clone(), xi.grad.clone()

    a, b = ln_grads(), ln_grads()
    for p, q in zip(a, b):
        assert torch.equal(p, q)
    torch.use_deterministic_algorithms(False)
    ref = ln_grads()
    torch.use_deterministic_algorithms(True)
    tol = 1e-5 if dtype == torch.float32 else 1e-2              # bf16: the gradients are stored in bf16
    for p, q in zip(a, ref):
        assert rel_err(p.float(), q.float()) < tol

    dyw = torch.randn(30000, 512, generator=g).to(DEV, torch.bfloat16)
    xw = torch.randn(30000, 256, generator=g).to(DEV, torch.bfloat16)
    dw1, db1 = ops.linear_wgrad_tc(dyw, xw, with_bias=True)
    dw2, db2 = ops.linear_wgrad_tc(dyw, xw, with_bias=True)
    assert torch.equal(dw1, dw2) and torch.equal(db1, db2)
    assert rel_err(dw1, dyw.double().t() @ xw.double()) < 1e-5 and rel_err(db1, dyw.double().sum(0)) < 1e-5
    acc_w = torch.randn(512, 256, generator=g).to(DEV)
    acc_b = torch.randn(512, generator=g).to(DEV)
    w0, b0 = acc_w.clone(), acc_b.clone()
    ops.linear_wgrad_into(dyw, xw, acc_w, acc_b)                # the gradient arena's accumulate-into form
    assert rel_err(acc_w, w0.double() + dyw.double().t() @ xw.double()) < 1e-5
    assert rel_err(acc_b, b0.double() + dyw.double().sum(0)) < 1e-5
    acc2_w, acc2_b = w0.clone(), b0.clone()
    ops.linear_wgrad_into(dyw, xw, acc2_w, acc2_b)
    assert torch.equal(acc_w, acc2_w) and torch.equal(acc_b, acc2_b)


def _reset_dropout_keys():
    """What a fresh process starts from: the per-site Philox keys and the device step counter."""
    ops._seed_counter[0] = 0
    ops._seed_state.clear()
    ops._seed_snap.clear()


@pytest.mark.parametrize("workload", ["tiny", "base"])
def test_encoder_train_step_reproducible(workload, det):
    """bf16, train mode with dropout, gradient arena with the side-stream overlap: two forward + backward passes from
    the same state give bit-identical gradients for every parameter and input."""
    w = syn.WORKLOADS[workload]
    from bevformer_b200.plugin import build_transformer_layer_sequence
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w))
    enc = enc.to(DEV, torch.bfloat16).train()
    enc.enable_grad_arena(overlap=True)
    inp = syn.make_encoder_inputs(w, bs=1, seed=0)
    for k in ("bev_query", "feat", "bev_pos", "prev_bev"):
        setattr(inp, k, getattr(inp, k).to(DEV, torch.bfloat16))
    inp.shift = inp.shift.to(DEV)
    inp.spatial_shapes, inp.level_start_index = inp.spatial_shapes.to(DEV), inp.level_start_index.to(DEV)
    proj = fixed_projection((1, w.num_query, 256)).to(DEV, torch.bfloat16)

    def run():
        _reset_dropout_keys()
        for p in enc.parameters():
            p.grad = None
        q = inp.bev_query.detach().clone().requires_grad_(True)
        f = inp.feat.detach().clone().requires_grad_(True)
        out = enc(q, f, f, **inp.kwargs())
        (out * proj).sum().backward()
        torch.cuda.synchronize()
        return out.detach().clone(), q.grad.clone(), f.grad.clone(), {k: p.grad.clone() for k, p in enc.named_parameters()}

    a, b = run(), run()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert a[3].keys() == b[3].keys()
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k


@pytest.mark.parametrize("workload", ["tiny", "base"])
def test_encoder_bf16_tracks_fp32_reference(workload, det):
    """The bars of test_backward_bf16_tracks_fp32_reference hold in deterministic mode."""
    g = golden("encoder_" + workload)
    w = syn.WORKLOADS[workload]
    from bevformer_b200.plugin import build_transformer_layer_sequence
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w, seed=0))
    enc = enc.to(DEV, torch.bfloat16).eval()
    inp = syn.make_encoder_inputs(w, bs=1, seed=0, with_prev=True)
    for k in ("bev_query", "feat", "bev_pos", "prev_bev"):
        setattr(inp, k, getattr(inp, k).to(DEV, torch.bfloat16))
    inp.shift = inp.shift.to(DEV)
    inp.spatial_shapes, inp.level_start_index = inp.spatial_shapes.to(DEV), inp.level_start_index.to(DEV)
    for t in (inp.bev_query, inp.feat, inp.bev_pos):
        t.requires_grad_(True)
    out = enc(inp.bev_query, inp.feat, inp.feat, **inp.kwargs())
    (out.float() * fixed_projection(out.shape).to(DEV)).sum().backward()
    torch.cuda.synchronize()
    for got, want in ((inp.bev_query.grad.float().cpu()[g["rows_q"]], g["grad_query_rows"]),
                      (inp.feat.grad.float().cpu()[:, g["rows_s"]], g["grad_feat_rows"]),
                      (inp.bev_pos.grad.float().cpu()[g["rows_q"]], g["grad_pos_rows"])):
        want = torch.from_numpy(want)
        cos = torch.nn.functional.cosine_similarity(got.double().flatten(), want.double().flatten(), dim=0).item()
        assert cos > 0.99 and ((got - want).norm() / want.norm()).item() < 0.12
    for k, p in enc.named_parameters():
        got, ref = stats(p.grad.float()), g["gstat:" + k]
        assert abs(got[2] - ref[2]) / max(ref[2], 1e-12) <= 0.10, k


def test_decoder_attention_reproducible(det):
    """CustomMSDeformableAttention (the op-class path through MultiScaleDeformableAttnFunction_fp32): two backward
    passes give the same bits."""
    from bevformer_b200.plugin import CustomMSDeformableAttention
    from tests.test_decoder_attention import make_case, make_sd
    levels, points = [(50, 50)], 4
    m = CustomMSDeformableAttention(num_levels=1, num_points=points)
    m.load_state_dict(make_sd(levels, points))
    m = m.to(DEV).eval()                 # (its output dropout draws from PyTorch's generator)
    case = make_case(levels, 900, 1, 2)
    proj = fixed_projection((900, 1, 256)).to(DEV)

    def run():
        m.zero_grad(set_to_none=True)
        q = case["query"].to(DEV).requires_grad_(True)
        v = case["value"].to(DEV).requires_grad_(True)
        out = m(q, value=v, query_pos=case["query_pos"].to(DEV), reference_points=case["reference_points"].to(DEV),
                spatial_shapes=case["spatial_shapes"].to(DEV), level_start_index=case["level_start_index"].to(DEV))
        (out * proj).sum().backward()
        return [q.grad, v.grad] + [p.grad for p in m.parameters()]

    for x, y in zip(run(), run()):
        assert torch.equal(x, y)


def test_dispatch(det, monkeypatch):
    """Flag off: the default kernels (the fixed-point path never runs).  Flag on: a backward without a deterministic
    implementation raises, or warns and runs under warn_only."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(9, 16)], 100, 8, 32, 4, seed=1, device=DEV)
    loc, attn = loc.flatten(0, 1).contiguous(), attn.flatten(0, 1).contiguous()
    row_map = torch.arange(2, device=DEV, dtype=torch.int32).repeat_interleave(100).contiguous()
    vd = v.to(torch.bfloat16)
    gout = fixed_projection((200, 256)).to(DEV, torch.bfloat16)
    with pytest.raises(RuntimeError, match="deterministic"):
        ops.msda_rows_backward_f16acc(vd, ss, lsi, loc, attn, row_map, gout)
    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gv, _, _ = ops.msda_rows_backward_f16acc(vd, ss, lsi, loc, attn, row_map, gout)
    assert gv.shape == v.shape and any("deterministic" in str(r.message) for r in rec)
    torch.use_deterministic_algorithms(False)

    def boom(*a, **k):
        raise AssertionError("fixed-point path used with the flag off")
    monkeypatch.setattr(ops, "msda_backward_fx", boom)
    ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout)
    ops.msda_backward(v, ss, lsi, loc.view(2, 100, 8, 1, 4, 2), attn.view(2, 100, 8, 1, 4),
                      fixed_projection((2, 100, 256)).to(DEV))
