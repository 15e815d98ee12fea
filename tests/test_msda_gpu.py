"""GPU parity tests of the sampler THROUGH THE C ABI (ops.py -> ctypes -> libbevformer_b200.so)
against (a) the committed golden vectors made from the reference's own modules and (b) Oracle-S
run on the same seeded inputs.  Bars: 1e-3 for fp32 storage, 1e-2 for bf16 storage
(BASELINE.json north_star), read as max|err| / max(1, max|ref|)."""
import numpy as np
import pytest
import torch

from bevformer_b200 import ops, synthetic as syn
from oracle import msda_oracle
from tests.util import fixed_projection, golden, max_err, msda_case_inputs, rel_err, stats, stats_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float32: 1e-3, torch.bfloat16: 1e-2}


def _run(v, ss, lsi, loc, attn, gout, dtype):
    vd = v.to(DEV, dtype).contiguous()
    out = ops.msda_forward(vd, ss.to(DEV), lsi.to(DEV), loc.to(DEV).float().contiguous(),
                           attn.to(DEV).float().contiguous())
    gv, gl, ga = ops.msda_backward(vd, ss.to(DEV), lsi.to(DEV), loc.to(DEV).float().contiguous(),
                                   attn.to(DEV).float().contiguous(),
                                   gout.to(DEV, dtype).contiguous())
    torch.cuda.synchronize()
    return out.float().cpu(), gv.cpu(), gl.cpu(), ga.cpu()


@pytest.mark.parametrize("case", ["kat", "kat_oob", "config0", "pyramid"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_against_golden(case, dtype):
    g = golden("msda_" + case)
    v, ss, lsi, loc, attn = msda_case_inputs(g, torch.float32)
    gout = fixed_projection((v.shape[0], loc.shape[1], v.shape[2] * v.shape[3]))
    out, gv, gl, ga = _run(v, ss, lsi, loc, attn, gout, dtype)
    rq, rs = g["rows_q"], g["rows_s"]
    tol = TOL[dtype]
    assert rel_err(out[:, rq], g["out_rows"]) < tol
    assert rel_err(gv[:, rs], g["grad_value_rows"]) < tol
    assert rel_err(ga[:, rq], g["grad_attn_rows"]) < tol
    assert rel_err(gl[:, rq], g["grad_loc_rows"]) < tol * 4   # carries the W_l / H_l factors
    assert stats_close(stats(out), g["out_stats"], 10 * tol)
    assert stats_close(stats(gv), g["grad_value_stats"], 10 * tol)


@pytest.mark.parametrize("dim", [4, 30, 32, 64, 71, 1025])   # mmcv's gradcheck channel list
def test_head_dims_against_oracle(dim):
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(6, 4), (3, 2)], 9, 2, dim, 2, seed=dim,
                                                 loc_range=(-0.3, 1.3))
    gout = fixed_projection((2, 9, 2 * dim))
    out, gv, gl, ga = _run(v, ss, lsi, loc, attn, gout, torch.float32)
    ref = msda_oracle.msda_forward(v, ss, lsi, loc, attn)
    rgv, rgl, rga = msda_oracle.msda_backward(v, ss, lsi, loc, attn, gout)
    assert max_err(out, ref) < 1e-4
    assert max_err(gv, rgv) < 1e-4 and max_err(gl, rgl) < 1e-3 and max_err(ga, rga) < 1e-4


@pytest.mark.parametrize("shape", [
    dict(bs=1, levels=[(1, 1)], nq=1, heads=1, pts=1),            # smallest possible
    dict(bs=3, levels=[(7, 5)], nq=33, heads=3, pts=5),           # ragged: heads not a power of two
    dict(bs=2, levels=[(9, 11), (5, 6), (3, 3), (2, 2), (1, 1)], nq=65, heads=8, pts=3),
    dict(bs=6, levels=[(15, 25)], nq=592, heads=8, pts=8),        # tiny's SCA shape (max_len 592)
])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_shapes_against_oracle(shape, dtype, backward_mode):
    v, ss, lsi, loc, attn = syn.make_msda_inputs(shape["bs"], shape["levels"], shape["nq"],
                                                 shape["heads"], 32, shape["pts"], seed=2,
                                                 loc_range=(-0.2, 1.2))
    if dtype == torch.bfloat16:   # compare against the oracle on the SAME (bf16-rounded) inputs
        v = v.to(dtype).float()
    gout = fixed_projection((shape["bs"], shape["nq"], shape["heads"] * 32))
    if dtype == torch.bfloat16:
        gout = gout.to(dtype).float()
    out, gv, gl, ga = _run(v, ss, lsi, loc, attn, gout, dtype)
    ref = msda_oracle.msda_forward(v, ss, lsi, loc, attn)
    rgv, rgl, rga = msda_oracle.msda_backward(v, ss, lsi, loc, attn, gout)
    otol = 1e-4 if dtype == torch.float32 else 1e-2       # bf16 output rounding
    assert rel_err(out, ref) < otol
    assert rel_err(gv, rgv) < 1e-4 and rel_err(ga, rga) < 1e-4 and rel_err(gl, rgl) < 1e-3


def test_empty_and_extreme_locations():
    ss = torch.tensor([[4, 5]], device=DEV); lsi = torch.tensor([0], device=DEV)
    value = torch.randn(1, 20, 1, 32, device=DEV)
    out = ops.msda_forward(value, ss, lsi, torch.zeros(1, 0, 1, 1, 1, 2, device=DEV),
                           torch.zeros(1, 0, 1, 1, 1, device=DEV))
    assert out.shape == (1, 0, 32)
    far = torch.tensor([[-0.5 / 5 - 1e-6, 0.5], [1.0 + 0.5 / 5, 0.5], [0.5, -0.125 - 1e-6],
                        [0.5, 1.125], [1e9, 0.5], [0.5, -1e9], [float("nan"), 0.5],
                        [float("inf"), 0.5]], device=DEV).view(1, 8, 1, 1, 1, 2)
    w = torch.ones(1, 8, 1, 1, 1, device=DEV)
    out = ops.msda_forward(value, ss, lsi, far.contiguous(), w)
    assert out.abs().max().item() == 0.0
    gv, gl, ga = ops.msda_backward(value, ss, lsi, far.contiguous(), w, torch.ones_like(out))
    assert gv.abs().max().item() == 0.0 and gl.abs().max().item() == 0.0 and ga.abs().max().item() == 0.0


def test_pixel_centres_reproduce_value_and_permutation():
    ss = torch.tensor([[6, 7]], device=DEV); lsi = torch.tensor([0], device=DEV)
    value = torch.randn(2, 42, 8, 32, device=DEV)
    ys, xs = torch.meshgrid(torch.arange(6.0), torch.arange(7.0), indexing="ij")
    loc = torch.stack([(xs + 0.5) / 7, (ys + 0.5) / 6], -1).reshape(1, 42, 1, 1, 1, 2)
    loc = loc.expand(2, 42, 8, 1, 1, 2).contiguous().to(DEV)
    w = torch.ones(2, 42, 8, 1, 1, device=DEV)
    out = ops.msda_forward(value, ss, lsi, loc, w)
    assert max_err(out, value.view(2, 42, 256)) < 1e-5
    perm = torch.randperm(42, device=DEV)
    out_p = ops.msda_forward(value, ss, lsi, loc[:, perm].contiguous(), w)
    assert torch.equal(out_p, out[:, perm])


def test_autograd_function_contract():
    """Same apply() signature and 6-tuple of grads as the reference class
    (multi_scale_deformable_attn_function.py:94-95,162-163)."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(5, 4), (3, 2)], 6, 4, 32, 2, seed=1, device=DEV)
    v.requires_grad_(); loc.requires_grad_(); attn.requires_grad_()
    out = ops.MultiScaleDeformableAttnFunction_fp32.apply(v, ss, lsi, loc, attn, 64)
    assert out.shape == (2, 6, 128)
    out.sum().backward()
    assert v.grad.shape == v.shape and loc.grad.shape == loc.shape and attn.grad.shape == attn.shape
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.MultiScaleDeformableAttnFunction_fp32.apply(v.detach().transpose(1, 2), ss, lsi,
                                                        loc.detach(), attn.detach(), 64)
    with pytest.raises(RuntimeError, match="im2col_step"):
        ops.MultiScaleDeformableAttnFunction_fp32.apply(v.detach()[:1].repeat(3, 1, 1, 1), ss, lsi,
                                                        loc.detach()[:1].repeat(3, 1, 1, 1, 1, 1),
                                                        attn.detach()[:1].repeat(3, 1, 1, 1, 1), 2)


@pytest.mark.parametrize("which", ["tsa", "sca"])
def test_base_shapes_properties(which):
    """Full BASELINE sizes: linearity in value / attn and agreement with Oracle-S on a row sample."""
    w = syn.WORKLOADS["base"]
    if which == "tsa":
        bs, levels, nq, pts = 2, [(200, 200)], 40000, 4
    else:
        bs, levels, nq, pts = 6, list(w.levels), 9507, 8
    v, ss, lsi, loc, attn = syn.make_msda_inputs(bs, levels, nq, 8, 32, pts, seed=0)
    vd, ld, ad = v.to(DEV), loc.to(DEV), attn.to(DEV)
    out = ops.msda_forward(vd, ss.to(DEV), lsi.to(DEV), ld, ad)
    out2 = ops.msda_forward(2 * vd, ss.to(DEV), lsi.to(DEV), ld, 0.5 * ad)
    assert max_err(out2, out) < 1e-4
    rows = np.sort(np.random.default_rng(0).choice(nq, 64, replace=False))
    ref = msda_oracle.msda_forward(v, ss, lsi, loc[:, rows].contiguous(), attn[:, rows].contiguous())
    assert max_err(out[:, rows].cpu(), ref) < 1e-4
    # backward: grad_value total mass equals sum over samples of in-range weight * attn * g (g = 1)
    g = torch.ones_like(out)
    gv, gl, ga = ops.msda_backward(vd, ss.to(DEV), lsi.to(DEV), ld, ad, g)
    rgv, rgl, rga = msda_oracle.msda_backward(v, ss, lsi, loc, attn, torch.ones(bs, nq, 256))
    assert rel_err(gv.cpu(), rgv) < 1e-3
    assert rel_err(ga.cpu(), rga) < 1e-3 and rel_err(gl.cpu(), rgl) < 1e-3


@pytest.fixture(params=[0, 1, 2], ids=["bwd_one_kernel", "bwd_split", "bwd_hybrid"])
def backward_mode(request):
    """Both grad_value strategies of the library (bevf_msda_set_backward_mode) must pass the same bars."""
    from bevformer_b200 import _lib
    lib = _lib.load()
    assert lib.bevf_msda_set_backward_mode(request.param) == 0
    yield request.param
    lib.bevf_msda_set_backward_mode(0)


@pytest.mark.parametrize("which", ["sca", "tsa", "tsa_rows"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_base_rig_geometry_against_oracle(which, dtype, backward_mode):
    """The launches the headline benchmark times: base shapes on the REAL geometry (SCA: the 44 511
    in-view (camera, query) pairs of the synthetic rig, 4 levels, 8 points, through the row-list entry
    points; TSA: 2 x 40 000 rows around each query's own cell), forward and backward, fp32 and bf16
    storage, every output element against Oracle-S on the same (storage-rounded) inputs.
    Bars: 1e-3 fp32 / 1e-2 bf16 (BASELINE.json north_star)."""
    from tools.bench_msda import rig_sca_inputs, rig_tsa_inputs, rig_tsa_rows_inputs
    tol = TOL[dtype]
    order = None
    if which == "sca":
        v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
    elif which == "tsa_rows":     # the encoder's TSA launch: interleaved (b, q, frame) rows + 8x8-tile group order
        v, ss, lsi, loc, attn, row_map, order = rig_tsa_rows_inputs(DEV)
    else:
        v, ss, lsi, loc, attn = rig_tsa_inputs(DEV)
        row_map = None
    vd = v.to(dtype)
    nrows = loc.shape[0] if row_map is not None else loc.shape[0] * loc.shape[1]
    gout = fixed_projection((nrows, 256)).to(DEV, dtype)
    if row_map is not None:
        out = ops.msda_rows_forward(vd, ss, lsi, loc, attn, row_map)
        gv, gl, ga = ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout, group_order=order)
    else:
        out = ops.msda_forward(vd, ss, lsi, loc, attn)
        gv, gl, ga = ops.msda_backward(vd, ss, lsi, loc, attn, gout.view(out.shape))
    torch.cuda.synchronize()
    out, gv, gl, ga = out.float().cpu(), gv.cpu(), gl.cpu(), ga.cpu()
    vr, gr = vd.float().cpu(), gout.float().cpu()
    loc_c, attn_c = loc.cpu(), attn.cpu()
    if row_map is not None:       # the oracle is dense: one call per camera map over that camera's rows
        rm = row_map.cpu().long()
        ref = torch.empty_like(out); rgv = torch.zeros_like(gv)
        rgl = torch.empty_like(gl); rga = torch.empty_like(ga)
        for cam in range(vr.shape[0]):
            idx = (rm == cam).nonzero().flatten()
            lc, ac = loc_c[idx][None].contiguous(), attn_c[idx][None].contiguous()
            ref[idx] = msda_oracle.msda_forward(vr[cam:cam + 1], ss.cpu(), lsi.cpu(), lc, ac)[0]
            a, b, c = msda_oracle.msda_backward(vr[cam:cam + 1], ss.cpu(), lsi.cpu(), lc, ac, gr[idx][None].contiguous())
            rgv[cam] = a[0]; rgl[idx] = b[0]; rga[idx] = c[0]
    else:
        ref = msda_oracle.msda_forward(vr, ss.cpu(), lsi.cpu(), loc_c, attn_c)
        rgv, rgl, rga = msda_oracle.msda_backward(vr, ss.cpu(), lsi.cpu(), loc_c, attn_c, gr.view(ref.shape))
    errs = dict(out=rel_err(out.view(ref.shape), ref), grad_value=rel_err(gv, rgv),
                grad_attn=rel_err(ga, rga), grad_loc=rel_err(gl, rgl))
    print(which, dtype, errs)
    assert errs["out"] < tol and errs["grad_value"] < tol and errs["grad_attn"] < tol, errs
    # grad_loc carries the W_l / H_l factors (up to 200) and is discontinuous at cell borders: a sample
    # whose coordinate rounds onto a border may take the other cell's slope -> compare the bulk
    ok, m = _robust(gl, rgl, 4 * tol)
    assert ok, ("grad_loc", m, errs)


def _robust(got, want, tol, max_outlier_frac=1e-4):
    got, want = got.double().flatten(), want.double().flatten()
    scale = max(1.0, want.abs().max().item())
    frac = ((got - want).abs() > tol * scale).double().mean().item()
    l2 = ((got - want).norm() / max(want.norm().item(), 1e-12)).item()
    return frac <= max_outlier_frac and l2 < 5 * tol, (l2, frac)


def _oracle_grad_value(vd, ss, lsi, loc, attn, row_map, gout):
    rm = row_map.cpu().long()
    vr, gr = vd.float().cpu(), gout.float().cpu()
    rgv = torch.zeros(vd.shape, dtype=torch.float32)
    for b in range(vr.shape[0]):
        idx = (rm == b).nonzero().flatten()
        if idx.numel() == 0:
            continue
        a, _, _ = msda_oracle.msda_backward(vr[b:b + 1], ss.cpu(), lsi.cpu(), loc.cpu()[idx][None].contiguous(),
                                            attn.cpu()[idx][None].contiguous(), gr[idx][None].contiguous())
        rgv[b] = a[0]
    return rgv


@pytest.mark.parametrize("which", ["tsa_rows", "sca_mixed", "sca_mixed2", "sca_all", "small", "small_mixed", "tiny_grads"])
def test_fp16_accumulated_grad_value(which):
    """grad_value accumulated in SCALED fp16 (bevf_msda_rows_backward_f16acc / _mixed + bevf_abs_max /
    bevf_gv16_unscale / bevf_gv_merge): one f16x2 vector reduction per lane and corner, the running sum rounded to 11
    bits at every addition, the scale taken from max|grad_out|.  On the launches of the headline benchmark -- TSA: 2 x
    40 000 rows, one 200 x 200 level, every level in fp16; SCA: 44 511 pairs, levels 0-1 in fp16 and levels 2-3 in fp32
    (what ops.gv_mode_for picks), also level 0 only -- the bf16 gradient must hold the bf16 bar against Oracle-S; grad_loc / grad_attn are those of the fp32 path bit for
    bit.  'tiny_grads': gradients of 1e-6 (what the scale is for)."""
    from tools.bench_msda import rig_sca_inputs, rig_tsa_rows_inputs
    order, nfine, gscale = None, 0, 1.0
    if which == "tsa_rows":
        v, ss, lsi, loc, attn, row_map, order = rig_tsa_rows_inputs(DEV)
    elif which.startswith("sca_"):
        v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
        nfine = {"sca_mixed": 1, "sca_mixed2": 2, "sca_all": 0}[which]     # 0: every level in fp16
    else:
        levels = [(12, 20), (6, 10)] if which != "tiny_grads" else [(9, 16)]
        v, ss, lsi, loc, attn = syn.make_msda_inputs(3, levels, 500, 8, 32, 4, seed=5, device=DEV)
        loc, attn = loc.flatten(0, 1).contiguous(), attn.flatten(0, 1).contiguous()
        row_map = torch.arange(3, device=DEV, dtype=torch.int32).repeat_interleave(500).contiguous()
        row_map[17:23] = -1                                   # unused rows
        nfine = 1 if which == "small_mixed" else 0
        gscale = 1e-6 if which == "tiny_grads" else 1.0
    vd = v.to(torch.bfloat16)
    gout = (fixed_projection((loc.shape[0], 256)) * gscale).to(DEV, torch.bfloat16)
    gv32, gl32, ga32 = ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout, group_order=order)
    if nfine:
        hw_host = [tuple(int(x) for x in r) for r in ss.tolist()]
        gv16, gl16, ga16 = ops.msda_rows_backward_mixed(vd, ss, lsi, hw_host, nfine, loc, attn, row_map, gout, order)
    else:
        gv16, gl16, ga16 = ops.msda_rows_backward_f16acc(vd, ss, lsi, loc, attn, row_map, gout, order)
    torch.cuda.synchronize()
    assert gv16.dtype == torch.bfloat16 and gv16.shape == gv32.shape
    used = row_map >= 0
    assert torch.equal(gl32[used], gl16[used]) and torch.equal(ga32[used], ga16[used])
    scale = max(gv32.abs().max().item(), 1e-30) if which == "tiny_grads" else None     # relative to max|ref| there
    def err(a, b):
        return (a.double() - b.double()).abs().max().item() / scale if scale else rel_err(a, b)
    e_acc = err(gv16.float().cpu(), gv32.cpu())
    e_round = err(gv32.to(torch.bfloat16).float().cpu(), gv32.cpu())      # what storing the result in bf16 costs anyway
    lsl = lsi.tolist() + [int(v.shape[1])]
    per_level = [err(gv16[:, lsl[i]:lsl[i + 1]].float().cpu(), gv32[:, lsl[i]:lsl[i + 1]].cpu()) for i in range(len(lsl) - 1)]
    print(which, "fp16-accumulated grad_value vs fp32 accumulation:", e_acc, per_level, "(bf16 rounding of the result alone:", e_round, ")")
    if which == "sca_all":
        # every level in fp16 is what ops.gv_mode_for must NOT choose: the error grows with the contributions per pixel
        # (10 / 41 / 164 / 630 on average at base; measured 5e-3 / 6e-3 / 1e-2 / 1.3e-2) -- only the fine half holds the bar
        assert per_level[0] < TOL[torch.bfloat16] and per_level[1] < TOL[torch.bfloat16], per_level
        assert per_level[3] > per_level[0]
        return
    assert e_acc < TOL[torch.bfloat16]
    if which in ("tsa_rows", "sca_mixed", "sca_mixed2"):
        rgv = _oracle_grad_value(vd, ss, lsi, loc, attn, row_map, gout)
        e = rel_err(gv16.float().cpu(), rgv)
        print(which, "fp16-accumulated grad_value vs Oracle-S:", e)
        assert e < TOL[torch.bfloat16]


def test_gv16_helpers_against_torch():
    """bevf_abs_max, the scale derived from it, bevf_gv16_unscale and bevf_gv_merge against tensor ops."""
    from bevformer_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    for dt, amp in ((torch.bfloat16, 37.5), (torch.float32, 3e-7), (torch.bfloat16, 0.0)):
        x = (torch.randn(4096 * 8, generator=g) * amp).to(DEV, dt)
        bits = ops.abs_max_bits(x)
        got = bits.view(torch.float32).item()
        assert got == x.float().abs().max().item()
    x = (torch.randn(1000 * 8, generator=g) * 5).to(DEV, torch.bfloat16)
    bits = ops.abs_max_bits(x)
    amax = bits.view(torch.float32).item()
    import math
    scale = 2.0 ** (3 - math.floor(math.log2(amax)))
    assert 8.0 <= amax * scale < 16.0
    acc = (torch.randn(2, 50, 8, 32, generator=g) * 9).to(DEV, torch.float16)
    out = torch.empty(acc.shape, device=DEV, dtype=torch.bfloat16)
    _lib.check(lib.bevf_gv16_unscale(acc.data_ptr(), bits.data_ptr(), out.data_ptr(), acc.numel(), 0), lib)
    torch.cuda.synchronize()
    assert torch.equal(out, (acc.float() / scale).to(torch.bfloat16))
    side = torch.randn(2, 30, 8, 32, generator=g).to(DEV)
    merged = torch.empty(2, 80, 8, 32, device=DEV, dtype=torch.bfloat16)
    _lib.check(lib.bevf_gv_merge(acc.data_ptr(), side.data_ptr(), bits.data_ptr(), merged.data_ptr(), 2, 80, 50, 256, 0), lib)
    torch.cuda.synchronize()
    assert torch.equal(merged[:, :50], (acc.float() / scale).to(torch.bfloat16))
    assert torch.equal(merged[:, 50:], side.to(torch.bfloat16))
