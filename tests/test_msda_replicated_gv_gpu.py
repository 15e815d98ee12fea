"""GPU tests of the replicated scaled-fp16 grad_value levels of the mixed sampler backward
(bevf_msda_rows_backward_replicated / bevf_sca_rows_backward_fused_replicated + bevf_gv_merge_replicated): the levels
between the fp16 prefix and the fp32 / dense suffix accumulate in k scaled-fp16 copies, pair row r into copy r % k,
and the merge sums the copies in fp32.  Bar: 1e-2 of max|ref| for the bf16 gradient, as for every fp16 level."""
import pytest
import torch

from bevformer_b200 import _lib, ops, synthetic as syn
from tests.test_msda_gpu import _oracle_grad_value
from tests.util import fixed_projection, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
BAR = 1e-2


@pytest.fixture(scope="module")
def base_rig():
    from tools.bench_msda import rig_sca_inputs
    v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
    vd = v.to(torch.bfloat16)
    gout = fixed_projection((loc.shape[0], 256)).to(DEV, torch.bfloat16)
    gv32, gl32, ga32 = ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout)
    rgv = _oracle_grad_value(vd, ss, lsi, loc, attn, row_map, gout)
    return vd, ss, lsi, loc, attn, row_map, gout, gv32, gl32, ga32, rgv


def _per_level(gv, ref, lsi, S):
    lsl = lsi.tolist() + [S]
    g, r = gv.float().cpu(), ref.float().cpu()
    return [rel_err(g[:, lsl[i]:lsl[i + 1]], r[:, lsl[i]:lsl[i + 1]]) for i in range(len(lsl) - 1)]


def _ranges(row_map, nb):
    per = torch.bincount(row_map[row_map >= 0].long(), minlength=nb)
    ends = per.cumsum(0)
    return torch.stack([ends - per, ends], 1).to(torch.int32).contiguous()


@pytest.mark.parametrize("dense", [False, True], ids=["fp32_level3", "dense_level3"])
def test_base_rig(base_rig, dense):
    vd, ss, lsi, loc, attn, row_map, gout, gv32, gl32, ga32, rgv = base_rig
    levels = [tuple(x) for x in syn.WORKLOADS["base"].levels]
    reps = ops.gv_replicas_for(row_map.numel() / vd.shape[0], loc.shape[3], levels)
    assert reps == {2: 3}
    kw = dict(map_range=_ranges(row_map, vd.shape[0]), first_dense_level=3) if dense else {}
    gv, gl, ga = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 2, loc, attn, row_map, gout, replicas=reps, **kw)
    gvm, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 2, loc, attn, row_map, gout, **kw)   # level 2 fp32
    gv1, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 3 if not dense else 2, loc, attn, row_map, gout,
                                             **({"replicas": {2: 1}} if dense else {}), **kw)   # one fp16 buffer
    torch.cuda.synchronize()
    used = row_map >= 0
    assert torch.equal(gl[used], gl32[used]) and torch.equal(ga[used], ga32[used])
    S = int(vd.shape[1])
    e_rep, e_mix, e_one = (_per_level(g, gv32, lsi, S) for g in (gv, gvm, gv1))
    o_rep, o_mix = _per_level(gv, rgv, lsi, S), _per_level(gvm, rgv, lsi, S)
    print("replicated vs fp32:", e_rep, "mixed:", e_mix, "one fp16 buffer:", e_one)
    print("replicated vs Oracle-S:", o_rep, "mixed vs Oracle-S:", o_mix)
    assert max(o_rep) < BAR and max(e_rep) < BAR, (o_rep, e_rep)
    # levels 0, 1 and 3 run the code they ran before (order-dependent atomics: the same error level, not the same bits)
    for l in (0, 1, 3):
        assert e_rep[l] < max(1.5 * e_mix[l], 1e-3), (l, e_rep, e_mix)
    assert e_rep[2] < e_one[2], (e_rep, e_one)
    if not dense:
        # k = 1 is the single fp16 buffer: the same error as level 2 in the fp16 prefix
        gk1, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 2, loc, attn, row_map, gout, replicas={2: 1})
        e_k1 = _per_level(gk1, gv32, lsi, S)[2]
        print("k = 1:", e_k1, "level 2 in the fp16 prefix:", e_one[2])
        assert abs(e_k1 - e_one[2]) < 0.3 * e_one[2]


def test_base_rig_copy_load(base_rig):
    """Overflow margin: the most contributions any (map, pixel, head, copy) of level 2 receives at base.  Each adds at
    most 16 (|grad_out| * scale < 16, bilinear weight x attention <= 1) to a running sum that overflows at 65504."""
    vd, ss, lsi, loc, attn, row_map, *_ = base_rig
    R, M, L, P, _ = loc.shape
    h, w = (int(x) for x in ss[2].tolist())
    k = 3
    xy = loc[:, :, 2].reshape(R, M, P, 2)
    x, y = xy[..., 0] * w - 0.5, xy[..., 1] * h - 0.5
    x0, y0 = torch.floor(x).long(), torch.floor(y).long()
    rows = torch.arange(R, device=DEV)
    copy = (rows % k)[:, None, None].expand(R, M, P)
    mp = row_map.long()[:, None, None].expand(R, M, P)
    head = torch.arange(M, device=DEV)[None, :, None].expand(R, M, P)
    counts = torch.zeros(vd.shape[0] * h * w * M * k, device=DEV, dtype=torch.int64)
    live = (row_map >= 0)[:, None, None].expand(R, M, P)
    for dy in (0, 1):
        for dx in (0, 1):
            cx, cy = x0 + dx, y0 + dy
            ok = live & (cx >= 0) & (cx < w) & (cy >= 0) & (cy < h)
            idx = (((mp * h + cy) * w + cx) * M + head) * k + copy
            counts.index_add_(0, idx[ok], torch.ones_like(idx[ok]))
    worst = int(counts.max().item())
    mean = counts.sum().item() / max(1, int((counts > 0).sum().item()))
    print(f"level 2 at base: at most {worst} contributions per (pixel, head, copy), {mean:.1f} on average where any")
    assert worst * 16 < 65504 / 4


@pytest.mark.parametrize("case", ["odd_pixels", "no_side", "tiny_grads"])
def test_small_cases(case):
    """A replicated level whose pixel count is no multiple of anything, rows with row_map = -1, replicated levels up
    to the last one (no fp32 side buffer) and gradients of 1e-6 (what the scale is for)."""
    levels = [(12, 20), (5, 7), (3, 3)]
    v, ss, lsi, loc, attn = syn.make_msda_inputs(3, levels, 500, 8, 32, 4, seed=7, device=DEV)
    loc, attn = loc.flatten(0, 1).contiguous(), attn.flatten(0, 1).contiguous()
    row_map = torch.arange(3, device=DEV, dtype=torch.int32).repeat_interleave(500).contiguous()
    row_map[17:23] = -1
    gscale = 1e-6 if case == "tiny_grads" else 1.0
    vd = v.to(torch.bfloat16)
    gout = (fixed_projection((loc.shape[0], 256)) * gscale).to(DEV, torch.bfloat16)
    reps = {1: 3, 2: 3} if case == "no_side" else {1: 3}
    gv32, gl32, ga32 = ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout)
    gv, gl, ga = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 1, loc, attn, row_map, gout, replicas=reps)
    torch.cuda.synchronize()
    used = row_map >= 0
    assert torch.equal(gl[used], gl32[used]) and torch.equal(ga[used], ga32[used])
    scale = gv32.abs().max().item()
    e = (gv.double() - gv32.double()).abs().max().item() / scale
    print(case, "replicated vs fp32:", e)
    assert e < BAR


def test_merge_against_torch():
    """bevf_gv_merge_replicated: fine pixels unscaled, replicated pixels the sum of their copies, side pixels cast."""
    lib = _lib.load()
    B, S, s_fine, s_rep, k, row = 2, 90, 40, 30, 3, 256
    g = torch.Generator().manual_seed(3)
    f16 = (torch.randn(B, s_fine + k * s_rep, row, generator=g) * 4).to(DEV, torch.float16)
    side = torch.randn(B, S - s_fine - s_rep, row, generator=g).to(DEV)
    bits = ops.abs_max_bits(torch.full((8,), 3.0, device=DEV))
    scale = 4.0                                          # max 3 -> the power of two that puts it in [8, 16)
    out = torch.empty(B, S, row, device=DEV, dtype=torch.bfloat16)
    _lib.check(lib.bevf_gv_merge_replicated(f16.data_ptr(), side.data_ptr(), bits.data_ptr(), out.data_ptr(), B, S,
                                            s_fine, s_rep, k, row, 0), lib)
    f = f16.float()
    rep = sum(f[:, s_fine + c * s_rep:s_fine + (c + 1) * s_rep] for c in range(k))
    want = torch.cat([f[:, :s_fine] / scale, rep / scale, side], 1).to(torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
