"""GPU tests of the mixed + dense sampler backward (bevf_msda_rows_backward_mixed_dense): grad_value of the fine
levels in scaled fp16, of a coarse suffix of the pyramid on the dense tensor-core kernel (csrc/msda_dense.cu), of the
levels between them in fp32 reductions, all but the fp16 part in the side buffer of the mixed layout.
Bar: 1e-2 for bf16 storage, max|err| / max(1, max|ref|) per level, as in test_msda_dense_gpu.py."""
import numpy as np
import pytest
import torch

from bevformer_b200 import _lib, ops, synthetic as syn
from oracle import msda_oracle
from tests.test_msda_dense_gpu import _ragged_case
from tests.util import fixed_projection, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def library_default():
    """Every test starts from and restores the library default (bevf_msda_set_dense_backward(-1))."""
    lib = _lib.load()
    assert lib.bevf_msda_set_dense_backward(-1) == 0
    yield
    lib.bevf_msda_set_dense_backward(-1)


def _ranges(row_map, nb):
    per = torch.bincount(row_map[row_map >= 0].long(), minlength=nb)
    ends = per.cumsum(0)
    return torch.stack([ends - per, ends], 1).to(torch.int32).contiguous()


@pytest.fixture(scope="module")
def base_rig():
    """The SCA launch of the headline benchmark and its Oracle-S grad_value (computed once)."""
    from tools.bench_msda import rig_sca_inputs
    v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
    vd = v.to(torch.bfloat16)
    gout = fixed_projection((loc.shape[0], 256)).to(DEV, torch.bfloat16)
    vr, gr, loc_c, attn_c, rm = vd.float().cpu(), gout.float().cpu(), loc.cpu(), attn.cpu(), row_map.cpu().long()
    rgv = torch.zeros(vr.shape)
    for cam in range(vr.shape[0]):
        idx = (rm == cam).nonzero().flatten()
        a, _, _ = msda_oracle.msda_backward(vr[cam:cam + 1], ss.cpu(), lsi.cpu(), loc_c[idx][None].contiguous(),
                                            attn_c[idx][None].contiguous(), gr[idx][None].contiguous())
        rgv[cam] = a[0]
    return vd, ss, lsi, loc, attn, row_map, gout, rgv


@pytest.mark.parametrize("mode", [1, 2], ids=["same_stream", "second_stream"])
@pytest.mark.parametrize("nfine,kd", [(1, 1), (2, 2), (2, 3)], ids=["k1", "k2", "fp16_01_dense_3"])
def test_base_rig_against_oracle(base_rig, nfine, kd, mode):
    vd, ss, lsi, loc, attn, row_map, gout, rgv = base_rig
    levels = [tuple(x) for x in syn.WORKLOADS["base"].levels]
    lib = _lib.load()
    assert lib.bevf_msda_set_dense_backward(mode) == 0
    rng = _ranges(row_map, vd.shape[0])
    gv, gl, ga = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, nfine, loc, attn, row_map, gout, map_range=rng,
                                              first_dense_level=kd)
    assert lib.bevf_msda_set_dense_backward(0) == 0
    gvp, glp, gap = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, nfine, loc, attn, row_map, gout)
    torch.cuda.synchronize()
    used = row_map >= 0
    assert torch.equal(gl[used], glp[used]) and torch.equal(ga[used], gap[used])   # same kernel, same arithmetic
    lsl = lsi.tolist() + [int(vd.shape[1])]
    gvc = gv.float().cpu()
    per_level = [rel_err(gvc[:, lsl[i]:lsl[i + 1]], rgv[:, lsl[i]:lsl[i + 1]]) for i in range(4)]
    print("mixed+dense", nfine, kd, mode, "per level vs Oracle-S:", per_level)
    assert max(per_level) < 1e-2, per_level


def test_setter_zero_runs_the_mixed_kernels(base_rig):
    """Mode 0: bevf_msda_rows_backward_mixed_dense is bevf_msda_rows_backward_mixed (no dense launch); the fp32 and fp16
    reductions are not reproducible run to run, so the bar is their reordering, not bit identity."""
    vd, ss, lsi, loc, attn, row_map, gout, _ = base_rig
    levels = [tuple(x) for x in syn.WORKLOADS["base"].levels]
    lib = _lib.load()
    assert lib.bevf_msda_set_dense_backward(0) == 0 and lib.bevf_msda_get_dense_backward() == 0
    rng = _ranges(row_map, vd.shape[0])
    n0 = _lib.launch_count()
    gv, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 2, loc, attn, row_map, gout, map_range=rng)
    n1 = _lib.launch_count()
    gvp, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 2, loc, attn, row_map, gout)
    torch.cuda.synchronize()
    assert n1 - n0 == _lib.launch_count() - n1                          # the same launches as the mixed entry
    assert rel_err(gv.float().cpu(), gvp.float().cpu()) < 1e-2     # reordered sums: a bf16 ulp (2^-8)


def test_library_default_and_rule():
    lib = _lib.load()
    assert lib.bevf_msda_get_dense_backward() == 2                     # second stream unless the caller says otherwise
    assert lib.bevf_msda_set_dense_backward(3) != 0 and lib.bevf_msda_set_dense_backward(-2) != 0
    base = [(116, 200), (58, 100), (29, 50), (15, 25)]
    assert ops.dense_levels_for(44511 / 6, 8, base) == 3               # 10 / 41 / 164 / 630 per pixel
    assert ops.dense_levels_for(44511 / 6, 8, base[:3]) is None
    assert ops.dense_levels_for(2500.0, 8, [(15, 25)]) is None        # 213 per pixel
    assert ops.dense_levels_for(4000.0, 8, [(15, 25)]) == 0           # 341


def test_suffix_the_dense_plan_cannot_take_falls_back_to_mixed():
    """A coarse level of 10 000 pixels (more than the dense kernel's 8 192) behind the fine one: no dense bin, the
    side level stays on the reduction path, the result is the mixed path's."""
    levels = [(100, 120), (100, 100)]
    v, ss, lsi, loc, attn, row_map, rng = _ragged_case(levels, [300, 0, 513], 8, 8, seed=5)
    vd = v.to(DEV, torch.bfloat16)
    ss, lsi, loc, attn, row_map, rng = (t.to(DEV) for t in (ss, lsi, loc, attn, row_map, rng))
    gout = fixed_projection((loc.shape[0], 256)).to(DEV, torch.bfloat16)
    lib = _lib.load()
    assert lib.bevf_msda_set_dense_backward(1) == 0
    gv, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 1, loc, attn, row_map, gout, map_range=rng)
    assert lib.bevf_msda_set_dense_backward(0) == 0
    gvp, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 1, loc, attn, row_map, gout)
    torch.cuda.synchronize()
    assert rel_err(gv.float().cpu(), gvp.float().cpu()) < 1e-2     # reordered sums: a bf16 ulp (2^-8)


def test_stale_host_shapes_degrade_to_mixed():
    """Host shapes with the right pixel counts but transposed: the dense kernel sees the mismatch and writes nothing,
    the reduction kernel keeps every side level -- the result is the mixed path's."""
    levels = [(20, 30), (10, 15), (5, 8), (3, 4)]
    v, ss, lsi, loc, attn, row_map, rng = _ragged_case(levels, [700, 40, 1300], 8, 8, seed=3)
    vd = v.to(DEV, torch.bfloat16)
    ss, lsi, loc, attn, row_map, rng = (t.to(DEV) for t in (ss, lsi, loc, attn, row_map, rng))
    gout = fixed_projection((loc.shape[0], 256)).to(DEV, torch.bfloat16)
    wrong = [(30, 20), (15, 10), (8, 5), (4, 3)]
    lib = _lib.load()
    assert lib.bevf_msda_set_dense_backward(1) == 0
    gv, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, wrong, 1, loc, attn, row_map, gout, map_range=rng)
    gvp, _, _ = ops.msda_rows_backward_mixed(vd, ss, lsi, levels, 1, loc, attn, row_map, gout)
    torch.cuda.synchronize()
    assert rel_err(gv.float().cpu(), gvp.float().cpu()) < 1e-2     # reordered sums: a bf16 ulp (2^-8)


def test_graph_capture_of_the_encoder_step_with_the_default():
    """The base encoder (bf16, eval: no dropout), forward + backward captured in one CUDA graph with the library
    default in effect (dense kernel on the second stream), replayed, against the eager step."""
    w = syn.WORKLOADS["base"]
    from bevformer_b200.plugin import build_transformer_layer_sequence
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w))
    enc = enc.to(DEV, torch.bfloat16).eval()
    inp = syn.make_encoder_inputs(w, bs=1, seed=0)
    dev_in = {k: getattr(inp, k).to(DEV, torch.bfloat16) for k in ("bev_query", "feat", "bev_pos", "prev_bev")}
    dev_in["bev_query"].requires_grad_(True)
    shift = inp.shift.to(DEV)
    ss, lsi = inp.spatial_shapes.to(DEV), inp.level_start_index.to(DEV)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in inp.img_metas], dtype=np.float32)).to(DEV)
    proj = fixed_projection((1, w.num_query, 256)).to(DEV, torch.bfloat16)

    def body():
        dev_in["bev_query"].grad = None
        out = enc(dev_in["bev_query"], dev_in["feat"], dev_in["feat"], bev_h=w.bev_h, bev_w=w.bev_w,
                  bev_pos=dev_in["bev_pos"], spatial_shapes=ss, level_start_index=lsi, prev_bev=dev_in["prev_bev"],
                  shift=shift, img_metas=inp.img_metas, lidar2img=l2i)
        (out.float() * proj.float()).sum().backward()
        return out

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = body().detach().clone()
        eager_grad = dev_in["bev_query"].grad.detach().clone()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert _lib.load().bevf_msda_get_dense_backward() == 2
    g = torch.cuda.CUDAGraph()
    dev_in["bev_query"].grad = None
    with torch.cuda.graph(g):
        out = body()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    enc.check_plan()
    assert rel_err(out.detach().float().cpu(), eager.float().cpu()) < 1e-3   # only the backward has the dense kernel
    err = rel_err(dev_in["bev_query"].grad.float().cpu(), eager_grad.float().cpu())
    print("graph vs eager grad(bev_query):", err)
    assert err < 1e-2
