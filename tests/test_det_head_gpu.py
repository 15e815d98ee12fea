"""The detection head on the GPU: bevf_det_branches_forward against the float64 restatement (tests/head_oracle.py)
per element with a bar derived from the storage dtype's rounding, BEVFormerHead's kernel and module paths, and a
captured detection frame of BEVStream."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

from bevformer_b200 import _lib, ops, synthetic as syn
from bevformer_b200.plugin import BEVStream
from tests import head_oracle as ho
from tests.test_head_golden_cpu import toy_head
from tests.util import golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PC = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def _branch_pair(seed, ncls=10):
    g = torch.Generator().manual_seed(seed)
    cls = nn.Sequential(nn.Linear(256, 256), nn.LayerNorm(256), nn.ReLU(inplace=True), nn.Linear(256, 256),
                        nn.LayerNorm(256), nn.ReLU(inplace=True), nn.Linear(256, ncls))
    reg = nn.Sequential(nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 10))
    with torch.no_grad():
        for m in list(cls) + list(reg):
            if isinstance(m, nn.Linear):
                m.weight.uniform_(-1 / 16, 1 / 16, generator=g)
                m.bias.uniform_(-0.5, 0.5, generator=g)
            elif isinstance(m, nn.LayerNorm):
                m.weight.copy_(1 + 0.2 * torch.randn(256, generator=g))
                m.bias.copy_(0.2 * torch.randn(256, generator=g))
    return cls, reg


def _refs(L, bs, nq, dtype, seed, clamps=False):
    g = torch.Generator().manual_seed(seed)
    ref0 = torch.rand(bs, nq, 3, generator=g)
    refs = torch.rand(L, bs, nq, 3, generator=g)
    if clamps:                        # the inverse-sigmoid clamps: 0, 1, within 1e-5 of either
        edge = torch.tensor([0.0, 1.0, 5e-6, 1 - 5e-6, 1e-5, 1 - 1e-5, 2e-5, 1 - 2e-5, -0.25, 1.5])
        ref0.view(-1)[: edge.numel() * 8] = edge.repeat(8)
        refs.view(-1)[: edge.numel() * 8] = edge.flip(0).repeat(8)
    return ref0.to(DEV, dtype), refs.to(DEV, dtype)


CASES = [  # (dtype, fp32 params, shared branches, bs, nq, L, reference-point dtype, clamps)
    (torch.bfloat16, False, False, 1, 900, 6, torch.bfloat16, False),
    (torch.float16, False, False, 1, 900, 6, torch.float16, False),
    (torch.bfloat16, True, False, 2, 77, 3, torch.float32, True),
    (torch.float16, True, True, 2, 77, 3, torch.float32, True),
    (torch.bfloat16, False, True, 2, 900, 2, torch.bfloat16, False),
    (torch.float16, True, False, 1, 150, 1, torch.float32, True),
]


@pytest.mark.parametrize("dtype,p32,shared,bs,nq,L,rdt,clamps", CASES)
def test_branches_kernel_against_fp64(dtype, p32, shared, bs, nq, L, rdt, clamps):
    pairs = [_branch_pair(7)] * L if shared else [_branch_pair(7 + lvl) for lvl in range(L)]
    pdt = torch.float32 if p32 else dtype
    pairs = [(c.to(DEV, pdt), r.to(DEV, pdt)) for c, r in pairs]
    tables = [ops.det_branch_params(c, r) for c, r in pairs]
    g = torch.Generator().manual_seed(3)
    states = torch.randn(L, bs, nq, 256, generator=g).to(DEV, dtype).permute(0, 2, 1, 3)   # a strided (L, nq, bs, C)
    ref0, refs = _refs(L, bs, nq, rdt, 5, clamps)
    with torch.no_grad():
        cls, box = ops.det_branches_forward(states, ref0, refs, tables, PC)
    torch.cuda.synchronize()
    assert cls.shape == (L, bs, nq, 10) and box.shape == (L, bs, nq, 10) and cls.dtype == dtype
    want_c, want_b, bar_c, bar_b = ho.branches_fp64(states, ref0, refs, tables, PC, dtype=dtype, with_err=True)
    for got, want, bar, name in ((cls, want_c, bar_c, "cls"), (box, want_b, bar_b, "box")):
        assert torch.isfinite(got).all(), name
        err = (got.double().cpu() - want).abs()
        worst = (err / bar).max().item()
        assert worst <= 1.0, f"{name}: error {err.max().item():.3g}, {worst:.3g} x the bar"


def test_branches_kernel_refuses_what_it_cannot_run():
    c, r = _branch_pair(1)
    tables = [ops.det_branch_params(c.to(DEV), r.to(DEV))]
    states = torch.zeros(1, 64, 1, 256, device=DEV)
    ref = torch.zeros(1, 64, 3, device=DEV)
    with pytest.raises(RuntimeError, match="bf16 or fp16"):
        ops.det_branches_forward(states, ref, ref[None], tables, PC)
    with pytest.raises(RuntimeError, match="256"):
        ops.det_branches_forward(torch.zeros(1, 64, 1, 128, device=DEV, dtype=torch.bfloat16), ref, ref[None],
                                 tables, PC)
    with pytest.raises(NotImplementedError):
        ops.det_branch_params(c[:4], r)


# ---- the head module --------------------------------------------------------------------------------------------
W = syn.WORKLOADS["toy"]


def head_cfg(num_query=100, with_box_refine=True, group_detr=None, max_num=60, score_threshold=None):
    cfg = dict(type="BEVFormerHead", bev_h=W.bev_h, bev_w=W.bev_w, num_query=num_query, num_classes=10,
               in_channels=256, sync_cls_avg_factor=True, with_box_refine=with_box_refine, as_two_stage=False,
               transformer=dict(type="PerceptionTransformer", num_feature_levels=len(W.levels), num_cams=W.num_cams,
                                embed_dims=256, rotate_center=[W.bev_h // 2, W.bev_w // 2],
                                encoder=syn.encoder_cfg(W), decoder=copy.deepcopy(syn.DECODER_CFG)),
               bbox_coder=dict(type="NMSFreeCoder", post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
                               pc_range=PC, max_num=max_num, score_threshold=score_threshold, num_classes=10),
               positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=W.bev_h,
                                        col_num_embed=W.bev_w),
               loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
               loss_bbox=dict(type="L1Loss", loss_weight=0.25), loss_iou=dict(type="GIoULoss", loss_weight=0.0))
    if group_detr:
        cfg.update(type="BEVFormerHead_GroupDETR", group_detr=group_detr)
    return cfg


def make_head(seed=0, **kw):
    from bevformer_b200.plugin.config import build_head
    h = build_head(head_cfg(**kw))
    h.load_state_dict(syn.make_random_state_dict(h, seed, scale=0.1))
    return h.to(DEV).eval()


def _frame_inputs(dtype, bs=1):
    inp = syn.make_perception_inputs(W, bs=bs, with_prev=True, device=DEV)
    return [f.to(dtype) for f in inp.mlvl_feats], inp.img_metas, inp.prev_bev.to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("group_detr", [None, 3])
def test_head_kernel_path_equals_its_module_path(dtype, group_detr):
    """The head's kernel path (no gradient, 16-bit) against its own module path on the same decoder output, and
    the GroupDETR eval slice (num_query // group_detr queries)."""
    head = make_head(num_query=100, group_detr=group_detr).to(dtype)
    feats, metas, prev = _frame_inputs(dtype, bs=2)
    with torch.no_grad():
        out = head(feats, metas, prev_bev=prev)
    nq = 100
    assert out["all_cls_scores"].shape == (3, 2, nq, 10) and out["all_bbox_preds"].shape == (3, 2, nq, 10)
    # the module path on the same transformer output
    with torch.no_grad():
        bev, hs, r0, rs = head.transformer(feats, head.bev_embedding.weight, head._object_query_embeds(dtype),
                                           W.bev_h, W.bev_w, grid_length=(head.real_h / W.bev_h,
                                                                          head.real_w / W.bev_w),
                                           bev_pos=head.positional_encoding(torch.zeros(2, W.bev_h, W.bev_w,
                                                                                        device=DEV)).to(dtype),
                                           reg_branches=head.reg_branches, img_metas=metas, prev_bev=prev)
        mc, mb = head._branches_modules(hs, r0, rs)
    tol = 5e-2 if dtype == torch.bfloat16 else 1e-2
    for got, want in ((out["all_cls_scores"], mc), (out["all_bbox_preds"], mb)):
        err = (got.float() - want.float()).abs().max().item()
        assert err <= tol * max(1.0, want.float().abs().max().item()), err


def test_head_fp32_and_autograd_take_the_modules():
    head = make_head()
    feats, metas, prev = _frame_inputs(torch.float32)
    before = _lib.launch_count()
    out = head(feats, metas, prev_bev=prev)
    loss = out["all_cls_scores"].sum() + out["all_bbox_preds"].sum()
    loss.backward()
    assert head.cls_branches[0][0].weight.grad is not None and head.query_embedding.weight.grad is not None
    assert _lib.launch_count() > before                 # the transformer ran on the library
    hs_grad_free = head.branches                      # fp32 without a gradient: still the modules (no kernel for fp32)
    with torch.no_grad():
        bev, hs, r0, rs = head.transformer(feats, head.bev_embedding.weight, head._object_query_embeds(torch.float32),
                                           W.bev_h, W.bev_w, grid_length=(head.real_h / W.bev_h,
                                                                          head.real_w / W.bev_w),
                                           bev_pos=head.positional_encoding(torch.zeros(1, W.bev_h, W.bev_w,
                                                                                        device=DEV)),
                                           reg_branches=head.reg_branches, img_metas=metas, prev_bev=prev)
        c1, b1 = hs_grad_free(hs, r0, rs)
        want_c, want_b = ho.branches_fp64(hs, r0, rs, [ops.det_branch_params(c, r) for c, r in
                                                       zip(head.cls_branches, head.reg_branches)], PC)
    assert (c1.double().cpu() - want_c).abs().max().item() < 1e-4
    assert (b1.double().cpu() - want_b).abs().max().item() < 1e-3


def test_head_under_autocast_reads_fp32_parameters():
    """Under autocast the kernel reads the fp32 branch parameters (rounding the weights as it stages them); the
    module path under the same autocast on the same decoder output agrees."""
    head = make_head()
    feats, metas, prev = _frame_inputs(torch.float32)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = head(feats, metas, prev_bev=prev)
        _, hs, r0, rs = head.transformer(feats, head.bev_embedding.weight, head._object_query_embeds(torch.float32),
                                         W.bev_h, W.bev_w, grid_length=(head.real_h / W.bev_h, head.real_w / W.bev_w),
                                         bev_pos=head.positional_encoding(torch.zeros(1, W.bev_h, W.bev_w,
                                                                                      device=DEV)),
                                         reg_branches=head.reg_branches, img_metas=metas, prev_bev=prev)
        assert hs.dtype == torch.bfloat16
        mc, mb = head._branches_modules(hs, r0, rs)
    assert out["all_cls_scores"].dtype == torch.bfloat16
    for got, want in ((out["all_cls_scores"], mc), (out["all_bbox_preds"], mb)):
        err = (got.float() - want.float()).abs().max().item()
        assert err <= 5e-2 * max(1.0, want.float().abs().max().item()), err


def test_get_bboxes_against_fp64_decode():
    head = make_head(max_num=60)
    feats, metas, prev = _frame_inputs(torch.bfloat16, bs=2)
    head = head.to(torch.bfloat16)
    with torch.no_grad():
        out = head(feats, metas, prev_bev=prev)
        res = head.get_bboxes(out, metas)
    want = ho.decode_fp64(out["all_cls_scores"][-1].float(), out["all_bbox_preds"][-1].float(), 60,
                          head.bbox_coder.post_center_range, None, z_shift=True)
    for (bb, sc, lb), w in zip(res, want):
        assert bb.shape[1] == 9 and len(bb) == len(w["bboxes"])
        assert torch.allclose(sc.double().cpu(), w["scores"], rtol=1e-6, atol=0)
        assert torch.equal(lb.cpu(), w["labels"])
        assert torch.allclose(bb.double().cpu(), w["bboxes"], rtol=1e-6, atol=1e-6)


# ---- against the reference head's goldens (tests/golden/head_toy.npz) ---------------------------------------------
@pytest.mark.parametrize("refine", [True, False])
def test_head_against_the_reference_golden(refine):
    """The golden case through this head on the GPU: the module path in fp32 (1e-3 of max|ref|), the kernel in bf16
    (1e-2 of max|ref|), get_bboxes of the fp32 outputs against the reference's, and the bf16 decode's selection
    wherever the score gap to the 100th score exceeds the bf16 score bar."""
    g = golden("head_toy")
    tag = "refine" if refine else "shared"
    hs, r0, rs = (t.to(DEV) for t in ho.head_case_inputs())
    ref_c, ref_b = (torch.from_numpy(g[f"{tag}_fp64_{k}"]) for k in ("cls", "box"))
    head = toy_head(refine, torch.float32).to(DEV)
    before = _lib.launch_count()
    with torch.no_grad():
        c32, b32 = head.branches(hs.float(), r0.float(), rs.float())
    assert _lib.launch_count() == before                # fp32: the modules
    head16 = toy_head(refine, torch.float32).to(DEV, torch.bfloat16)
    with torch.no_grad():
        c16, b16 = head16.branches(hs.bfloat16(), r0.float(), rs.float())
    assert _lib.launch_count() == before + 1            # bf16: one fused launch
    for got, want, tol in ((c32, ref_c, 1e-3), (b32, ref_b, 1e-3), (c16, ref_c, 1e-2), (b16, ref_b, 1e-2)):
        err = (got.double().cpu() - want).abs().max().item()
        assert err <= tol * want.abs().max().item(), (tol, err)
    # get_bboxes of the fp32 outputs against the reference head's get_bboxes of its own fp32 outputs
    ret = head.get_bboxes(dict(all_cls_scores=c32, all_bbox_preds=b32), None)
    cut = np.cumsum(g[f"{tag}_fp32_dec_num"])[:-1]
    for (bb, sc, lb), wb, ws, wl in zip(ret, *(np.split(g[f"{tag}_fp32_dec_{k}"], cut)
                                                 for k in ("bboxes", "scores", "labels"))):
        np.testing.assert_array_equal(lb.cpu().numpy(), wl)
        np.testing.assert_allclose(sc.cpu().numpy(), ws, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(bb.cpu().numpy(), wb, rtol=1e-4, atol=1e-3)
    # bf16: the selected flat indices, except candidates whose reference score is within the bar of the 100th
    big = [-1e4] * 3 + [1e4] * 3
    bboxes, _, labels, num = ops.nms_free_decode(c16[-1].contiguous(), b16[-1].contiguous(), 100, big)
    bar = 0.25 * (c16[-1].double().cpu() - ref_c[-1]).abs().max().item()      # sigmoid' <= 1/4
    for i in range(ho.HEAD_BS):
        s_ref = torch.sigmoid(ref_c[-1, i]).reshape(-1)
        kth = s_ref.sort(descending=True).values[99].item()
        vx, vy = (b16[-1, i, :, c].float().cpu() for c in (8, 9))     # the query of a detection: its velocity
        q = ((bboxes[i, :, 7].cpu()[:, None] == vx[None, :]) &
             (bboxes[i, :, 8].cpu()[:, None] == vy[None, :])).float().argmax(1)
        got = set((q * ho.HEAD_NCLS + labels[i].cpu()).tolist())
        sure_in = set(torch.nonzero(s_ref > kth + 2 * bar).reshape(-1).tolist())
        sure_out = set(torch.nonzero(s_ref < kth - 2 * bar).reshape(-1).tolist())
        assert sure_in <= got and not (got & sure_out)


def test_module_path_gradients_against_the_reference_golden():
    g = golden("head_toy")
    hs, r0, rs = (t.to(DEV).float() for t in ho.head_case_inputs())
    hs.requires_grad_(True)
    head = toy_head(True, torch.float32).to(DEV)
    cls, box = head.branches(hs, r0, rs)                # a gradient is needed: the modules
    gen = torch.Generator().manual_seed(44000)
    pc = torch.randn(cls.shape, generator=gen, dtype=torch.float64).to(DEV, torch.float32)
    pb = torch.randn(box.shape, generator=gen, dtype=torch.float64).to(DEV, torch.float32)
    ((cls * pc).sum() + (box * pb).sum()).backward()
    for got, key in ((hs.grad, "grad_hs"), (head.cls_branches[0][0].weight.grad, "grad_cls0_w0"),
                     (head.reg_branches[2][4].bias.grad, "grad_reg2_b4")):
        want = torch.from_numpy(g[key])
        assert (got.double().cpu() - want).abs().max().item() <= 1e-4 * want.abs().max().item(), key


# ---- capture -------------------------------------------------------------------------------------------------------
def _sequence(dtype, frames=4):
    from tests.golden.make_golden import sequence_inputs
    feats, _, _, metas = sequence_inputs(W, frames)
    cb = torch.as_tensor(np.array([m["can_bus"] for m in metas], dtype=np.float64)).to(DEV)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in metas], dtype=np.float32)).to(DEV)
    bare = [{k: v for k, v in m.items() if k not in ("can_bus", "lidar2img")} for m in metas]
    return [f.to(DEV, dtype) for f in feats], cb, l2i, bare


def test_detection_frame_does_not_synchronise():
    head = make_head().to(torch.bfloat16)
    feats, cb, l2i, bare = _sequence(torch.bfloat16)
    with torch.no_grad():
        first = head([f[:, 0] for f in feats], bare[:1], can_bus=cb[0:1], lidar2img=l2i[0:1])
        head.bbox_coder.decode_device(first)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = head([f[:, 1] for f in feats], bare[1:2], prev_bev=first["bev_embed"], can_bus=cb[1:2],
                       lidar2img=l2i[1:2])
            dec = head.bbox_coder.decode_device(out)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert dec["bboxes"].shape == (1, 60, 9) and dec["num"].shape == (1,)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_captured_detection_stream_equals_eager(dtype):
    head = make_head().to(dtype)
    feats, cb, l2i, bare = _sequence(dtype)
    stream = BEVStream(head.transformer)
    eager, launches = [], []
    for i in range(4):                                   # scene-a x 3, then scene-b
        before = _lib.launch_count()
        res = stream.step([f[:, i] for f in feats], [bare[i]], can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1],
                          head=head)
        launches.append(_lib.launch_count() - before)
        assert stream.prev_frame_info["prev_bev"] is res["bev_embed"]
        eager.append({k: v.clone() for k, v in res.items()})
    # the head adds exactly two library launches to the transformer's frame (16-bit: branches + decode; fp32: the
    # branches are modules, the decode is one launch)
    plain = BEVStream(head.transformer)
    for i in range(2):
        before = _lib.launch_count()
        with torch.no_grad():
            plain.step([f[:, i] for f in feats], [bare[i]], head.bev_embedding.weight.to(dtype), W.bev_h, W.bev_w,
                       head.positional_encoding(torch.zeros(1, W.bev_h, W.bev_w, device=DEV)).to(dtype),
                       (head.real_h / W.bev_h, head.real_w / W.bev_w), can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1],
                       object_query_embed=head.query_embedding.weight.to(dtype), reg_branches=head.reg_branches)
        extra = launches[i] - (_lib.launch_count() - before)
        assert extra == (2 if dtype != torch.float32 else 1), (i, extra)
    stream = BEVStream(head.transformer)
    static = stream.capture([f[:, 0] for f in feats], [bare[0]], can_bus=cb[0:1], lidar2img=l2i[0:1], head=head)
    assert static["can_bus"].shape == (1, 18)
    before = _lib.launch_count()
    for i in range(4):
        res = stream.step([f[:, i] for f in feats], [bare[i]], can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1])
        got = {k: v.clone() for k, v in res.items()}
        torch.cuda.synchronize()
        for k in got:
            assert torch.equal(got[k], eager[i][k]), (i, k)
    assert _lib.launch_count() == before
