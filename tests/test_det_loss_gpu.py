"""BEVFormerHead's training loss on the GPU: the cost kernel per element against the float64 cost, the assignment
against the reference's, the loss values and gradients against the reference's loss (tests/golden/ref_det_loss_*.npz)
in fp32 / bf16 / fp16, bitwise reproducibility, one host synchronisation per call, and a toy head trained end to end
against the same head with the float64 restatement's loss."""
import copy
import types
import warnings

import numpy as np
import pytest
import torch

from bevformer_b200 import ops, synthetic as syn
from bevformer_b200.plugin import head as head_mod
from bevformer_b200.plugin.config import build_head
from tests import det_loss_oracle as dlo
from tests import head_oracle as ho
from tests.test_det_loss_cpu import case_data
from tests.test_head_golden_cpu import W
from tests.util import golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
U = 2.0 ** -24                                   # unit roundoff of fp32


def test_scipy_imports():
    from scipy.optimize import linear_sum_assignment
    r, c = linear_sum_assignment(np.array([[1.0, 0.0], [0.0, 1.0]], np.float32))
    assert c.tolist() == [1, 0]


def _loss_head(st, groups=1, sync=True):
    """The state ``BEVFormerHead._loss`` reads, for the settings of a golden case."""
    reg_cost = {"l1": "BBox3DL1Cost", "smooth_l1": "SmoothL1Cost"}[st["cost_reg_kind"]]
    loss_bbox = dict(type="L1Loss" if st["reg_kind"] == "l1" else "SmoothL1Loss", loss_weight=st["bbox_loss_weight"])
    return types.SimpleNamespace(
        train_cfg=dict(assigner=dict(type="HungarianAssigner3D",
                                     cls_cost=dict(type="FocalLossCost", weight=st["cls_cost_weight"]),
                                     reg_cost=dict(type=reg_cost, weight=st["reg_cost_weight"]),
                                     iou_cost=dict(type="IoUCost", weight=0.0), pc_range=dlo.PC_RANGE)),
        loss_cls=head_mod._loss_cfg(dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25,
                                         loss_weight=st["cls_loss_weight"])),
        loss_bbox=head_mod._loss_cfg(loss_bbox), sync_cls_avg_factor=sync,
        code_weights=torch.tensor(dlo.CODE_WEIGHTS, device=DEV), group_detr=groups)


class Boxes:
    """The two attributes the loss reads of mmdet3d's LiDARInstance3DBoxes, for gravity-centred (n, 9) boxes."""

    def __init__(self, g):
        g = g.float().to(DEV)
        self.gravity_center = g[:, :3]
        self.tensor = torch.cat((g[:, :2], g[:, 2:3] - g[:, 5:6] * 0.5, g[:, 3:]), 1)


def _run(name, dtype, requires_grad=True):
    cls, box, gts, labels, st, groups = case_data(name)
    c = cls.to(DEV, dtype).requires_grad_(requires_grad)
    b = box.to(DEV, dtype).requires_grad_(requires_grad)
    head = _loss_head(st, groups)
    preds = dict(all_cls_scores=c, all_bbox_preds=b, enc_cls_scores=None, enc_bbox_preds=None)
    losses = head_mod.BEVFormerHead._loss(head, [Boxes(g) for g in gts], [lab.to(DEV) for lab in labels], preds,
                                          None, groups)
    return losses, c, b


@pytest.mark.parametrize("name", sorted(dlo.CASES))
def test_cost_kernel_against_fp64(name):
    """Per element, within |c| * 4u + max|c| * 2e-7: the kernel rounds its double result to fp32 once (u); the fp32
    differences 1 - p (exact for p >= 1/2, else u relative, times gamma = 2 in (1 - p)^2) and p + eps (u relative,
    inside log: u absolute) add at most 3u of the class term; log / pow / the 8-term sum in double add nothing
    visible.  The float64 cost takes p = torch.sigmoid in fp32, the rounding the kernel keeps on purpose."""
    cls, box, gts, labels, st, groups = case_data(name)
    L, bs, nq, ncls = cls.shape
    G = max(g.shape[0] for g in gts)
    gt = torch.zeros(bs, G, 9)
    lab = torch.zeros(bs, G, dtype=torch.int64)
    for i, (g, l_) in enumerate(zip(gts, labels)):
        gt[i, :len(g)], lab[i, :len(g)] = g.float(), l_
    n = torch.tensor([len(g) for g in gts], dtype=torch.int32)
    cost = ops.det_match_cost(cls.to(DEV, torch.float32), box.to(DEV, torch.float32), gt.to(DEV), lab.to(DEV),
                              n.to(DEV), st["cost_reg_kind"], st["cls_cost_weight"], st["reg_cost_weight"]).cpu()
    p32 = torch.sigmoid(cls.to(DEV, torch.float32)).double().cpu()
    for l in range(L):
        for b in range(bs):
            k = len(gts[b])
            got = cost[l * bs + b]
            assert (got[:, k:] == 0).all()
            if not k:
                continue
            ref = dlo.match_cost(cls[l, b], box[l, b], gts[b].float().double(), labels[b], st, sigmoid=p32[l, b])
            err = (got[:, :k].double() - ref).abs()
            bar = ref.abs() * 4 * U + ref.abs().max() * 2e-7
            assert (err <= bar).all(), (l, b, (err / bar).max().item())


@pytest.mark.parametrize("name", sorted(dlo.CASES))
def test_assignment_equals_the_reference(name):
    cls, box, gts, labels, st, groups = case_data(name)
    L, bs, nq, _ = cls.shape
    nqg = nq // groups
    G = max(g.shape[0] for g in gts)
    gt = torch.zeros(bs, G, 9)
    lab = torch.zeros(bs, G, dtype=torch.int64)
    for i, (g, l_) in enumerate(zip(gts, labels)):
        gt[i, :len(g)], lab[i, :len(g)] = g.float(), l_
    n = [len(g) for g in gts]
    cost = ops.det_match_cost(cls.to(DEV, torch.float32), box.to(DEV, torch.float32), gt.to(DEV), lab.to(DEV),
                              torch.tensor(n, dtype=torch.int32, device=DEV), st["cost_reg_kind"],
                              st["cls_cost_weight"], st["reg_cost_weight"]).cpu().numpy()
    a = np.full((L * bs, nq), -1, np.int32)
    for p in range(L * bs):
        for g in range(groups):
            if n[p % bs]:
                r, c = dlo.assign(cost[p, g * nqg:(g + 1) * nqg, :n[p % bs]])
                a[p, g * nqg + r] = c
    assert (a == golden(f"ref_det_loss_{name}")["assign"]).all()


def test_assignment_is_optimal_without_a_margin():
    """Random logits in [-4, 4] and boxes with no planted match: the float64 total of the assignment made on the
    kernel's fp32 cost is within n_gt * 1e-5 of the float64 optimum."""
    g = torch.Generator().manual_seed(7)
    nq, n, ncls = 300, 30, 10
    cls = torch.rand(1, 1, nq, ncls, generator=g, dtype=torch.float64) * 8 - 4
    box = torch.rand(1, 1, nq, 10, generator=g, dtype=torch.float64) * 4 - 2
    gt = torch.rand(n, 9, generator=g, dtype=torch.float64) * 3 + 0.5
    gt = gt.float().double()
    lab = torch.randint(0, ncls, (n,), generator=g)
    cls, box = cls.float().double(), box.float().double()
    for st in (dlo.BASE, dlo.V2):
        cost = ops.det_match_cost(cls.to(DEV, torch.float32), box.to(DEV, torch.float32), gt[None].float().to(DEV),
                                  lab[None].to(DEV), torch.tensor([n], dtype=torch.int32, device=DEV),
                                  st["cost_reg_kind"], st["cls_cost_weight"], st["reg_cost_weight"]).cpu().numpy()
        r, c = dlo.assign(cost[0])
        c64 = dlo.match_cost(cls[0, 0], box[0, 0], gt, lab, st).numpy()
        r64, c64i = dlo.assign(c64)
        assert c64[r, c].sum() - c64[r64, c64i].sum() <= n * 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", sorted(dlo.CASES))
def test_loss_values_and_gradients(name, dtype):
    """Loss values within 2e-5 relative of the reference's fp32 and fp64 losses (the predictions lie on the bf16
    grid, so every dtype sees the same numbers).  Gradients per element within max|g| * 2^-20 + |g| * 2^-20: the
    kernel's p is fp32 (an error of u in p moves a focal gradient by at most ~2u of its scale), the rest is double
    rounded once to fp32; 16-bit gradients are those fp32 values rounded to the input dtype."""
    g = golden(f"ref_det_loss_{name}")
    losses, c, b = _run(name, dtype)
    for k, v in losses.items():
        assert v.dtype == torch.float32 and v.dim() == 0
        for tag in ("fp32", "fp64"):
            ref = float(g[f"{tag}_{k}"])
            assert abs(v.item() - ref) <= 2e-5 * abs(ref), (k, tag, v.item(), ref)
    sum(losses.values()).backward()
    assert c.grad.dtype == dtype and b.grad.dtype == dtype
    rows = torch.as_tensor(g["grad_rows"], device=DEV)
    if dtype == torch.float32:
        for t, key in ((c, "cls"), (b, "box")):
            got = t.grad.reshape(-1, t.shape[-1])[rows].double().cpu().numpy()
            ref = g[f"fp64_grad_{key}"]
            bar = np.abs(ref).max() * 2.0 ** -20 + np.abs(ref) * 2.0 ** -20
            assert (np.abs(got - ref) <= bar).all(), (key, (np.abs(got - ref) / bar).max())
    else:
        l32, c32, b32 = _run(name, torch.float32)
        sum(l32.values()).backward()
        assert torch.equal(c.grad, c32.grad.to(dtype)) and torch.equal(b.grad, b32.grad.to(dtype))


@pytest.mark.parametrize("name", ["base", "group"])
def test_bitwise_reproducible(name):
    outs = []
    for _ in range(2):
        losses, c, b = _run(name, torch.float32)
        sum(losses.values()).backward()
        outs.append([v.detach().clone() for v in losses.values()] + [c.grad.clone(), b.grad.clone()])
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize("name", ["base", "group"])
def test_one_synchronisation_per_call(name):
    cls, box, gts, labels, st, groups = case_data(name)
    head = _loss_head(st, groups)
    preds = dict(all_cls_scores=cls.to(DEV, torch.float32), all_bbox_preds=box.to(DEV, torch.float32),
                 enc_cls_scores=None, enc_bbox_preds=None)
    gts_d, labels_d = [Boxes(g) for g in gts], [lab.to(DEV) for lab in labels]
    head_mod.BEVFormerHead._loss(head, gts_d, labels_d, preds, None, groups)          # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            head_mod.BEVFormerHead._loss(head, gts_d, labels_d, preds, None, groups)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in rec if "synchroniz" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]


def _toy_train_head_cfg():
    """A toy BEVFormerHead with bevformer_tiny.py's loss settings and train_cfg (its transformer unused)."""
    return dict(type="BEVFormerHead", bev_h=W.bev_h, bev_w=W.bev_w, num_query=ho.HEAD_NQ, num_classes=ho.HEAD_NCLS,
                in_channels=256, with_box_refine=True, sync_cls_avg_factor=True,
                transformer=dict(type="PerceptionTransformer", num_feature_levels=len(W.levels), num_cams=W.num_cams,
                                 embed_dims=256, encoder=syn.encoder_cfg(W), decoder=copy.deepcopy(syn.DECODER_CFG)),
                bbox_coder=dict(type="NMSFreeCoder", post_center_range=ho.POST_CENTER_RANGE, pc_range=ho.PC_RANGE,
                                max_num=100, num_classes=ho.HEAD_NCLS),
                positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=W.bev_h,
                                         col_num_embed=W.bev_w),
                loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
                loss_bbox=dict(type="L1Loss", loss_weight=0.25), loss_iou=dict(type="GIoULoss", loss_weight=0.0),
                train_cfg=dict(assigner=dict(type="HungarianAssigner3D",
                                             cls_cost=dict(type="FocalLossCost", weight=2.0),
                                             reg_cost=dict(type="BBox3DL1Cost", weight=0.25),
                                             iou_cost=dict(type="IoUCost", weight=0.0), pc_range=ho.PC_RANGE)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_toy_head_trains_end_to_end(dtype):
    """forward (branches) -> loss -> sum.backward on the toy head in train mode, against the same head whose loss is
    the float64 restatement evaluated in torch on the GPU: every parameter gradient with cosine >= 0.9999 (fp32) or
    energy within 1 % (bf16 autocast)."""
    cfg = _toy_train_head_cfg()
    head = build_head(copy.deepcopy(cfg))
    head.load_state_dict(ho.branch_state(True), strict=False)
    head = head.to(DEV).train()
    twin = copy.deepcopy(head)
    hs, r0, rs = (t.float().to(DEV) for t in ho.head_case_inputs())
    g = torch.Generator().manual_seed(3)
    gts = [torch.cat((torch.rand(n, 2, generator=g) * 80 - 40, torch.rand(n, 1, generator=g) * 2 - 2,
                      torch.rand(n, 3, generator=g) * 3 + 0.5, torch.rand(n, 1, generator=g) * 6 - 3,
                      torch.randn(n, 2, generator=g)), 1).to(DEV) for n in (8, 5)]
    labels = [torch.randint(0, ho.HEAD_NCLS, (len(x),), generator=g).to(DEV) for x in gts]
    grads = []
    for h, lib in ((head, True), (twin, False)):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
            cls, box = h.branches(hs, r0, rs)
        if lib:
            losses = h.loss(gts, labels, dict(all_cls_scores=cls, all_bbox_preds=box, enc_cls_scores=None,
                                              enc_bbox_preds=None))
        else:
            gc = [torch.cat((x[:, :2], x[:, 2:3] + x[:, 5:6] * 0.5, x[:, 3:]), 1) for x in gts]
            losses, _ = dlo.loss(cls.float(), box.float(), gc, labels, dlo.BASE, 1,
                                 h.code_weights.tolist())
        sum(losses.values()).backward()
        grads.append({k: p.grad.double().clone() for k, p in h.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys() and any(k.startswith("cls_branches") for k in grads[0])
    for k in grads[0]:
        a, b = grads[0][k].flatten(), grads[1][k].flatten()
        if dtype == torch.float32:
            cos = (a @ b) / (a.norm() * b.norm()).clamp(min=1e-300)
            assert cos >= 0.9999 or (a.norm() == 0 and b.norm() == 0), (k, cos.item())
        else:
            ea, eb = (a @ a).item(), (b @ b).item()
            assert abs(ea - eb) <= 0.01 * max(eb, 1e-30), (k, ea, eb)
