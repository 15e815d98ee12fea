"""Generates the detection-loss goldens from the REFERENCE'S OWN BEVFormerHead.loss / loss_single / get_targets
(dense_heads/bevformer_head.py), BEVFormerHead_GroupDETR.loss, HungarianAssigner3D
(core/bbox/assigners/hungarian_assigner_3d.py), BBox3DL1Cost / SmoothL1Cost (core/bbox/match_costs/match_cost.py) and
normalize_bbox (core/bbox/util.py), imported unmodified behind oracle/mmcv_stub.py and the loader of
make_golden_head.py, with the mmdet 2.14 / mmcv 1.4 pieces they import restated below.  Needs a reference checkout
(BEVF_REFERENCE_ROOT) and scipy; the test suite does not need the reference:

    python tests/golden/make_golden_loss.py

Writes ref_det_loss_<case>.npz for the cases of tests/det_loss_oracle.py (inputs regenerated from the seed there):
  fp64_<loss key> / fp32_<loss key>       the loss dict, predictions and ground truth in float64 / float32
  assign                                  (L * bs, nq) int32 ground-truth index of every query (-1 unmatched), equal
                                          in both precisions
  grad_rows                               flat row indices (l * bs + b) * nq + q: every matched row and every 8th row
  fp64_grad_cls / _box, fp32_grad_*       d(sum of the loss dict) / d(all_cls_scores / all_bbox_preds) on those rows
  margin                                  the smallest rise of the fp32 optimum when one matched pair is forbidden
The "tiny" case is a head built from bevformer_tiny.py's pts_bbox_head and train_cfg['pts'] dicts (its transformer
replaced by fixed outputs); it also stores those dicts for bevformer_tiny / base and bevformerv2 as JSON.
"""
from __future__ import annotations

import copy
import importlib.util
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bevformer_b200.plugin import config  # noqa: E402
from oracle import mmcv_stub  # noqa: E402
from oracle.mmcv_stub import Registry, build_from_cfg  # noqa: E402
from tests import det_loss_oracle as dlo  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
PLUGIN = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "mmdet3d_plugin")
FLT_MIN = float(np.finfo(np.float32).tiny)
GRAD_ROW_STRIDE = 8


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


mgh = _load("_bevf_make_golden_head", os.path.join(OUT, "make_golden_head.py"))


# ---- mmcv 1.4 / mmdet 2.14 pieces the reference loss imports, restated --------------------------------------------
class _SigmoidFocalLossCUDA(torch.autograd.Function):
    """mmcv 1.4 ops/csrc/common/cuda/sigmoid_focal_loss_cuda_kernel.cuh, forward and analytic backward, elementwise
    (reduction 'none', no weight)."""

    @staticmethod
    def forward(ctx, x, target, gamma, alpha):
        flag_p = (target[:, None] == torch.arange(x.shape[1])[None]).to(x.dtype)
        p = 1.0 / (1.0 + torch.exp(-x))
        term_p = (1.0 - p).pow(gamma) * torch.log(p.clamp(min=FLT_MIN))
        term_n = p.pow(gamma) * torch.log((1.0 - p).clamp(min=FLT_MIN))
        ctx.save_for_backward(x, flag_p)
        ctx.gamma, ctx.alpha = gamma, alpha
        return -flag_p * alpha * term_p - (1 - flag_p) * (1.0 - alpha) * term_n

    @staticmethod
    def backward(ctx, grad):
        x, flag_p = ctx.saved_tensors
        gamma, alpha = ctx.gamma, ctx.alpha
        p = 1.0 / (1.0 + torch.exp(-x))
        term_p = (1.0 - p).pow(gamma) * (1.0 - p - gamma * p * torch.log(p.clamp(min=FLT_MIN)))
        term_n = p.pow(gamma) * (gamma * (1.0 - p) * torch.log((1.0 - p).clamp(min=FLT_MIN)) - p)
        g = -flag_p * alpha * term_p - (1 - flag_p) * (1.0 - alpha) * term_n
        return g * grad, None, None, None


def weight_reduce_loss(loss, weight=None, reduction="mean", avg_factor=None):
    """mmdet 2.14 models/losses/utils.py."""
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        return loss.mean() if reduction == "mean" else (loss.sum() if reduction == "sum" else loss)
    if reduction == "mean":
        return loss.sum() / avg_factor
    if reduction != "none":
        raise ValueError('avg_factor can not be used with reduction="sum"')
    return loss


class FocalLoss(torch.nn.Module):
    """mmdet 2.14 models/losses/focal_loss.py, use_sigmoid=True on CUDA (mmcv's sigmoid_focal_loss)."""

    def __init__(self, type=None, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction="mean", loss_weight=1.0):
        super().__init__()
        assert use_sigmoid
        self.use_sigmoid, self.gamma, self.alpha = use_sigmoid, gamma, alpha
        self.reduction, self.loss_weight = reduction, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        reduction = reduction_override if reduction_override else self.reduction
        loss = _SigmoidFocalLossCUDA.apply(pred.contiguous(), target, self.gamma, self.alpha)
        if weight is not None and weight.shape != loss.shape and weight.size(0) == loss.size(0):
            weight = weight.view(-1, 1)
        return self.loss_weight * weight_reduce_loss(loss, weight, reduction, avg_factor)


class L1Loss(torch.nn.Module):
    """mmdet 2.14 models/losses/smooth_l1_loss.py:L1Loss (with @weighted_loss)."""

    def __init__(self, type=None, reduction="mean", loss_weight=1.0):
        super().__init__()
        self.reduction, self.loss_weight = reduction, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        reduction = reduction_override if reduction_override else self.reduction
        loss = pred.sum() * 0 if target.numel() == 0 else torch.abs(pred - target)
        return self.loss_weight * weight_reduce_loss(loss, weight, reduction, avg_factor)


class SmoothL1Loss(torch.nn.Module):
    """mmdet 2.14 models/losses/smooth_l1_loss.py:SmoothL1Loss (with @weighted_loss)."""

    def __init__(self, type=None, beta=1.0, reduction="mean", loss_weight=1.0):
        super().__init__()
        self.beta, self.reduction, self.loss_weight = beta, reduction, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        reduction = reduction_override if reduction_override else self.reduction
        if target.numel() == 0:
            loss = pred.sum() * 0
        else:
            diff = torch.abs(pred - target)
            loss = torch.where(diff < self.beta, 0.5 * diff * diff / self.beta, diff - 0.5 * self.beta)
        return self.loss_weight * weight_reduce_loss(loss, weight, reduction, avg_factor)


LOSSES = {"FocalLoss": FocalLoss, "L1Loss": L1Loss, "SmoothL1Loss": SmoothL1Loss}


class FocalLossCost:
    """mmdet 2.14 core/bbox/match_costs/match_cost.py:FocalLossCost."""

    def __init__(self, weight=1., alpha=0.25, gamma=2, eps=1e-12):
        self.weight, self.alpha, self.gamma, self.eps = weight, alpha, gamma, eps

    def __call__(self, cls_pred, gt_labels):
        cls_pred = cls_pred.sigmoid()
        neg_cost = -(1 - cls_pred + self.eps).log() * (1 - self.alpha) * cls_pred.pow(self.gamma)
        pos_cost = -(cls_pred + self.eps).log() * self.alpha * (1 - cls_pred).pow(self.gamma)
        cls_cost = pos_cost[:, gt_labels] - neg_cost[:, gt_labels]
        return cls_cost * self.weight


class IoUCost:
    """mmdet 2.14 IoUCost: built by the assigner, never called by HungarianAssigner3D."""

    def __init__(self, iou_mode="giou", weight=1.):
        self.weight, self.iou_mode = weight, iou_mode


class AssignResult:
    """mmdet 2.14 core/bbox/assigners/assign_result.py (the fields the head reads)."""

    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels


class BaseAssigner:
    pass


class SamplingResult:
    """mmdet 2.14 core/bbox/samplers/sampling_result.py (but for the empty-ground-truth case below)."""

    def __init__(self, pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags):
        self.pos_inds, self.neg_inds = pos_inds, neg_inds
        self.pos_bboxes, self.neg_bboxes = bboxes[pos_inds], bboxes[neg_inds]
        self.pos_is_gt = gt_flags[pos_inds]
        self.num_gts = gt_bboxes.shape[0]
        self.pos_assigned_gt_inds = assign_result.gt_inds[pos_inds] - 1
        if gt_bboxes.numel() == 0:
            # mmdet views the empty targets as (0, 4), which torch refuses to assign to the head's 9-column targets;
            # the box width is kept here, so a sample without ground truth has every query background
            assert self.pos_assigned_gt_inds.numel() == 0
            self.pos_gt_bboxes = torch.empty_like(gt_bboxes).view(-1, gt_bboxes.shape[-1])
        else:
            if len(gt_bboxes.shape) < 2:
                gt_bboxes = gt_bboxes.view(-1, 4)
            self.pos_gt_bboxes = gt_bboxes[self.pos_assigned_gt_inds, :]


class PseudoSampler:
    """mmdet 2.14 core/bbox/samplers/pseudo_sampler.py."""

    def __init__(self, **kwargs):
        pass

    def sample(self, assign_result, bboxes, gt_bboxes, **kwargs):
        pos_inds = torch.nonzero(assign_result.gt_inds > 0, as_tuple=False).squeeze(-1).unique()
        neg_inds = torch.nonzero(assign_result.gt_inds == 0, as_tuple=False).squeeze(-1).unique()
        gt_flags = bboxes.new_zeros(bboxes.shape[0], dtype=torch.uint8)
        return SamplingResult(pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags)


BBOX_ASSIGNERS, MATCH_COST = Registry("bbox_assigner"), Registry("match_cost")
for _c in (FocalLossCost, IoUCost):
    MATCH_COST.register_module(name=_c.__name__, module=_c)


class DETRHead(mgh.DETRHead):
    """mmdet 2.14 DETRHead.__init__ with its training part: the weight checks, the assigner of train_cfg, the
    PseudoSampler and the built losses."""

    def __init__(self, *args, loss_cls=None, loss_bbox=None, loss_iou=dict(type="GIoULoss", loss_weight=2.0),
                 train_cfg=None, **kwargs):
        super().__init__(*args, loss_cls=loss_cls, loss_bbox=loss_bbox, loss_iou=loss_iou, train_cfg=train_cfg,
                         **kwargs)
        assert train_cfg and "assigner" in train_cfg
        assigner = copy.deepcopy(train_cfg["assigner"])
        assert loss_cls["loss_weight"] == assigner["cls_cost"]["weight"]
        assert loss_bbox["loss_weight"] == assigner["reg_cost"]["weight"]
        assert loss_iou["loss_weight"] == assigner["iou_cost"]["weight"]
        self.assigner = build_from_cfg(assigner, BBOX_ASSIGNERS)
        self.sampler = PseudoSampler()
        self.loss_cls = LOSSES[loss_cls["type"]](**loss_cls)
        self.loss_bbox = LOSSES[loss_bbox["type"]](**loss_bbox)


def load_reference_loss():
    """(BEVFormerHead, BEVFormerHead_GroupDETR, hungarian_assigner_3d module) of the reference, unmodified."""
    mgh.DETRHead = DETRHead
    mmcv_stub.install_stub()
    sys.modules["mmcv"].jit = lambda *a, **k: (lambda fn: fn)
    util = _load("_bevf_ref_bbox_util_loss", os.path.join(PLUGIN, "core", "bbox", "util.py"))
    extra = {
        "mmdet": mmcv_stub._mod("mmdet"), "mmdet.core": mmcv_stub._mod("mmdet.core"),
        "mmdet.core.bbox": mmcv_stub._mod("mmdet.core.bbox"),
        "mmdet.core.bbox.builder": mmcv_stub._mod("mmdet.core.bbox.builder", BBOX_ASSIGNERS=BBOX_ASSIGNERS),
        "mmdet.core.bbox.assigners": mmcv_stub._mod("mmdet.core.bbox.assigners", AssignResult=AssignResult,
                                                    BaseAssigner=BaseAssigner),
        "mmdet.core.bbox.match_costs": mmcv_stub._mod(
            "mmdet.core.bbox.match_costs", build_match_cost=lambda cfg: build_from_cfg(cfg, MATCH_COST)),
        "mmdet.core.bbox.match_costs.builder": mmcv_stub._mod("mmdet.core.bbox.match_costs.builder",
                                                              MATCH_COST=MATCH_COST),
        "mmdet.models": mmcv_stub._mod("mmdet.models"), "mmdet.models.utils": mmcv_stub._mod("mmdet.models.utils"),
        "mmdet.models.utils.transformer": mmcv_stub._mod("mmdet.models.utils.transformer",
                                                         inverse_sigmoid=mgh.inverse_sigmoid),
        "projects.mmdet3d_plugin.core": mmcv_stub._mod("projects.mmdet3d_plugin.core"),
        "projects.mmdet3d_plugin.core.bbox": mmcv_stub._mod("projects.mmdet3d_plugin.core.bbox"),
        "projects.mmdet3d_plugin.core.bbox.util": util,
    }
    saved = {k: sys.modules.get(k) for k in extra}
    sys.modules.update(extra)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            costs = _load("_bevf_ref_match_cost", os.path.join(PLUGIN, "core", "bbox", "match_costs",
                                                               "match_cost.py"))
            assigner = _load("_bevf_ref_hungarian_assigner_3d", os.path.join(PLUGIN, "core", "bbox", "assigners",
                                                                            "hungarian_assigner_3d.py"))
    finally:
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    for name in ("BBox3DL1Cost", "SmoothL1Cost"):
        MATCH_COST.register_module(name=name, module=getattr(costs, name), force=True)
    BBOX_ASSIGNERS.register_module(name="HungarianAssigner3D", module=assigner.HungarianAssigner3D, force=True)
    Head, HeadG, _, _ = mgh.load_reference_head()
    return Head, HeadG, assigner


class _Boxes:
    """The two attributes BEVFormerHead.loss reads of mmdet3d's LiDARInstance3DBoxes."""

    def __init__(self, gravity_boxes):
        self.gravity_center = gravity_boxes[:, :3]
        self.tensor = torch.cat((gravity_boxes[:, :2], gravity_boxes[:, 2:3] - gravity_boxes[:, 5:6] * 0.5,
                                 gravity_boxes[:, 3:]), dim=1)


def head_cfg(settings, L, nq, groups, ncls):
    st = dlo.BASE if settings == "base" else dlo.V2
    reg_cost = {"l1": "BBox3DL1Cost", "smooth_l1": "SmoothL1Cost"}[st["cost_reg_kind"]]
    loss_bbox = (dict(type="L1Loss", loss_weight=st["bbox_loss_weight"]) if st["reg_kind"] == "l1" else
                 dict(type="SmoothL1Loss", loss_weight=st["bbox_loss_weight"], beta=st["beta"]))
    cfg = dict(num_query=nq // groups, num_classes=ncls, in_channels=256, sync_cls_avg_factor=True,
               with_box_refine=True, as_two_stage=False, bev_h=4, bev_w=5,
               transformer=dict(type="FixedDecoderOutputs", num_layers=L),
               bbox_coder=dict(type="NMSFreeCoder", post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
                               pc_range=dlo.PC_RANGE, max_num=300, num_classes=ncls),
               positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=4,
                                        col_num_embed=5),
               loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25,
                             loss_weight=st["cls_loss_weight"]),
               loss_bbox=loss_bbox, loss_iou=dict(type="GIoULoss", loss_weight=0.0),
               train_cfg=dict(assigner=dict(type="HungarianAssigner3D",
                                            cls_cost=dict(type="FocalLossCost", weight=st["cls_cost_weight"]),
                                            reg_cost=dict(type=reg_cost, weight=st["reg_cost_weight"]),
                                            iou_cost=dict(type="IoUCost", weight=0.0), pc_range=dlo.PC_RANGE)))
    if groups > 1:
        cfg["group_detr"] = groups
    return cfg


def run_case(name, case, hcfg=None):
    Head, HeadG, assigner_mod = load_reference_loss()
    L, bs, groups, nqg, ncls, n_gt, settings, nan_frac = case
    nq = groups * nqg
    seed = dlo.case_seed(name)
    cls64, box64, gts, labels = dlo.case_inputs(L, bs, groups, nqg, ncls, n_gt, nan_frac, seed)
    if hcfg is None:
        hcfg = head_cfg(settings, L, nq, groups, ncls)
    out, assigns, costs = {}, {}, {}
    for dt, tag in ((torch.float64, "fp64"), (torch.float32, "fp32")):
        record = []
        lsa = assigner_mod.linear_sum_assignment

        def recording(cost, record=record, lsa=lsa):
            r, c = lsa(cost)
            record.append((cost.numpy().copy(), r, c))
            return r, c
        assigner_mod.linear_sum_assignment = recording
        head = (HeadG if groups > 1 else Head)(**copy.deepcopy(hcfg))
        cls = cls64.to(dt).clone().requires_grad_(True)
        box = box64.to(dt).clone().requires_grad_(True)
        preds = dict(all_cls_scores=cls, all_bbox_preds=box, enc_cls_scores=None, enc_bbox_preds=None)
        losses = head.loss([_Boxes(g.to(dt)) for g in gts], [lab.clone() for lab in labels], preds)
        assigner_mod.linear_sum_assignment = lsa
        sum(v.sum() for v in losses.values()).backward()
        for k, v in losses.items():
            out[f"{tag}_{k}"] = np.asarray(v.detach().reshape(()).numpy())
        # the solver's calls come in the order (group,) layer, sample; samples without ground truth make none
        a = np.full((L * bs, nq), -1, np.int32)
        it = iter(record)
        for g in range(groups):
            for l in range(L):
                for b in range(bs):
                    if n_gt[b] == 0:
                        continue
                    cost, r, c = next(it)
                    a[l * bs + b, g * nqg + r] = c
                    costs.setdefault(tag, []).append((cost, r, c))
        assert next(it, None) is None
        assigns[tag] = a
        matched = (a >= 0).reshape(-1)
        rows = np.nonzero(matched | (np.arange(L * bs * nq) % nq % GRAD_ROW_STRIDE == 0))[0]
        out["grad_rows"] = rows
        out[f"{tag}_grad_cls"] = cls.grad.reshape(-1, ncls)[rows].numpy()
        out[f"{tag}_grad_box"] = box.grad.reshape(-1, 10)[rows].numpy()
    assert (assigns["fp64"] == assigns["fp32"]).all(), f"{name}: fp32 and fp64 assignments differ"
    out["assign"] = assigns["fp32"]
    margin = np.inf
    from scipy.optimize import linear_sum_assignment
    for cost, r, c in costs["fp32"]:
        best = cost[r, c].astype(np.float64).sum()
        for i, j in zip(r, c):
            alt = cost.copy()
            alt[i, j] = 1e30
            r2, c2 = linear_sum_assignment(alt)
            margin = min(margin, alt[r2, c2].astype(np.float64).sum() - best)
    assert margin >= 1e-3, f"{name}: assignment margin {margin} below 1e-3"
    out["margin"] = np.float64(margin)
    return out


def configs():
    """pts_bbox_head and train_cfg['pts'] of the shipped configs, as JSON."""
    out = {}
    for name, path in (("tiny", "bevformer/bevformer_tiny.py"), ("base", "bevformer/bevformer_base.py"),
                       ("v2", "bevformerv2/bevformerv2-r50-t1-24ep.py")):
        cfg = config.load_config(os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs", path))
        out[f"{name}_pts_bbox_head"] = np.array(json.dumps(cfg["model"]["pts_bbox_head"]))
        out[f"{name}_train_cfg"] = np.array(json.dumps(cfg["model"]["train_cfg"]["pts"]))
    return out


def tiny_head_cfg(cfgs):
    """bevformer_tiny.py's pts_bbox_head with its train_cfg, the transformer replaced by fixed decoder outputs."""
    h = json.loads(str(cfgs["tiny_pts_bbox_head"]))
    h.pop("type")
    h["transformer"] = dict(type="FixedDecoderOutputs", num_layers=h["transformer"]["decoder"]["num_layers"])
    h["train_cfg"] = json.loads(str(cfgs["tiny_train_cfg"]))
    return h


if __name__ == "__main__":
    if not mmcv_stub.reference_available():
        raise SystemExit("needs a reference checkout (set BEVF_REFERENCE_ROOT)")
    cfgs = configs()
    for name, case in dlo.CASES.items():
        hcfg = tiny_head_cfg(cfgs) if name == "tiny" else None
        out = run_case(name, case, hcfg)
        if name == "tiny":
            out.update(cfgs)
        path = os.path.join(OUT, f"ref_det_loss_{name}.npz")
        np.savez_compressed(path, **out)
        assert os.path.getsize(path) < 1 << 20, path
        print(f"ref_det_loss_{name}: margin {float(out['margin']):.4g}, loss_cls {float(out['fp64_loss_cls']):.6g}, "
              f"loss_bbox {float(out['fp64_loss_bbox']):.6g}, {os.path.getsize(path)} bytes")
