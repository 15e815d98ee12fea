"""BEVFormer's detection head and its NMS-free box coder on the CUDA library.

Drop-ins for the reference classes of the same names (projects/mmdet3d_plugin/bevformer/dense_heads/bevformer_head.py,
projects/mmdet3d_plugin/core/bbox/coders/nms_free_coder.py, mmdet 2.14's LearnedPositionalEncoding): same constructor
arguments, parameter names and return values, and ``loss`` with the reference's signature and loss dict.

What changes underneath:
  * the classification / regression branches of every decoder level and the box-centre arithmetic after them run as
    one kernel (``ops.det_branches_forward``) for bf16 / fp16 decoder states; fp32 states and calls that need a
    gradient run the head's own ``nn.Sequential`` branches and the reference's arithmetic in torch;
  * the coder's sigmoid / top-k / denormalisation / score threshold / centre-range filter is one kernel per batch
    (``ops.nms_free_decode``) with fixed-capacity outputs and no host synchronisation (``decode_device``);
    ``decode`` and ``get_bboxes`` synchronise once to slice the detections;
  * ``loss`` builds the matching cost of every decoder layer, group and sample in one kernel
    (``ops.det_match_cost``), copies it to the host once -- the call's only synchronisation -- and runs the
    reference's own ``scipy.optimize.linear_sum_assignment`` on each (layer, group, sample) slice; targets, focal and
    L1 / smooth-L1 losses and their gradients are one kernel each way (``ops.DetLoss``), with the avg factors kept
    in device memory.
"""
from __future__ import annotations

import copy
import math
import types

import torch
import torch.nn as nn

from .. import ops
from .decoder import _run_branch, inverse_sigmoid
from .registry import BBOX_CODERS, HEADS, POSITIONAL_ENCODING, TRANSFORMER, _register, build_from_cfg


def bias_init_with_prob(prior_prob):
    """mmcv.cnn.bias_init_with_prob: the bias whose sigmoid is ``prior_prob``."""
    return float(-math.log((1 - prior_prob) / prior_prob))


class LearnedPositionalEncoding(nn.Module):
    """mmdet 2.14 (models/utils/positional_encoding.py): ``pos[b, :, i, j] = cat(col_embed[j], row_embed[i])``,
    (bs, 2 * num_feats, h, w) for a (bs, h, w) mask.  ``init_weights`` draws both tables from U(0, 1), the
    ``init_cfg=dict(type='Uniform', layer='Embedding')`` of the original."""

    def __init__(self, num_feats, row_num_embed=50, col_num_embed=50, init_cfg=None):
        super().__init__()
        self.row_embed = nn.Embedding(row_num_embed, num_feats)
        self.col_embed = nn.Embedding(col_num_embed, num_feats)
        self.num_feats = num_feats
        self.row_num_embed = row_num_embed
        self.col_num_embed = col_num_embed
        self.init_cfg = init_cfg

    def init_weights(self):
        nn.init.uniform_(self.row_embed.weight)
        nn.init.uniform_(self.col_embed.weight)

    def forward(self, mask):
        h, w = mask.shape[-2:]
        x_embed = self.col_embed(torch.arange(w, device=mask.device))
        y_embed = self.row_embed(torch.arange(h, device=mask.device))
        pos = torch.cat((x_embed.unsqueeze(0).repeat(h, 1, 1), y_embed.unsqueeze(1).repeat(1, w, 1)), dim=-1)
        return pos.permute(2, 0, 1).unsqueeze(0).repeat(mask.shape[0], 1, 1, 1)


class NMSFreeCoder:
    """nms_free_coder.py:9-121 on ``ops.nms_free_decode``.  ``decode`` returns the reference's list of dicts (one
    host synchronisation, to slice each sample's detections); ``decode_device`` returns the fixed-capacity tensors
    without synchronising.  Candidates with equal scores come in ascending flat-index order."""

    def __init__(self, pc_range, voxel_size=None, post_center_range=None, max_num=100, score_threshold=None,
                 num_classes=10):
        self.pc_range = pc_range
        self.voxel_size = voxel_size
        self.post_center_range = post_center_range
        self.max_num = max_num
        self.score_threshold = score_threshold
        self.num_classes = num_classes

    def encode(self):
        pass

    def decode_device(self, preds_dicts, z_shift=False):
        """Last decoder level of ``preds_dicts`` -> dict(bboxes (bs, max_num, 9) f32, scores (bs, max_num) f32,
        labels (bs, max_num) i64, num (bs,) i32); sample i's detections are its first num[i] rows, the rest zero.
        ``z_shift``: BEVFormerHead.get_bboxes' bottom-centre z (z - h / 2)."""
        cls_scores = preds_dicts["all_cls_scores"][-1]
        bbox_preds = preds_dicts["all_bbox_preds"][-1]
        if cls_scores.shape[-1] != self.num_classes:
            raise RuntimeError(f"NMSFreeCoder: {cls_scores.shape[-1]} score channels for num_classes="
                               f"{self.num_classes}")
        bboxes, scores, labels, num = ops.nms_free_decode(cls_scores.contiguous(), bbox_preds.contiguous(),
                                                          self.max_num, self.post_center_range,
                                                          self.score_threshold, z_shift)
        return dict(bboxes=bboxes, scores=scores, labels=labels, num=num)

    def decode(self, preds_dicts, z_shift=False):
        out = self.decode_device(preds_dicts, z_shift)
        return [dict(bboxes=out["bboxes"][i, :n], scores=out["scores"][i, :n], labels=out["labels"][i, :n])
                for i, n in enumerate(out["num"].tolist())]


def _loss_cfg(cfg):
    """A loss config kept for its settings, with mmdet 2.14's defaults: ``use_sigmoid`` (FocalLoss: True),
    ``loss_weight`` 1, FocalLoss's ``gamma`` 2 / ``alpha`` 0.25, SmoothL1Loss's ``beta`` 1."""
    cfg = dict(cfg or {})
    cfg.setdefault("use_sigmoid", cfg.get("type") == "FocalLoss")
    cfg.setdefault("loss_weight", 1.0)
    if cfg.get("type") == "FocalLoss":
        cfg.setdefault("gamma", 2.0)
        cfg.setdefault("alpha", 0.25)
    if cfg.get("type") == "SmoothL1Loss":
        cfg.setdefault("beta", 1.0)
    return types.SimpleNamespace(**cfg)


_REG_COSTS = {"BBox3DL1Cost": "l1", "SmoothL1Cost": "smooth_l1"}
_REG_LOSSES = {"L1Loss": "l1", "SmoothL1Loss": "smooth_l1"}


def _loss_settings(head):
    """The assigner's and losses' settings ``loss`` runs with (``train_cfg['assigner']``, ``loss_cls``,
    ``loss_bbox``), checked as mmdet 2.14's DETRHead checks them: the cost and loss weights must agree.  Only the
    costs and losses the shipped configs use are implemented; anything else raises."""
    assigner = (head.train_cfg or {}).get("assigner")
    if assigner is None:
        raise RuntimeError(f"{type(head).__name__}.loss: train_cfg has no 'assigner' (the detector passes "
                           "train_cfg['pts'] of the config, which holds HungarianAssigner3D's settings)")
    if assigner.get("type", "HungarianAssigner3D") != "HungarianAssigner3D":
        raise NotImplementedError(f"loss: assigner {assigner.get('type')!r}; only HungarianAssigner3D is implemented")
    cls_cost = dict(assigner.get("cls_cost", dict(type="ClassificationCost", weight=1.0)))
    reg_cost = dict(assigner.get("reg_cost", dict(type="BBoxL1Cost", weight=1.0)))
    if cls_cost.get("type") != "FocalLossCost":
        raise NotImplementedError(f"loss: cls_cost {cls_cost.get('type')!r}; only FocalLossCost is implemented")
    if reg_cost.get("type") not in _REG_COSTS:
        raise NotImplementedError(f"loss: reg_cost {reg_cost.get('type')!r}; only {sorted(_REG_COSTS)} are "
                                  "implemented")
    lc, lb = head.loss_cls, head.loss_bbox
    if getattr(lc, "type", None) != "FocalLoss" or not lc.use_sigmoid:
        raise NotImplementedError(f"loss: loss_cls {getattr(lc, 'type', None)!r}; only FocalLoss(use_sigmoid=True) "
                                  "is implemented")
    if getattr(lb, "type", None) not in _REG_LOSSES:
        raise NotImplementedError(f"loss: loss_bbox {getattr(lb, 'type', None)!r}; only {sorted(_REG_LOSSES)} are "
                                  "implemented")
    for name, loss in (("loss_cls", lc), ("loss_bbox", lb)):
        if getattr(loss, "reduction", "mean") != "mean":
            raise NotImplementedError(f"loss: {name} with reduction={loss.reduction!r}; only 'mean' is implemented")
    cls_w, reg_w = cls_cost.get("weight", 1.0), reg_cost.get("weight", 1.0)
    if lc.loss_weight != cls_w:
        raise ValueError(f"loss: the classification weight for loss and matcher should be exactly the same "
                         f"(loss_cls.loss_weight {lc.loss_weight}, cls_cost.weight {cls_w})")
    if lb.loss_weight != reg_w:
        raise ValueError(f"loss: the regression weight for loss and matcher should be exactly the same "
                         f"(loss_bbox.loss_weight {lb.loss_weight}, reg_cost.weight {reg_w})")
    return dict(cost_reg_kind=_REG_COSTS[reg_cost["type"]], cls_cost_weight=float(cls_w),
                reg_cost_weight=float(reg_w), cost_alpha=float(cls_cost.get("alpha", 0.25)),
                cost_gamma=float(cls_cost.get("gamma", 2)), cost_eps=float(cls_cost.get("eps", 1e-12)),
                reg_kind=_REG_LOSSES[lb.type], cls_loss_weight=float(lc.loss_weight),
                bbox_loss_weight=float(lb.loss_weight), alpha=float(lc.alpha), gamma=float(lc.gamma),
                beta=float(getattr(lb, "beta", 1.0)))


def gravity_center_boxes(boxes):
    """``cat(gravity_center, tensor[:, 3:])`` (bevformer_head.py:441-443) as an (n, 9) float32 tensor.  Takes an
    object with ``gravity_center`` and ``tensor`` (mmdet3d's LiDARInstance3DBoxes) or a plain (n, 9) tensor in that
    class's layout (x, y, z_bottom, w, l, h, yaw, vx, vy), whose gravity centre is z + h / 2."""
    if hasattr(boxes, "gravity_center") and hasattr(boxes, "tensor"):
        out = torch.cat((boxes.gravity_center, boxes.tensor[:, 3:]), dim=1)
    elif torch.is_tensor(boxes):
        if boxes.dim() != 2:
            raise ValueError(f"loss: ground-truth boxes of shape {tuple(boxes.shape)}; need (n, 9)")
        out = torch.cat((boxes[:, :2], boxes[:, 2:3] + boxes[:, 5:6] * 0.5, boxes[:, 3:]), dim=1)
    else:
        raise TypeError(f"loss: ground-truth boxes of type {type(boxes).__name__}; need LiDARInstance3DBoxes-like "
                        "objects or (n, 9) tensors")
    if out.shape[1] != 9:
        raise ValueError(f"loss: ground-truth boxes with {out.shape[1]} columns; need 9 (x, y, z, w, l, h, yaw, vx, "
                         "vy)")
    return out.float()


def _to_device(host, device):
    """A small host tensor on ``device`` without a synchronisation (pinned, non-blocking)."""
    if device.type != "cuda":
        return host
    return host.pin_memory().to(device, non_blocking=True)


def avg_factors(counts, num_layers, device, sync_cls_avg_factor):
    """(num_layers * groups, 2) float32 avg factors before max(., 1), in device memory: ``counts[g]`` is
    num_total_pos of group g (the same for every layer).  Column 1 (regression) is ``reduce_mean`` of the counts; column
    0 (classification) too with ``sync_cls_avg_factor``, else the local count.  Under torch.distributed the mean is ONE
    all_reduce of every slot's count divided by the world size, and nothing is read back."""
    import torch.distributed as dist
    host = torch.tensor(counts, dtype=torch.float32).repeat(num_layers)[:, None].repeat(1, 2)
    avg = _to_device(host, device)
    if dist.is_available() and dist.is_initialized():
        red = avg[:, 1].clone().div_(dist.get_world_size())
        dist.all_reduce(red)
        avg[:, 1] = red
        if sync_cls_avg_factor:
            avg[:, 0] = red
    return avg


def _linear_sum_assignment():
    try:
        from scipy.optimize import linear_sum_assignment
    except ImportError as e:
        raise ImportError('Please run "pip install scipy" to install scipy first.') from e
    return linear_sum_assignment


class BEVFormerHead(nn.Module):
    """bevformer_head.py:16-213 and 482-509 (with mmdet 2.14 DETRHead's constructor).  ``forward`` passes the
    device-path keywords (``can_bus=``, ``lidar2img=``, ``ego_state=``, ``ego_mode=``) through to the transformer."""

    def __init__(self, num_classes, in_channels, num_query=100, num_reg_fcs=2, transformer=None,
                 sync_cls_avg_factor=False, positional_encoding=dict(type="SinePositionalEncoding", num_feats=128,
                                                                     normalize=True),
                 loss_cls=dict(type="CrossEntropyLoss", bg_cls_weight=0.1, use_sigmoid=False, loss_weight=1.0,
                               class_weight=1.0),
                 loss_bbox=dict(type="L1Loss", loss_weight=5.0), loss_iou=dict(type="GIoULoss", loss_weight=2.0),
                 train_cfg=None, test_cfg=dict(max_per_img=100), init_cfg=None, with_box_refine=False,
                 as_two_stage=False, bbox_coder=None, num_cls_fcs=2, code_weights=None, bev_h=30, bev_w=30,
                 code_size=10, **kwargs):
        super().__init__()
        if as_two_stage:
            raise NotImplementedError("BEVFormerHead: as_two_stage=True has no implementation (the reference "
                                      "transformer has no two-stage path either)")
        self.bev_h, self.bev_w = bev_h, bev_w
        self.fp16_enabled = False
        self.with_box_refine = with_box_refine
        self.as_two_stage = as_two_stage
        self.code_size = code_size
        self.code_weights = code_weights if code_weights is not None else [1.0] * 8 + [0.2, 0.2]
        self.bbox_coder = build_from_cfg(bbox_coder, BBOX_CODERS)
        self.pc_range = self.bbox_coder.pc_range
        self.real_w = self.pc_range[3] - self.pc_range[0]
        self.real_h = self.pc_range[4] - self.pc_range[1]
        self.num_cls_fcs = num_cls_fcs - 1
        self.init_cfg = init_cfg
        # DETRHead.__init__ (mmdet 2.14 dense_heads/detr_head.py)
        self.bg_cls_weight = 0
        self.sync_cls_avg_factor = sync_cls_avg_factor
        self.num_query = num_query
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.num_reg_fcs = num_reg_fcs
        self.train_cfg = train_cfg
        self.test_cfg = test_cfg
        self.loss_cls = _loss_cfg(loss_cls)
        self.loss_bbox = _loss_cfg(loss_bbox)
        self.loss_iou = _loss_cfg(loss_iou)
        self.cls_out_channels = num_classes if self.loss_cls.use_sigmoid else num_classes + 1
        self.activate = nn.ReLU(inplace=True)
        self.positional_encoding = build_from_cfg(positional_encoding, POSITIONAL_ENCODING)
        self.transformer = build_from_cfg(transformer, TRANSFORMER)
        self.embed_dims = self.transformer.embed_dims
        assert positional_encoding["num_feats"] * 2 == self.embed_dims
        self._init_layers()
        self.code_weights = nn.Parameter(torch.tensor(self.code_weights, requires_grad=False), requires_grad=False)

    def _init_layers(self):
        cls_branch = []
        for _ in range(self.num_reg_fcs):
            cls_branch += [nn.Linear(self.embed_dims, self.embed_dims), nn.LayerNorm(self.embed_dims),
                           nn.ReLU(inplace=True)]
        cls_branch.append(nn.Linear(self.embed_dims, self.cls_out_channels))
        fc_cls = nn.Sequential(*cls_branch)
        reg_branch = []
        for _ in range(self.num_reg_fcs):
            reg_branch += [nn.Linear(self.embed_dims, self.embed_dims), nn.ReLU()]
        reg_branch.append(nn.Linear(self.embed_dims, self.code_size))
        reg_branch = nn.Sequential(*reg_branch)
        num_pred = self.transformer.decoder.num_layers
        if self.with_box_refine:
            self.cls_branches = nn.ModuleList([copy.deepcopy(fc_cls) for _ in range(num_pred)])
            self.reg_branches = nn.ModuleList([copy.deepcopy(reg_branch) for _ in range(num_pred)])
        else:
            self.cls_branches = nn.ModuleList([fc_cls for _ in range(num_pred)])
            self.reg_branches = nn.ModuleList([reg_branch for _ in range(num_pred)])
        self.bev_embedding = nn.Embedding(self.bev_h * self.bev_w, self.embed_dims)
        self.query_embedding = nn.Embedding(self.num_query, self.embed_dims * 2)

    def init_weights(self):
        self.transformer.init_weights()
        if self.loss_cls.use_sigmoid:
            bias_init = bias_init_with_prob(0.01)
            for m in self.cls_branches:
                nn.init.constant_(m[-1].bias, bias_init)

    def _object_query_embeds(self, dtype):
        return self.query_embedding.weight.to(dtype)

    def forward(self, mlvl_feats, img_metas, prev_bev=None, only_bev=False, **device_kwargs):
        """Returns dict(bev_embed, all_cls_scores (L, bs, nq, cls_out_channels), all_bbox_preds (L, bs, nq, 10),
        enc_cls_scores=None, enc_bbox_preds=None); with ``only_bev`` the BEV features alone."""
        if self.fp16_enabled:                              # mmcv's auto_fp16(apply_to=('mlvl_feats'))
            mlvl_feats = [f.half() for f in mlvl_feats]
        bs = mlvl_feats[0].shape[0]
        dtype = mlvl_feats[0].dtype
        object_query_embeds = self._object_query_embeds(dtype)
        bev_queries = self.bev_embedding.weight.to(dtype)
        bev_mask = torch.zeros((bs, self.bev_h, self.bev_w), device=bev_queries.device).to(dtype)
        bev_pos = self.positional_encoding(bev_mask).to(dtype)
        grid_length = (self.real_h / self.bev_h, self.real_w / self.bev_w)
        if only_bev:
            return self.transformer.get_bev_features(mlvl_feats, bev_queries, self.bev_h, self.bev_w,
                                                     grid_length=grid_length, bev_pos=bev_pos, img_metas=img_metas,
                                                     prev_bev=prev_bev, **device_kwargs)
        bev_embed, hs, init_reference, inter_references = self.transformer(
            mlvl_feats, bev_queries, object_query_embeds, self.bev_h, self.bev_w, grid_length=grid_length,
            bev_pos=bev_pos, reg_branches=self.reg_branches if self.with_box_refine else None, cls_branches=None,
            img_metas=img_metas, prev_bev=prev_bev, **device_kwargs)
        cls_scores, bbox_preds = self.branches(hs, init_reference, inter_references)
        return {"bev_embed": bev_embed, "all_cls_scores": cls_scores, "all_bbox_preds": bbox_preds,
                "enc_cls_scores": None, "enc_bbox_preds": None}

    def branches(self, hs, init_reference, inter_references):
        """The per-level branches and box-centre arithmetic on the decoder output hs (L, nq, bs, C).  16-bit CUDA
        states without a gradient to compute: one ``bevf_det_branches_forward`` launch; otherwise the modules."""
        params = [p for m in (self.cls_branches, self.reg_branches) for p in m.parameters()]
        needs_grad = torch.is_grad_enabled() and (hs.requires_grad or any(p.requires_grad for p in params))
        if hs.is_cuda and hs.dtype in ops.TC_DTYPES and not needs_grad:
            tables = [ops.det_branch_params(c, r) for c, r in zip(self.cls_branches, self.reg_branches)]
            pdt = tables[0][0].dtype
            if pdt not in (hs.dtype, torch.float32) or any(t.dtype != pdt for ts in tables for t in ts):
                tables = [[t.float() for t in ts] for ts in tables]
            with torch.no_grad():
                return ops.det_branches_forward(hs, init_reference, inter_references, tables, self.pc_range,
                                                self.cls_branches[0][1].eps)
        return self._branches_modules(hs, init_reference, inter_references)

    def _branches_modules(self, hs, init_reference, inter_references):
        """bevformer_head.py:172-203 as written."""
        hs = hs.permute(0, 2, 1, 3)
        outputs_classes, outputs_coords = [], []
        for lvl in range(hs.shape[0]):
            reference = inverse_sigmoid(init_reference if lvl == 0 else inter_references[lvl - 1])
            outputs_class = _run_branch(self.cls_branches[lvl], hs[lvl])
            tmp = _run_branch(self.reg_branches[lvl], hs[lvl])
            assert reference.shape[-1] == 3
            tmp[..., 0:2] += reference[..., 0:2]
            tmp[..., 0:2] = tmp[..., 0:2].sigmoid()
            tmp[..., 4:5] += reference[..., 2:3]
            tmp[..., 4:5] = tmp[..., 4:5].sigmoid()
            tmp[..., 0:1] = tmp[..., 0:1] * (self.pc_range[3] - self.pc_range[0]) + self.pc_range[0]
            tmp[..., 1:2] = tmp[..., 1:2] * (self.pc_range[4] - self.pc_range[1]) + self.pc_range[1]
            tmp[..., 4:5] = tmp[..., 4:5] * (self.pc_range[5] - self.pc_range[2]) + self.pc_range[2]
            outputs_classes.append(outputs_class)
            outputs_coords.append(tmp)
        return torch.stack(outputs_classes), torch.stack(outputs_coords)

    def loss(self, gt_bboxes_list, gt_labels_list, preds_dicts, gt_bboxes_ignore=None, img_metas=None):
        """bevformer_head.py:395-480: dict(loss_cls, loss_bbox, d0.loss_cls, d0.loss_bbox, ..., d{L-2}.*) of the
        last and the earlier decoder layers.  ``gt_bboxes_list``: per sample, LiDARInstance3DBoxes-like objects or
        (n, 9) tensors (``gravity_center_boxes``); ``gt_labels_list``: per sample, (n,) class indices.  Synchronises
        with the host once (the cost matrix for scipy's assignment); not capturable."""
        return self._loss(gt_bboxes_list, gt_labels_list, preds_dicts, gt_bboxes_ignore, 1)

    def _loss(self, gt_bboxes_list, gt_labels_list, preds_dicts, gt_bboxes_ignore, groups):
        assert gt_bboxes_ignore is None, \
            f"{self.__class__.__name__} only supports for gt_bboxes_ignore setting to None."
        if preds_dicts.get("enc_cls_scores") is not None or preds_dicts.get("enc_bbox_preds") is not None:
            raise NotImplementedError("loss: encoder proposals (as_two_stage) have no implementation")
        st = _loss_settings(self)
        cls, box = preds_dicts["all_cls_scores"], preds_dicts["all_bbox_preds"]
        L, bs, nq, ncls = cls.shape
        if len(gt_bboxes_list) != bs or len(gt_labels_list) != bs:
            raise ValueError(f"loss: {len(gt_bboxes_list)} box lists and {len(gt_labels_list)} label lists for a "
                             f"batch of {bs}")
        if nq % groups:
            raise ValueError(f"loss: {nq} queries do not split into {groups} groups")
        nqg = nq // groups
        device = cls.device
        # 1. the ground truth, padded to the batch's largest count
        boxes = [gravity_center_boxes(b) for b in gt_bboxes_list]
        n = [int(b.shape[0]) for b in boxes]
        for b, lab in zip(boxes, gt_labels_list):
            if lab.numel() != b.shape[0]:
                raise ValueError(f"loss: {lab.numel()} labels for {b.shape[0]} boxes")
        G = max(n)
        gt = torch.zeros((bs, G, 9), dtype=torch.float32, device=device)
        labels = torch.zeros((bs, G), dtype=torch.int64, device=device)
        for i, (b, lab) in enumerate(zip(boxes, gt_labels_list)):
            if n[i]:
                gt[i, :n[i]].copy_(b, non_blocking=True)
                labels[i, :n[i]].copy_(lab.reshape(-1), non_blocking=True)
        n_gt = _to_device(torch.tensor(n, dtype=torch.int32), device)
        # num_total_pos of each group is known from the shapes: every sample matches min(n_gt, queries per group)
        avg = avg_factors([sum(min(k, nqg) for k in n)] * groups, L, device, self.sync_cls_avg_factor)
        # 2-4. one cost launch, one device-to-host copy, scipy per (layer, group, sample)
        assign = torch.full((L * bs, nq), -1, dtype=torch.int32)
        if G:
            cost = ops.det_match_cost(cls, box, gt, labels, n_gt, st["cost_reg_kind"], st["cls_cost_weight"],
                                      st["reg_cost_weight"], st["cost_alpha"], st["cost_gamma"],
                                      st["cost_eps"]).cpu().numpy()
            lsa = _linear_sum_assignment()
            a = assign.numpy()
            for p in range(L * bs):
                k = n[p % bs]
                if not k:
                    continue
                for g in range(groups):
                    rows, cols = lsa(cost[p, g * nqg:(g + 1) * nqg, :k])
                    a[p, g * nqg + rows] = cols
        # 5-6. the assignment back to the device, one loss launch
        assign = _to_device(assign, device)
        cfg = dict(groups=groups, reg_kind=st["reg_kind"], cls_loss_weight=st["cls_loss_weight"],
                   bbox_loss_weight=st["bbox_loss_weight"], alpha=st["alpha"], gamma=st["gamma"], beta=st["beta"])
        slots = ops.DetLoss.apply(cls, box, assign, gt, labels, n_gt, self.code_weights.float(), avg, cfg)
        # GroupDETR: each layer's losses summed over groups divided by group_detr (bevformer_head.py:666-682)
        per_layer = slots if groups == 1 else (slots.view(L, groups, 2) / groups).sum(1)
        layers = [row.unbind(0) for row in per_layer.unbind(0)]
        loss_dict = {"loss_cls": layers[-1][0], "loss_bbox": layers[-1][1]}
        for i, (lc, lb) in enumerate(layers[:-1]):
            loss_dict[f"d{i}.loss_cls"] = lc
            loss_dict[f"d{i}.loss_bbox"] = lb
        return loss_dict

    def get_bboxes(self, preds_dicts, img_metas, rescale=False):
        """bevformer_head.py:482-509: [[bboxes, scores, labels]] per sample, boxes with a bottom-centre z.  The
        boxes are wrapped in ``img_metas[i]['box_type_3d']`` when the meta carries one, else the (n, 9) tensor."""
        out = self.bbox_coder.decode_device(preds_dicts, z_shift=True)
        ret_list = []
        for i, n in enumerate(out["num"].tolist()):
            bboxes = out["bboxes"][i, :n]
            if img_metas is not None and "box_type_3d" in img_metas[i]:
                bboxes = img_metas[i]["box_type_3d"](bboxes, bboxes.shape[-1])
            ret_list.append([bboxes, out["scores"][i, :n], out["labels"][i, :n]])
        return ret_list


class BEVFormerHead_GroupDETR(BEVFormerHead):
    """bevformer_head.py:512-601: ``group_detr`` groups of ``num_query`` object queries in training; eval uses the
    first group only."""

    def __init__(self, *args, group_detr=1, **kwargs):
        self.group_detr = group_detr
        assert "num_query" in kwargs
        kwargs["num_query"] = group_detr * kwargs["num_query"]
        super().__init__(*args, **kwargs)

    def _object_query_embeds(self, dtype):
        q = self.query_embedding.weight.to(dtype)
        return q if self.training else q[:self.num_query // self.group_detr]

    def loss(self, gt_bboxes_list, gt_labels_list, preds_dicts, gt_bboxes_ignore=None, img_metas=None):
        """bevformer_head.py:603-683: ``BEVFormerHead.loss`` per group of ``num_query // group_detr`` queries, each
        layer's losses summed over the groups divided by ``group_detr``.  Still one cost launch, one synchronisation
        and one loss launch for all groups."""
        return self._loss(gt_bboxes_list, gt_labels_list, preds_dicts, gt_bboxes_ignore, self.group_detr)


_register(POSITIONAL_ENCODING, LearnedPositionalEncoding)
_register(BBOX_CODERS, NMSFreeCoder)
_register(HEADS, BEVFormerHead)
_register(HEADS, BEVFormerHead_GroupDETR)
