"""Float64 restatement of BEVFormerHead's training loss (dense_heads/bevformer_head.py:215-480 and 603-683) with
HungarianAssigner3D (core/bbox/assigners/hungarian_assigner_3d.py:52-131), mmdet 2.14's FocalLossCost, the 3D match
costs (core/bbox/match_costs/match_cost.py), normalize_bbox (core/bbox/util.py:4-24), mmcv's sigmoid focal loss and
mmdet's L1Loss / SmoothL1Loss.  Plain torch: runs on any device and dtype and is differentiable, so the GPU tests can
put it behind a head in place of the library's loss.  Also the golden cases' inputs (``case_inputs``).
"""
from __future__ import annotations

import numpy as np
import torch

PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
# the head keeps them in an fp32 Parameter: 0.2 is fp32's 0.2 in every precision
CODE_WEIGHTS = torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2], dtype=torch.float32).tolist()
FLT_MIN = float(np.finfo(np.float32).tiny)

# BEVFormer configs: FocalLoss(2.0) / FocalLossCost(2.0), L1Loss(0.25) / BBox3DL1Cost(0.25);
# BEVFormerV2 configs: the same focal terms, SmoothL1Loss(0.75, beta 1) / SmoothL1Cost(0.75)
BASE = dict(cost_reg_kind="l1", cls_cost_weight=2.0, reg_cost_weight=0.25, cost_alpha=0.25, cost_gamma=2.0,
            cost_eps=1e-12, reg_kind="l1", cls_loss_weight=2.0, bbox_loss_weight=0.25, alpha=0.25, gamma=2.0,
            beta=1.0)
V2 = dict(BASE, cost_reg_kind="smooth_l1", reg_cost_weight=0.75, reg_kind="smooth_l1", bbox_loss_weight=0.75)


def normalize_bbox(b):
    return torch.cat((b[..., 0:2], b[..., 3:4].log(), b[..., 4:5].log(), b[..., 2:3], b[..., 5:6].log(),
                      b[..., 6:7].sin(), b[..., 6:7].cos(), b[..., 7:9]), dim=-1)


def match_cost(cls, box, gt, labels, st, sigmoid=None):
    """(nq, n) cost of one (layer, group, sample): FocalLossCost + BBox3DL1Cost / SmoothL1Cost.  ``sigmoid`` overrides
    p = sigmoid(cls) (the GPU test passes torch.sigmoid's fp32 rounding, as the library's kernel takes it)."""
    p = cls.sigmoid() if sigmoid is None else sigmoid
    a, g, eps = st["cost_alpha"], st["cost_gamma"], st["cost_eps"]
    neg = -(1 - p + eps).log() * (1 - a) * p.pow(g)
    pos = -(p + eps).log() * a * (1 - p).pow(g)
    cls_cost = (pos[:, labels] - neg[:, labels]) * st["cls_cost_weight"]
    d = (box[:, None, :8] - normalize_bbox(gt)[None, :, :8]).abs()
    if st["cost_reg_kind"] == "l1":
        reg = d.sum(-1)
    else:
        reg = torch.where(d < 1.0, 0.5 * d * d, d - 0.5).sum(-1)
    return cls_cost + reg * st["reg_cost_weight"]


def assign(cost):
    """scipy's linear_sum_assignment on a (nq, n) cost: (rows, cols)."""
    from scipy.optimize import linear_sum_assignment
    return linear_sum_assignment(np.asarray(cost))


def focal_loss(x, target, alpha, gamma):
    """mmcv 1.4's sigmoid_focal_loss forward, elementwise; target (rows,) with num_classes for background."""
    p = x.sigmoid()
    onehot = torch.nn.functional.one_hot(target, x.shape[-1] + 1)[:, :x.shape[-1]].to(x.dtype)
    term_p = (1 - p).pow(gamma) * p.clamp(min=FLT_MIN).log()
    term_n = p.pow(gamma) * (1 - p).clamp(min=FLT_MIN).log()
    return -onehot * alpha * term_p - (1 - onehot) * (1 - alpha) * term_n


def slot_loss(cls, box, gts, labels, rows_cols, st, code_weights, cls_avg, reg_avg):
    """loss_single of one (layer, group): cls (bs, q, ncls), box (bs, q, 10); rows_cols[b] = (rows, cols) of the
    assignment.  Returns (loss_cls, loss_bbox) after nan_to_num."""
    bs, nq, ncls = cls.shape
    tgt_lab, tgt_box, pos = [], [], []
    for b in range(bs):
        rows, cols = (torch.as_tensor(np.asarray(v), dtype=torch.long, device=cls.device) for v in rows_cols[b])
        lab = torch.full((nq,), ncls, dtype=torch.long, device=cls.device)
        lab[rows] = labels[b].to(cls.device)[cols]
        tb = torch.zeros((nq, 9), dtype=cls.dtype, device=cls.device)
        tb[rows] = gts[b].to(cls.device, cls.dtype)[cols]
        w = torch.zeros((nq,), dtype=cls.dtype, device=cls.device)
        w[rows] = 1.0
        tgt_lab.append(lab), tgt_box.append(tb), pos.append(w)
    lab, tb, w = torch.cat(tgt_lab), torch.cat(tgt_box), torch.cat(pos)
    loss_cls = focal_loss(cls.reshape(-1, ncls), lab, st["alpha"], st["gamma"]).sum() / max(cls_avg, 1.0)
    loss_cls = loss_cls * st["cls_loss_weight"]
    nt = normalize_bbox(tb)
    keep = torch.isfinite(nt).all(-1)
    weights = (w[:, None] * torch.as_tensor(code_weights, dtype=cls.dtype, device=cls.device))[keep]
    d = (box.reshape(-1, 10)[keep] - nt[keep]).abs()
    if st["reg_kind"] == "l1":
        elem = d
    else:
        elem = torch.where(d < st["beta"], 0.5 * d * d / st["beta"], d - 0.5 * st["beta"])
    loss_bbox = (elem * weights).sum() / max(reg_avg, 1.0) * st["bbox_loss_weight"]
    return torch.nan_to_num(loss_cls), torch.nan_to_num(loss_bbox)


def loss(all_cls, all_box, gts, labels, st, groups=1, code_weights=CODE_WEIGHTS, assignment=None):
    """BEVFormerHead(_GroupDETR).loss on (L, bs, nq, ncls) / (L, bs, nq, 10) predictions and gravity-centred (n, 9)
    ground truth.  ``assignment[l][g][b] = (rows, cols)``, computed here from this restatement's own cost when None.
    Returns (loss dict, assignment)."""
    L, bs, nq, _ = all_cls.shape
    nqg = nq // groups
    count = float(sum(min(int(g.shape[0]), nqg) for g in gts))
    if assignment is None:
        assignment = []
        for l in range(L):
            per_group = []
            for g in range(groups):
                per_b = []
                for b in range(bs):
                    if gts[b].shape[0] == 0:
                        per_b.append((np.zeros(0, np.int64), np.zeros(0, np.int64)))
                        continue
                    c = match_cost(all_cls[l, b, g * nqg:(g + 1) * nqg].detach(),
                                   all_box[l, b, g * nqg:(g + 1) * nqg].detach(),
                                   gts[b].to(all_cls.device, all_cls.dtype), labels[b].to(all_cls.device), st)
                    per_b.append(assign(c.cpu().numpy()))
                per_group.append(per_b)
            assignment.append(per_group)
    out = {}
    for l in range(L):
        acc = [0, 0]
        for g in range(groups):
            lc, lb = slot_loss(all_cls[l, :, g * nqg:(g + 1) * nqg], all_box[l, :, g * nqg:(g + 1) * nqg], gts, labels,
                               assignment[l][g], st, code_weights, count, count)
            acc = [acc[0] + lc / groups, acc[1] + lb / groups] if groups > 1 else [lc, lb]
        key = "" if l == L - 1 else f"d{l}."
        out[key + "loss_cls"], out[key + "loss_bbox"] = acc
    return out, assignment


def assignment_array(assignment, L, bs, nq, groups):
    """``assignment`` as the (L * bs, nq) int32 array of ground-truth indices (-1 unmatched)."""
    a = np.full((L * bs, nq), -1, np.int32)
    nqg = nq // groups
    for l in range(L):
        for g in range(groups):
            for b in range(bs):
                rows, cols = assignment[l][g][b]
                a[l * bs + b, g * nqg + np.asarray(rows, np.int64)] = cols
    return a


# ---- golden cases ----------------------------------------------------------------------------------------------
CASES = {
    # name: (L, bs, groups, queries per group, ncls, n_gt per sample, settings, NaN-velocity fraction)
    "base": (6, 2, 1, 900, 10, (37, 0), "base", 0.0),
    "nanvel": (2, 2, 1, 200, 10, (24, 9), "base", 0.4),
    "group": (3, 2, 3, 50, 10, (60, 5), "v2", 0.0),
    "tiny": (6, 1, 1, 900, 10, (20,), "base", 0.1),       # a head built from bevformer_tiny.py's dicts
}


def case_seed(name):
    return 51000 + sorted(CASES).index(name)


def _bf16_grid(t):
    """Round to bf16 and keep |v| >= 2^-14, so the same values are exact in fp32, bf16 and fp16."""
    t = t.to(torch.bfloat16).to(torch.float64)
    small = t.abs() < 2.0 ** -14
    return torch.where(small, torch.full_like(t, 2.0 ** -14), t)


def case_inputs(L, bs, groups, nqg, ncls, n_gt, nan_frac, seed):
    """Predictions (L, bs, nq, ncls) logits in about [-12, 12] and boxes (L, bs, nq, 10), ground truth (n, 9) per
    sample with labels; each gt has a planted query per (layer, group) whose box and logit match it closely, so the
    optimal assignment is unique by a wide margin.  All prediction values lie on the bf16 grid."""
    g = torch.Generator().manual_seed(seed)
    nq = groups * nqg
    cls = torch.rand((L, bs, nq, ncls), generator=g, dtype=torch.float64) * 20 - 14
    box = torch.empty((L, bs, nq, 10), dtype=torch.float64)
    box[..., 0:2] = torch.rand((L, bs, nq, 2), generator=g, dtype=torch.float64) * 100 - 50
    box[..., 2:4] = torch.rand((L, bs, nq, 2), generator=g, dtype=torch.float64) * 2
    box[..., 4] = torch.rand((L, bs, nq), generator=g, dtype=torch.float64) * 4 - 3
    box[..., 5] = torch.rand((L, bs, nq), generator=g, dtype=torch.float64) * 1.5
    box[..., 6:8] = torch.rand((L, bs, nq, 2), generator=g, dtype=torch.float64) * 2 - 1
    box[..., 8:10] = torch.randn((L, bs, nq, 2), generator=g, dtype=torch.float64)
    gts, labels = [], []
    for b, n in enumerate(n_gt):
        gt = torch.empty((n, 9), dtype=torch.float64)
        gt[:, 0:2] = torch.rand((n, 2), generator=g, dtype=torch.float64) * 90 - 45
        gt[:, 2] = torch.rand((n,), generator=g, dtype=torch.float64) * 3 - 2
        gt[:, 3:6] = torch.rand((n, 3), generator=g, dtype=torch.float64) * 4 + 0.5
        gt[:, 6] = torch.rand((n,), generator=g, dtype=torch.float64) * 6.2 - 3.1
        gt[:, 7:9] = torch.randn((n, 2), generator=g, dtype=torch.float64)
        nan = torch.rand((n,), generator=g) < nan_frac
        gt[nan, 7:9] = float("nan")
        gt = gt.float().double()
        lab = torch.randint(0, ncls, (n,), generator=g)
        nt = normalize_bbox(gt)
        for l in range(L):
            for grp in range(groups):
                qs = grp * nqg + torch.randperm(nqg, generator=g)[:min(n, nqg)]
                k = len(qs)
                box[l, b, qs, :8] = nt[:k, :8] + torch.randn((k, 8), generator=g, dtype=torch.float64) * 0.05
                box[l, b, qs, 8:] = torch.randn((k, 2), generator=g, dtype=torch.float64)
                cls[l, b, qs, lab[:k]] = torch.rand((k,), generator=g, dtype=torch.float64) * 4 + 8
        gts.append(gt)
        labels.append(lab)
    return _bf16_grid(cls), _bf16_grid(box), gts, labels
