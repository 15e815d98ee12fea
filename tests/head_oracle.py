"""Float64 restatements of BEVFormerHead's branch tail and NMSFreeCoder.decode, the yardsticks of the detection-head
kernels (tests/test_det_head_gpu.py, tests/test_nms_decode_gpu.py).

``branches_fp64`` restates bevformer_head.py:172-203 (mmdet's inverse_sigmoid, eps 1e-5) and gives per-element bars
for bevf_det_branches_forward: one storage ulp of error at each point where the kernel rounds (each Linear /
LayerNorm output, fp32 weights, the result), propagated through the network as independent errors.

``decode_fp64`` restates nms_free_coder.py:40-121 and util.py:26-53 per sample, with the candidates ordered by
(score descending, flat index ascending).
"""
from __future__ import annotations

import torch

UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}   # one ulp relative, upper bound


def inverse_sigmoid(x, eps=1e-5):
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


def _layers(table):
    """(cls layers, reg layers) of one level's 16-tensor table (ops.det_branch_params order) in float64."""
    t = [p.detach().double().cpu() for p in table]
    cls = [("lin", t[0], t[1]), ("ln", t[2], t[3]), ("relu",), ("lin", t[4], t[5]), ("ln", t[6], t[7]), ("relu",),
           ("lin", t[8], t[9])]
    reg = [("lin", t[10], t[11]), ("relu",), ("lin", t[12], t[13]), ("relu",), ("lin", t[14], t[15])]
    return cls, reg


def _mlp(x, layers, dtype, eps, with_err, weights_rounded):
    """x (rows, 256) float64.  Returns (y, var): var is the variance model of |y - y_kernel| (None unless
    with_err): each rounding to ``dtype`` adds an error of at most one ulp, u |value|, independent of the others,
    and the errors propagate linearly (squared weights) through the Linear and LayerNorm layers."""
    u = UNIT_ROUNDOFF.get(dtype, 0.0)
    var = torch.zeros_like(x) if with_err else None
    last = len(layers) - 1
    for i, layer in enumerate(layers):
        if layer[0] == "lin":
            w = layer[1]
            z = x @ w.t() + layer[2]
            if with_err:
                var = var @ (w * w).t() + (256 * 2.0 ** -24) ** 2 * (x.abs() @ w.abs().t()) ** 2
                if weights_rounded:           # fp32 weights and biases rounded to the storage type in the kernel
                    var = var + (u * u) * ((x * x) @ (w * w).t()) + (u * layer[2]) ** 2
                var = var + (u * z) ** 2      # the layer's output rounding (the last one: rounding of the result)
            x = z
        elif layer[0] == "ln":
            mean = x.mean(-1, keepdim=True)
            rstd = 1 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
            y = (x - mean) * rstd * layer[1] + layer[2]
            if with_err:
                var = 2 * (rstd * layer[1]) ** 2 * (var + var.mean(-1, keepdim=True)) + (u * y) ** 2
            x = y
        else:
            x = x.clamp(min=0)
    return x, var


def branches_fp64(hs, init_reference, inter_references, tables, pc_range, eps=1e-5, dtype=None, with_err=False,
                  sigmas=6.0):
    """hs (L, nq, bs, 256); tables: L lists of ops.det_branch_params.  Returns (cls (L, bs, nq, ncls),
    box (L, bs, nq, 10)) in float64 on the CPU, and with ``with_err`` per-element bars for a kernel that stores in
    ``dtype``: ``sigmas`` standard deviations of the rounding-error model of ``_mlp``."""
    hs = hs.detach().double().cpu().permute(0, 2, 1, 3)
    L, bs, nq, C = hs.shape
    pc = [float(v) for v in pc_range]
    outs = ([], [], [], [])
    for lvl in range(L):
        ref = (init_reference if lvl == 0 else inter_references[lvl - 1]).detach().double().cpu()
        cls_l, reg_l = _layers(tables[lvl])
        rounded = tables[lvl][0].dtype == torch.float32
        x = hs[lvl].reshape(bs * nq, C)
        cls, vcls = _mlp(x, cls_l, dtype, eps, with_err, rounded)
        tmp, vbox = _mlp(x, reg_l, dtype, eps, with_err, rounded)
        inv = inverse_sigmoid(ref.reshape(bs * nq, 3))
        tmp = tmp.clone()
        u = UNIT_ROUNDOFF.get(dtype, 0.0)
        for col, c in ((0, 0), (1, 1), (4, 2)):
            pre = tmp[:, col] + inv[:, c]
            tmp[:, col] = torch.sigmoid(pre) * (pc[c + 3] - pc[c]) + pc[c]
            if with_err:                      # through the sigmoid and the scale, then one rounding of the result
                d = torch.sigmoid(pre) * (1 - torch.sigmoid(pre)) * abs(pc[c + 3] - pc[c])
                vbox[:, col] = d ** 2 * vbox[:, col] + (u * tmp[:, col]) ** 2
        outs[0].append(cls.reshape(bs, nq, -1))
        outs[1].append(tmp.reshape(bs, nq, -1))
        if with_err:
            for k, v, y in ((2, vcls, cls), (3, vbox, tmp)):
                outs[k].append((sigmas * v.sqrt() + 2.0 ** -20 * (1 + y.abs())).reshape(bs, nq, -1))
    res = (torch.stack(outs[0]), torch.stack(outs[1]))
    return res + ((torch.stack(outs[2]), torch.stack(outs[3])) if with_err else ())


def denormalize_bbox(b):
    rot = torch.atan2(b[..., 6:7], b[..., 7:8])
    return torch.cat([b[..., 0:1], b[..., 1:2], b[..., 4:5], b[..., 2:3].exp(), b[..., 3:4].exp(), b[..., 5:6].exp(),
                      rot, b[..., 8:9], b[..., 9:10]], dim=-1)


def decode_fp64(cls_logits, bbox_preds, max_num, post_center_range, score_threshold=None, z_shift=False,
                scores=None):
    """NMSFreeCoder.decode_single per sample in float64 (CPU).  cls_logits (bs, nq, ncls), bbox_preds (bs, nq, 10).
    ``scores``: use these (bs, nq * ncls) scores instead of the float64 sigmoid (to decode from the device's
    fp32 scores).  Returns a list of dicts (bboxes, scores, labels, index) with the candidates in (score descending,
    flat index ascending) order."""
    res = []
    bs, nq, ncls = cls_logits.shape
    for i in range(bs):
        s = (torch.sigmoid(cls_logits[i].double().cpu().reshape(-1)) if scores is None
             else scores[i].double().cpu().reshape(-1))
        order = torch.sort(s, descending=True, stable=True).indices[:max_num]
        sc = s[order]
        labels = order % ncls
        boxes = denormalize_bbox(bbox_preds[i].double().cpu()[order // ncls])
        if score_threshold is not None:
            thresh_mask = sc > score_threshold
            tmp = score_threshold
            while thresh_mask.sum() == 0:
                tmp *= 0.9
                if tmp < 0.01:
                    thresh_mask = sc > -1
                    break
                thresh_mask = sc >= tmp
        pcr = torch.tensor(post_center_range, dtype=torch.float64)
        mask = (boxes[..., :3] >= pcr[:3]).all(1) & (boxes[..., :3] <= pcr[3:]).all(1)
        if score_threshold:
            mask &= thresh_mask
        boxes = boxes[mask]
        if z_shift:
            boxes[:, 2] = boxes[:, 2] - boxes[:, 5] * 0.5
        res.append(dict(bboxes=boxes, scores=sc[mask], labels=labels[mask], index=order[mask]))
    return res


# ---- the toy head case shared by tests/golden/make_golden_head.py and the tests that read its goldens -------------
PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
POST_CENTER_RANGE = [-61.2, -61.2, -10.0, 61.2, 61.2, 10.0]
HEAD_L, HEAD_NQ, HEAD_BS, HEAD_NCLS = 3, 30, 2, 10


def branch_state(refine, L=HEAD_L, ncls=HEAD_NCLS, seed=0):
    """Seeded ``cls_branches.*`` / ``reg_branches.*`` entries under BEVFormerHead's names (num_reg_fcs 2); without box
    refinement every level holds the same values, as the shared module does."""
    g = torch.Generator().manual_seed(41000 + seed)

    def lin(o, i):
        return (torch.rand(o, i, generator=g) * 2 - 1) / 16, torch.rand(o, generator=g) - 0.5

    sd, cls, reg = {}, {}, {}
    for lvl in range(L):
        if refine or lvl == 0:
            cls, reg = {}, {}
            for i, o in ((0, 256), (3, 256), (6, ncls)):
                cls[f"{i}.weight"], cls[f"{i}.bias"] = lin(o, 256)
            for i in (1, 4):
                cls[f"{i}.weight"] = 1 + 0.2 * torch.randn(256, generator=g)
                cls[f"{i}.bias"] = 0.2 * torch.randn(256, generator=g)
            for i, o in ((0, 256), (2, 256), (4, 10)):
                reg[f"{i}.weight"], reg[f"{i}.bias"] = lin(o, 256)
        sd.update({f"cls_branches.{lvl}.{k}": v.clone() for k, v in cls.items()})
        sd.update({f"reg_branches.{lvl}.{k}": v.clone() for k, v in reg.items()})
    return sd


def head_case_inputs(seed=0):
    """Decoder outputs of the toy head case: hs (L, nq, bs, 256), init_reference (bs, nq, 3), inter_references
    (L, bs, nq, 3) in float64, with reference points at the inverse-sigmoid clamps (0, 1, within 1e-5 of either)."""
    g = torch.Generator().manual_seed(42000 + seed)
    hs = torch.randn(HEAD_L, HEAD_NQ, HEAD_BS, 256, generator=g, dtype=torch.float64)
    ref0 = torch.rand(HEAD_BS, HEAD_NQ, 3, generator=g, dtype=torch.float64)
    refs = torch.rand(HEAD_L, HEAD_BS, HEAD_NQ, 3, generator=g, dtype=torch.float64)
    edge = torch.tensor([0.0, 1.0, 5e-6, 1 - 5e-6, 1e-5, 1 - 1e-5], dtype=torch.float64)
    ref0.view(-1)[:12] = edge.repeat(2)
    refs.view(-1)[:12] = edge.flip(0).repeat(2)
    return hs, ref0, refs


def branch_tables(state, L=HEAD_L):
    """The per-level 16-tensor tables (ops.det_branch_params order) of a ``branch_state`` dict."""
    out = []
    for lvl in range(L):
        c, r = f"cls_branches.{lvl}.", f"reg_branches.{lvl}."
        names = [c + n for n in ("0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias", "4.weight",
                                 "4.bias", "6.weight", "6.bias")]
        names += [r + n for n in ("0.weight", "0.bias", "2.weight", "2.bias", "4.weight", "4.bias")]
        out.append([state[n] for n in names])
    return out


# the coder cases of tests/golden/ref_nms_decode_<name>.npz: (score_threshold, logit shift, box scale)
NMS_CASES = {
    "decay": (0.97, 0.0, 40.0),          # top score ~0.9: the decay loop runs and stops at 0.97 * 0.9^k
    "fallthrough": (0.5, -10.0, 40.0),   # every score < 0.01: the loop falls through to > -1
    "zero": (0.0, 0.0, 40.0),            # a threshold of 0.0 is falsy: no threshold mask
    "none": (None, 0.0, 60.0),           # no threshold; many centres outside post_center_range
}


def nms_case_inputs(name, seed=0):
    """(cls logits (2, 300, 10), normalised boxes (2, 300, 10)) of a coder case, float64."""
    _, shift, box_scale = NMS_CASES[name]
    g = torch.Generator().manual_seed(43000 + seed + sum(map(ord, name)))
    cls = 1.0 * torch.randn(2, 300, 10, generator=g, dtype=torch.float64) - 2.0 + shift
    box = torch.randn(2, 300, 10, generator=g, dtype=torch.float64)
    box[..., 0:2] *= box_scale
    box[..., 4] *= 6.0
    return cls, box
