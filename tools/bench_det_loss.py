"""Times one BEVFormerHead loss call (forward + backward of the loss, not of the head) on the library against the
reference's arithmetic restated in torch on the same GPU: per (layer, group, sample) a cost matrix copied to the
host for scipy, and a ``.item()`` per loss slot.  Prints one JSON line per shape with the time per call (CUDA events
around calls that end in a synchronise), scipy's share (host timer around every linear_sum_assignment call; both
paths run the same solver on the same matrices), the host synchronisations counted under
torch.cuda.set_sync_debug_mode('warn'), the device-to-host bytes from the shapes, and the card's name and power limit.

    python tools/bench_det_loss.py [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bevformer_b200.plugin import head as head_mod  # noqa: E402
from tests import det_loss_oracle as dlo  # noqa: E402

DEV = torch.device("cuda")
SHAPES = {  # name: (layers, bs, groups, queries per group, n_gt per sample, settings)
    "base_ngt40": (6, 1, 1, 900, (40,), dlo.BASE),
    "base_ngt150": (6, 1, 1, 900, (150,), dlo.BASE),
    "v2_ngt40": (6, 1, 11, 900, (40,), dlo.V2),
}
SCIPY_S = [0.0]


def _timed_lsa():
    from scipy.optimize import linear_sum_assignment

    def lsa(cost):
        t = time.perf_counter()
        out = linear_sum_assignment(cost)
        SCIPY_S[0] += time.perf_counter() - t
        return out
    return lsa


def _inputs(L, bs, groups, nqg, n_gt, seed=0):
    cls, box, gts, labels = dlo.case_inputs(L, bs, groups, nqg, 10, n_gt, 0.1, seed)
    c = cls.float().to(DEV).requires_grad_(True)
    b = box.float().to(DEV).requires_grad_(True)
    return c, b, [g.float().to(DEV) for g in gts], [lab.to(DEV) for lab in labels]


class _Boxes:
    """LiDARInstance3DBoxes' two attributes the library's loss reads, for gravity-centred (n, 9) boxes."""

    def __init__(self, g):
        self.gravity_center = g[:, :3]
        self.tensor = torch.cat((g[:, :2], g[:, 2:3] - g[:, 5:6] * 0.5, g[:, 3:]), 1)


def _loss_state(st):
    """The head state ``BEVFormerHead._loss`` reads, built once outside the timed calls."""
    reg = {"l1": "BBox3DL1Cost", "smooth_l1": "SmoothL1Cost"}[st["cost_reg_kind"]]
    import types
    return types.SimpleNamespace(
        train_cfg=dict(assigner=dict(cls_cost=dict(type="FocalLossCost", weight=st["cls_cost_weight"]),
                                     reg_cost=dict(type=reg, weight=st["reg_cost_weight"]))),
        loss_cls=head_mod._loss_cfg(dict(type="FocalLoss", loss_weight=st["cls_loss_weight"])),
        loss_bbox=head_mod._loss_cfg(dict(type="L1Loss" if st["reg_kind"] == "l1" else "SmoothL1Loss",
                                          loss_weight=st["bbox_loss_weight"])),
        sync_cls_avg_factor=True, code_weights=torch.tensor(dlo.CODE_WEIGHTS, device=DEV))


def library_call(head, groups, c, b, boxes, labels):
    preds = dict(all_cls_scores=c, all_bbox_preds=b, enc_cls_scores=None, enc_bbox_preds=None)
    losses = head_mod.BEVFormerHead._loss(head, boxes, labels, preds, None, groups)
    sum(losses.values()).backward()


def reference_call(st, groups, c, b, gts, labels):
    """The reference's flow in torch: per-slot cost.cpu() + scipy, per-slot .item() of the regression avg factor."""
    L, bs, nq, _ = c.shape
    nqg = nq // groups
    lsa = _timed_lsa()
    count = float(sum(min(g.shape[0], nqg) for g in gts))
    total = 0
    for grp in range(groups):
        for l in range(L):
            rc = []
            for s in range(bs):
                if gts[s].shape[0] == 0:
                    rc.append(([], []))
                    continue
                cost = dlo.match_cost(c[l, s, grp * nqg:(grp + 1) * nqg].detach(),
                                      b[l, s, grp * nqg:(grp + 1) * nqg].detach(), gts[s], labels[s], st)
                rc.append(lsa(cost.cpu()))
            avg = torch.clamp(c.new_tensor([count]), min=1).item()
            lc, lb = dlo.slot_loss(c[l, :, grp * nqg:(grp + 1) * nqg], b[l, :, grp * nqg:(grp + 1) * nqg], gts,
                                   labels, rc, st, dlo.CODE_WEIGHTS, count, avg)
            total = total + (lc + lb) / groups
    total.backward()


def _syncs(fn, *args):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            fn(*args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in rec)


def _time(fn, args, iters, warmup):
    for _ in range(warmup):
        fn(*args)
    torch.cuda.synchronize()
    SCIPY_S[0] = 0.0
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn(*args)
        torch.cuda.synchronize()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters, SCIPY_S[0] * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det_loss: needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    head_mod._linear_sum_assignment = _timed_lsa
    for name, (L, bs, groups, nqg, n_gt, st) in SHAPES.items():
        c, b, gts, labels = _inputs(L, bs, groups, nqg, n_gt)
        args = (st, groups, c, b, gts, labels)
        lib_args = (_loss_state(st), groups, c, b, [_Boxes(g) for g in gts], labels)
        lib_ms, lib_scipy = _time(library_call, lib_args, a.iters, a.warmup)
        ref_ms, ref_scipy = _time(reference_call, args, a.iters, a.warmup)
        nq = groups * nqg
        slots = L * groups * sum(1 for n in n_gt if n)
        print(json.dumps(dict(
            shape=name, layers=L, bs=bs, groups=groups, queries_per_group=nqg, n_gt=list(n_gt),
            library_ms=round(lib_ms, 3), library_scipy_ms=round(lib_scipy, 3),
            library_syncs=_syncs(library_call, *lib_args), library_d2h_bytes=L * bs * nq * max(n_gt) * 4,
            reference_ms=round(ref_ms, 3), reference_scipy_ms=round(ref_scipy, 3),
            reference_syncs=_syncs(reference_call, *args),
            reference_d2h_bytes=L * groups * sum(nqg * n * 4 for n in n_gt) + 4 * L * groups,
            reference_slots_with_gt=slots, gpu=q[0] if q else "unknown")), flush=True)


if __name__ == "__main__":
    main()
