"""BEVFormerHead's training loss on the host: the float64 restatement (tests/det_loss_oracle.py) against the reference's
own loss (tests/golden/ref_det_loss_*.npz), the heads of the shipped configs reading their assigner and loss settings,
the refusals, and the avg-factor reduction across 2 gloo ranks -- no GPU needed."""
import copy
import json
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from bevformer_b200.plugin import head as head_mod
from bevformer_b200.plugin.config import build_head
from tests import det_loss_oracle as dlo
from tests.util import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def case_data(name):
    L, bs, groups, nqg, ncls, n_gt, settings, nan_frac = dlo.CASES[name]
    cls, box, gts, labels = dlo.case_inputs(L, bs, groups, nqg, ncls, n_gt, nan_frac, dlo.case_seed(name))
    st = dlo.BASE if settings == "base" else dlo.V2
    return cls, box, gts, labels, st, groups


def golden_assignment(g, L, bs, nq, groups):
    a = g["assign"]
    nqg = nq // groups
    out = []
    for l in range(L):
        per_g = []
        for grp in range(groups):
            per_b = []
            for b in range(bs):
                row = a[l * bs + b, grp * nqg:(grp + 1) * nqg]
                rows = np.nonzero(row >= 0)[0]
                per_b.append((rows, row[rows].astype(np.int64)))
            per_g.append(per_b)
        out.append(per_g)
    return out


@pytest.mark.parametrize("name", sorted(dlo.CASES))
def test_restatement_equals_the_reference_loss(name):
    """Loss dict, assignment and gradients of the float64 restatement against the reference's loss in float64:
    the isnotnan drop of NaN-velocity targets, the empty sample and the GroupDETR sum included."""
    g = golden(f"ref_det_loss_{name}")
    cls, box, gts, labels, st, groups = case_data(name)
    L, bs, nq, _ = cls.shape
    cls, box = cls.clone().requires_grad_(True), box.clone().requires_grad_(True)
    losses, assignment = dlo.loss(cls, box, gts, labels, st, groups)
    assert (dlo.assignment_array(assignment, L, bs, nq, groups) == g["assign"]).all()
    want_keys = {"loss_cls", "loss_bbox"} | {f"d{i}.loss_{k}" for i in range(L - 1) for k in ("cls", "bbox")}
    assert set(losses) == want_keys
    for k, v in losses.items():
        ref = float(g[f"fp64_{k}"])
        assert abs(v.item() - ref) <= 1e-12 * max(1.0, abs(ref)), (k, v.item(), ref)
    sum(losses.values()).backward()
    rows = g["grad_rows"]
    for t, key in ((cls, "cls"), (box, "box")):
        got = t.grad.reshape(-1, t.shape[-1])[rows].numpy()
        ref = g[f"fp64_grad_{key}"]
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    if name == "nanvel":                       # positives with a NaN velocity: no regression term, still counted
        assert float(g["fp64_loss_bbox"]) > 0
        nan_gt = [torch.nonzero(~torch.isfinite(gt).all(-1)).flatten().tolist() for gt in gts]
        a = g["assign"]
        for p in range(L * bs):
            dropped = np.isin(a[p], nan_gt[p % bs]) & (a[p] >= 0)
            assert dropped.any()
            flat = p * nq + np.nonzero(dropped)[0]
            sel = np.isin(rows, flat)
            assert sel.any() and (g["fp64_grad_box"][sel] == 0).all()
    if name == "base":                         # the sample without ground truth is all background
        assert (g["assign"][1::2] == -1).all()


def _config_head(name, **train_cfg_changes):
    g = golden("ref_det_loss_tiny")
    hcfg = json.loads(str(g[f"{name}_pts_bbox_head"]))
    tcfg = json.loads(str(g[f"{name}_train_cfg"]))
    for k, v in train_cfg_changes.items():
        tcfg["assigner"][k] = v
    hcfg["train_cfg"] = tcfg
    return build_head(hcfg), hcfg


@pytest.mark.parametrize("name", ["tiny", "base", "v2"])
def test_config_heads_read_their_loss_settings(name):
    head, hcfg = _config_head(name)
    assert callable(head.loss)
    st = head_mod._loss_settings(head)
    want = dlo.V2 if name == "v2" else dlo.BASE
    assert st == want
    assert (type(head).__name__ == "BEVFormerHead_GroupDETR") == (name == "v2")
    if name == "v2":
        assert head.group_detr == 11 and head.num_query == 11 * 900


@pytest.mark.parametrize("change, err, match", [
    (dict(cls_cost=dict(type="ClassificationCost", weight=2.0)), NotImplementedError, "FocalLossCost"),
    (dict(reg_cost=dict(type="BBoxL1Cost", weight=0.25)), NotImplementedError, "reg_cost"),
    (dict(cls_cost=dict(type="FocalLossCost", weight=1.0)), ValueError, "classification weight"),
    (dict(reg_cost=dict(type="BBox3DL1Cost", weight=0.5)), ValueError, "regression weight"),
])
def test_loss_refuses_unsupported_or_inconsistent_assigners(change, err, match):
    head, _ = _config_head("tiny", **change)
    with pytest.raises(err, match=match):
        head_mod._loss_settings(head)


@pytest.mark.parametrize("field, value, match", [
    ("loss_cls", dict(type="CrossEntropyLoss", use_sigmoid=False, loss_weight=2.0), "loss_cls"),
    ("loss_bbox", dict(type="GIoULoss", loss_weight=0.25), "loss_bbox"),
])
def test_loss_refuses_unsupported_losses(field, value, match):
    _, hcfg = _config_head("tiny")
    hcfg = copy.deepcopy(hcfg)
    hcfg[field] = value
    head = build_head(hcfg)
    with pytest.raises(NotImplementedError, match=match):
        head_mod._loss_settings(head)


def test_loss_needs_an_assigner_but_construction_does_not():
    g = golden("ref_det_loss_tiny")
    hcfg = json.loads(str(g["tiny_pts_bbox_head"]))
    head = build_head(copy.deepcopy(hcfg))              # no train_cfg: builds, as before
    assert head.train_cfg is None
    with pytest.raises(RuntimeError, match="assigner"):
        head_mod._loss_settings(head)
    hcfg["train_cfg"] = dict(grid_size=[512, 512, 1])
    with pytest.raises(RuntimeError, match="assigner"):
        head_mod._loss_settings(build_head(hcfg))


def test_ground_truth_formats():
    t = torch.tensor([[1.0, 2.0, -1.0, 2.0, 4.0, 1.5, 0.3, 0.1, -0.2]])
    got = head_mod.gravity_center_boxes(t)
    assert torch.equal(got, torch.tensor([[1.0, 2.0, -0.25, 2.0, 4.0, 1.5, 0.3, 0.1, -0.2]]))

    class Boxes:                                 # LiDARInstance3DBoxes' two attributes
        gravity_center = got[:, :3]
        tensor = t
    assert torch.equal(head_mod.gravity_center_boxes(Boxes()), got)
    with pytest.raises(ValueError, match="columns"):
        head_mod.gravity_center_boxes(t[:, :7])
    with pytest.raises(TypeError):
        head_mod.gravity_center_boxes([1, 2, 3])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _avg_worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from bevformer_b200.plugin import head as hm
    calls = []
    real = dist.all_reduce

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)
    dist.all_reduce = counting
    counts = [10.0 + 7 * rank, 3.0 * rank]                      # two groups, different per rank
    synced = hm.avg_factors(counts, 3, torch.device("cpu"), True)
    n_synced = len(calls)
    local = hm.avg_factors(counts, 3, torch.device("cpu"), False)
    out[rank] = (synced.tolist(), local.tolist(), n_synced, len(calls) - n_synced)
    dist.destroy_process_group()


def test_avg_factors_are_one_all_reduce_mean_across_ranks():
    world = 2
    out = mp.Manager().dict()
    mp.spawn(_avg_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    mean = [(10.0 + 17.0) / 2, 3.0 / 2]
    for rank in range(world):
        synced, local, n1, n2 = out[rank]
        assert n1 == 1 and n2 == 1
        assert synced == [[mean[i % 2]] * 2 for i in range(6)]
        mine = [10.0 + 7 * rank, 3.0 * rank]
        assert local == [[mine[i % 2], mean[i % 2]] for i in range(6)]
