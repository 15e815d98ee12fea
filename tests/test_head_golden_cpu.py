"""The head and coder against what the reference's own BEVFormerHead / NMSFreeCoder returned
(tests/golden/head_toy.npz, head_keys.npz, ref_nms_decode_*.npz; tests/golden/make_golden_head.py), on the CPU: the
float64 restatements of tests/head_oracle.py -- the yardsticks of the GPU tests --, the head's module path, its
gradients, and the parameter names of the head built from the configs' own pts_bbox_head dicts."""
import copy
import json

import numpy as np
import pytest
import torch

from bevformer_b200 import synthetic as syn
from bevformer_b200.plugin.config import build_head, head_cfg_from_config
from tests import head_oracle as ho
from tests.util import golden

W = syn.WORKLOADS["toy"]


def toy_head(refine, dtype=torch.float64):
    """This package's BEVFormerHead with the golden case's branches (its transformer is not used here)."""
    cfg = dict(type="BEVFormerHead", bev_h=W.bev_h, bev_w=W.bev_w, num_query=ho.HEAD_NQ, num_classes=ho.HEAD_NCLS,
               in_channels=256, with_box_refine=refine,
               transformer=dict(type="PerceptionTransformer", num_feature_levels=len(W.levels), num_cams=W.num_cams,
                                embed_dims=256, encoder=syn.encoder_cfg(W), decoder=copy.deepcopy(syn.DECODER_CFG)),
               bbox_coder=dict(type="NMSFreeCoder", post_center_range=ho.POST_CENTER_RANGE, pc_range=ho.PC_RANGE,
                               max_num=100, num_classes=ho.HEAD_NCLS),
               positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=W.bev_h,
                                        col_num_embed=W.bev_w),
               loss_cls=dict(type="FocalLoss", use_sigmoid=True))
    head = build_head(cfg)
    head.load_state_dict(ho.branch_state(refine), strict=False)
    return head.to(dtype).eval()


@pytest.mark.parametrize("refine", [True, False])
def test_restatement_and_module_path_equal_the_reference_head(refine):
    g = golden("head_toy")
    tag = "refine" if refine else "shared"
    hs, r0, rs = ho.head_case_inputs()
    tables = ho.branch_tables(ho.branch_state(refine))
    cls, box = ho.branches_fp64(hs, r0, rs, tables, ho.PC_RANGE)
    np.testing.assert_allclose(cls.numpy(), g[f"{tag}_fp64_cls"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(box.numpy(), g[f"{tag}_fp64_box"], rtol=1e-12, atol=1e-11)
    head = toy_head(refine)
    with torch.no_grad():
        mc, mb = head._branches_modules(hs, r0, rs)
    np.testing.assert_allclose(mc.numpy(), g[f"{tag}_fp64_cls"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(mb.numpy(), g[f"{tag}_fp64_box"], rtol=1e-12, atol=1e-11)
    head32 = toy_head(refine, torch.float32)
    with torch.no_grad():
        mc, mb = head32._branches_modules(*(t.float() for t in (hs, r0, rs)))
    np.testing.assert_allclose(mc.numpy(), g[f"{tag}_fp32_cls"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(mb.numpy(), g[f"{tag}_fp32_box"], rtol=1e-5, atol=1e-4)


def test_module_path_gradients_equal_the_reference_head():
    g = golden("head_toy")
    hs, r0, rs = ho.head_case_inputs()
    hs.requires_grad_(True)
    head = toy_head(True)
    cls, box = head._branches_modules(hs, r0, rs)
    gen = torch.Generator().manual_seed(44000)
    pc = torch.randn(cls.shape, generator=gen, dtype=torch.float64)
    pb = torch.randn(box.shape, generator=gen, dtype=torch.float64)
    ((cls * pc).sum() + (box * pb).sum()).backward()
    np.testing.assert_allclose(hs.grad.numpy(), g["grad_hs"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(head.cls_branches[0][0].weight.grad.numpy(), g["grad_cls0_w0"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(head.reg_branches[2][4].bias.grad.numpy(), g["grad_reg2_b4"], rtol=1e-10, atol=1e-10)


def _split(g, prefix):
    n = g[f"{prefix}_num"]
    cut = np.cumsum(n)[:-1]
    return [dict(bboxes=b, scores=s, labels=lab) for b, s, lab in
            zip(np.split(g[f"{prefix}_bboxes"], cut), np.split(g[f"{prefix}_scores"], cut),
                np.split(g[f"{prefix}_labels"], cut))]


def _same_decode(got, want):
    assert len(got) == len(want)
    for gd, wd in zip(got, want):
        assert len(gd["scores"]) == len(wd["scores"])
        np.testing.assert_array_equal(gd["labels"].numpy(), wd["labels"])
        np.testing.assert_allclose(gd["scores"].numpy(), wd["scores"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(gd["bboxes"].numpy(), wd["bboxes"], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("refine", [True, False])
def test_decode_restatement_equals_get_bboxes_of_the_reference(refine):
    g = golden("head_toy")
    tag = "refine" if refine else "shared"
    cls = torch.from_numpy(g[f"{tag}_fp64_cls"])
    box = torch.from_numpy(g[f"{tag}_fp64_box"])
    got = ho.decode_fp64(cls[-1], box[-1], 100, ho.POST_CENTER_RANGE, None, z_shift=True)
    _same_decode(got, _split(g, f"{tag}_fp64_dec"))


@pytest.mark.parametrize("case", sorted(ho.NMS_CASES))
def test_decode_restatement_equals_the_reference_coder(case):
    """Every threshold branch of the reference's loop (decay, fall-through to > -1, the falsy 0.0, none) and boxes
    outside post_center_range."""
    g = golden(f"ref_nms_decode_{case}")
    cls, box = ho.nms_case_inputs(case)
    got = ho.decode_fp64(cls, box, 100, ho.POST_CENTER_RANGE, ho.NMS_CASES[case][0])
    _same_decode(got, _split(g, "fp64"))


@pytest.mark.parametrize("name", ["tiny", "small", "base", "v2"])
def test_build_head_from_config_has_the_reference_keys(name):
    """The head built from the config's own pts_bbox_head dict (stored in the golden with the keys the reference
    head had when built from the same file)."""
    g = golden("head_keys")
    head_cfg = json.loads(str(g[f"{name}_pts_bbox_head"]))
    head = build_head(head_cfg_from_config({"model": {"pts_bbox_head": head_cfg}}))
    assert sorted(head.state_dict()) == list(g[name]), str(g[f"{name}_config"])
