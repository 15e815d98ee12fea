"""BEVFormerHead / NMSFreeCoder / LearnedPositionalEncoding on the host: registration under the config type names,
construction (parameter names, initialisation, GroupDETR query count), and the refusals -- no GPU needed."""
import copy
import math

import numpy as np
import pytest
import torch

from bevformer_b200 import synthetic as syn
from bevformer_b200.plugin import (BBOX_CODERS, HEADS, POSITIONAL_ENCODING, BEVFormerHead, BEVFormerHead_GroupDETR,
                                   LearnedPositionalEncoding, NMSFreeCoder, PerceptionTransformer)
from bevformer_b200.plugin.config import build_head
from tests.util import golden

W = syn.WORKLOADS["toy"]
PC = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def head_cfg(**kw):
    cfg = dict(type="BEVFormerHead", bev_h=W.bev_h, bev_w=W.bev_w, num_query=100, num_classes=10, in_channels=256,
               sync_cls_avg_factor=True, with_box_refine=True, as_two_stage=False,
               transformer=dict(type="PerceptionTransformer", num_feature_levels=len(W.levels), num_cams=W.num_cams,
                                embed_dims=256, rotate_center=[W.bev_h // 2, W.bev_w // 2],
                                encoder=syn.encoder_cfg(W), decoder=copy.deepcopy(syn.DECODER_CFG)),
               bbox_coder=dict(type="NMSFreeCoder", post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
                               pc_range=PC, max_num=300, num_classes=10),
               positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=W.bev_h,
                                        col_num_embed=W.bev_w),
               loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
               loss_bbox=dict(type="L1Loss", loss_weight=0.25), loss_iou=dict(type="GIoULoss", loss_weight=0.0))
    cfg.update(kw)
    return cfg


def test_registries_resolve_the_config_type_names():
    assert HEADS.get("BEVFormerHead") is BEVFormerHead
    assert HEADS.get("BEVFormerHead_GroupDETR") is BEVFormerHead_GroupDETR
    assert BBOX_CODERS.get("NMSFreeCoder") is NMSFreeCoder
    assert POSITIONAL_ENCODING.get("LearnedPositionalEncoding") is LearnedPositionalEncoding
    from projects.mmdet3d_plugin.bevformer.dense_heads import BEVFormerHead as H
    from projects.mmdet3d_plugin.core.bbox.coders import NMSFreeCoder as C
    assert H is BEVFormerHead and C is NMSFreeCoder


@pytest.mark.parametrize("refine", [True, False])
def test_parameter_names_are_the_reference_heads(refine):
    """bevformer_head.py:69-107 and mmdet's DETRHead: the transformer's names under ``transformer.``, the branches
    (cloned with box refinement, one shared module otherwise -- still listed per level), the embeddings, the
    positional-encoding tables and the frozen code_weights."""
    head = build_head(head_cfg(with_box_refine=refine))
    keys = set(head.state_dict())
    pt = PerceptionTransformer(num_feature_levels=len(W.levels), num_cams=W.num_cams, encoder=syn.encoder_cfg(W),
                               decoder=copy.deepcopy(syn.DECODER_CFG), embed_dims=256)
    want = {"transformer." + k for k in pt.state_dict()}
    want |= {"code_weights", "bev_embedding.weight", "query_embedding.weight", "positional_encoding.row_embed.weight",
             "positional_encoding.col_embed.weight"}
    for lvl in range(syn.DECODER_CFG["num_layers"]):
        want |= {f"cls_branches.{lvl}.{i}.{p}" for i in (0, 1, 3, 4, 6) for p in ("weight", "bias")}
        want |= {f"reg_branches.{lvl}.{i}.{p}" for i in (0, 2, 4) for p in ("weight", "bias")}
    assert keys == want
    # the transformer part is the reference PerceptionTransformer's (key list of the reference class, committed)
    g = golden("perception_forward_toy")
    assert sorted(k[len("transformer."):] for k in keys if k.startswith("transformer.")) == list(g["keys"])
    assert (head.cls_branches[0] is head.cls_branches[1]) == (not refine)
    assert head.query_embedding.weight.shape == (100, 512) and head.bev_embedding.weight.shape == (W.num_query, 256)


def test_init_weights_sets_the_focal_prior_and_code_weights():
    head = build_head(head_cfg())
    head.init_weights()
    bias = -math.log((1 - 0.01) / 0.01)
    for m in head.cls_branches:
        assert torch.allclose(m[-1].bias, torch.full((10,), bias))
    assert head.code_weights.tolist() == pytest.approx([1.0] * 8 + [0.2, 0.2])
    assert not head.code_weights.requires_grad and head.cls_out_channels == 10
    ce = build_head(head_cfg(loss_cls=dict(type="CrossEntropyLoss", use_sigmoid=False), code_weights=[2.0] * 10))
    assert ce.cls_out_channels == 11 and ce.code_weights.tolist() == [2.0] * 10


def test_group_detr_queries():
    head = build_head(head_cfg(type="BEVFormerHead_GroupDETR", group_detr=3))
    assert head.num_query == 300 and head.query_embedding.weight.shape == (300, 512)
    assert head.train()._object_query_embeds(torch.float32).shape == (300, 512)
    assert head.eval()._object_query_embeds(torch.float32).shape == (100, 512)


def test_learned_positional_encoding():
    pe = LearnedPositionalEncoding(4, row_num_embed=3, col_num_embed=5)
    pos = pe(torch.zeros(2, 3, 5))
    assert pos.shape == (2, 8, 3, 5)
    for i in range(3):
        for j in range(5):
            assert torch.equal(pos[1, :, i, j], torch.cat([pe.col_embed.weight[j], pe.row_embed.weight[i]]))
    pe.init_weights()
    assert 0 <= pe.row_embed.weight.min() and pe.row_embed.weight.max() <= 1


def test_refusals():
    with pytest.raises(NotImplementedError, match="two_stage"):
        build_head(head_cfg(as_two_stage=True))
    coder = NMSFreeCoder(pc_range=PC, post_center_range=None)
    preds = dict(all_cls_scores=torch.zeros(1, 1, 5, 10), all_bbox_preds=torch.zeros(1, 1, 5, 10))
    with pytest.raises(NotImplementedError):
        coder.decode(preds)
    with pytest.raises(RuntimeError, match="CUDA"):
        NMSFreeCoder(pc_range=PC, post_center_range=[0] * 6, max_num=5).decode(preds)


def test_fp64_decode_restatement_threshold_quirks():
    """The restatement the GPU tests measure against keeps the reference's quirks: a 0.0 threshold applies no mask,
    the decay loop stops at the first threshold the top score passes, below 0.01 everything passes."""
    from tests import head_oracle as ho
    logits = torch.tensor([[[2.0, -1.0], [0.0, -3.0]]], dtype=torch.float64)   # scores .881 .269 .5 .047
    box = torch.zeros(1, 2, 10, dtype=torch.float64)
    box[..., 7] = 1.0
    pcr = [-1.0] * 3 + [1.0] * 3
    n = lambda thr: len(ho.decode_fp64(logits, box, 4, pcr, thr)[0]["scores"])   # noqa: E731
    assert n(None) == 4 and n(0.0) == 4 and n(0.4) == 2 and n(0.95) == 1 and n(-0.5) == 4
    assert len(ho.decode_fp64(logits - 10, box, 4, pcr, 0.5)[0]["scores"]) == 4       # falls through to > -1
    order = ho.decode_fp64(logits, box, 4, pcr)[0]["index"].tolist()
    assert order == [0, 2, 1, 3] and np.isclose(ho.decode_fp64(logits, box, 1, pcr)[0]["scores"][0].item(),
                                                1 / (1 + math.exp(-2.0)))
