"""Generates the detection-head goldens from the REFERENCE'S OWN BEVFormerHead / BEVFormerHead_GroupDETR
(dense_heads/bevformer_head.py), NMSFreeCoder (core/bbox/coders/nms_free_coder.py) and denormalize_bbox
(core/bbox/util.py), imported unmodified behind oracle/mmcv_stub.py plus the third-party pieces those files import,
restated below.  Needs a reference checkout (BEVF_REFERENCE_ROOT); the test suite does not:

    python tests/golden/make_golden_head.py

Writes
  head_toy.npz               the head's forward (all_cls_scores, all_bbox_preds) on the toy decoder outputs of
                             tests/head_oracle.py (head_case_inputs / branch_state), fp64 and fp32, with and without
                             box refinement, bs 2; get_bboxes of those outputs; gradients of a fixed projection of the
                             fp64 outputs (box refinement) with respect to the decoder states and two branch tensors
  head_keys.npz              sorted state_dict keys of the head built from bevformer_{tiny,small,base}.py and
                             bevformerv2-r50-t1-24ep.py, with each config's pts_bbox_head dict (JSON)
  ref_nms_decode_<case>.npz  NMSFreeCoder.decode on tests/head_oracle.py's coder cases, fp64 and fp32
"""
from __future__ import annotations

import copy
import functools
import importlib.util
import json
import os
import sys
import types
import warnings

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bevformer_b200.plugin import config  # noqa: E402
from oracle import mmcv_stub  # noqa: E402
from oracle.mmcv_stub import BaseModule, Registry, build_from_cfg  # noqa: E402
from tests import head_oracle as ho  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
PLUGIN = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "mmdet3d_plugin")


# ---- third-party pieces the reference head / coder import, restated --------------------------------------------
def inverse_sigmoid(x, eps=1e-5):
    """mmdet 2.14 mmdet/models/utils/transformer.py:inverse_sigmoid."""
    x = x.clamp(min=0, max=1)
    x1 = x.clamp(min=eps)
    x2 = (1 - x).clamp(min=eps)
    return torch.log(x1 / x2)


def bias_init_with_prob(prior_prob):
    """mmcv 1.4 mmcv/cnn/utils/weight_init.py:bias_init_with_prob."""
    return float(-np.log((1 - prior_prob) / prior_prob))


def multi_apply(func, *args, **kwargs):
    """mmdet 2.14 mmdet/core/utils/misc.py:multi_apply."""
    pfunc = functools.partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def reduce_mean(tensor):
    """mmdet 2.14 mmdet/core/utils/dist_utils.py:reduce_mean, single process."""
    return tensor


class BaseBBoxCoder:
    """mmdet 2.14 mmdet/core/bbox/coder/base_bbox_coder.py (abstract encode / decode)."""

    def __init__(self, **kwargs):
        pass


class LearnedPositionalEncoding(BaseModule):
    """mmdet 2.14 mmdet/models/utils/positional_encoding.py:LearnedPositionalEncoding."""

    def __init__(self, num_feats, row_num_embed=50, col_num_embed=50,
                 init_cfg=dict(type="Uniform", layer="Embedding")):
        super().__init__(init_cfg)
        self.row_embed = nn.Embedding(row_num_embed, num_feats)
        self.col_embed = nn.Embedding(col_num_embed, num_feats)
        self.num_feats = num_feats
        self.row_num_embed = row_num_embed
        self.col_num_embed = col_num_embed

    def forward(self, mask):
        h, w = mask.shape[-2:]
        x = torch.arange(w, device=mask.device)
        y = torch.arange(h, device=mask.device)
        x_embed = self.col_embed(x)
        y_embed = self.row_embed(y)
        pos = torch.cat((x_embed.unsqueeze(0).repeat(h, 1, 1), y_embed.unsqueeze(1).repeat(1, w, 1)),
                        dim=-1).permute(2, 0, 1).unsqueeze(0).repeat(mask.shape[0], 1, 1, 1)
        return pos


class _Loss(nn.Module):
    """A built loss as the head's constructor sees it: mmdet's FocalLoss defaults ``use_sigmoid`` to True, the
    others to False; no parameters."""

    def __init__(self, type=None, use_sigmoid=None, **kwargs):
        super().__init__()
        self.use_sigmoid = (type == "FocalLoss") if use_sigmoid is None else use_sigmoid


HEADS, BBOX_CODERS, TRANSFORMER = Registry("head"), Registry("bbox_coder"), Registry("transformer")
POSITIONAL_ENCODING = mmcv_stub.POSITIONAL_ENCODING


class DETRHead(BaseModule):
    """mmdet 2.14 mmdet/models/dense_heads/detr_head.py:DETRHead.__init__ (the constructor surface BEVFormerHead
    relies on; the assigner / sampler of ``train_cfg`` are not modules and are not built here)."""

    def __init__(self, num_classes, in_channels, num_query=100, num_reg_fcs=2, transformer=None,
                 sync_cls_avg_factor=False,
                 positional_encoding=dict(type="SinePositionalEncoding", num_feats=128, normalize=True),
                 loss_cls=dict(type="CrossEntropyLoss", bg_cls_weight=0.1, use_sigmoid=False, loss_weight=1.0,
                               class_weight=1.0),
                 loss_bbox=dict(type="L1Loss", loss_weight=5.0), loss_iou=dict(type="GIoULoss", loss_weight=2.0),
                 train_cfg=None, test_cfg=dict(max_per_img=100), init_cfg=None, **kwargs):
        super().__init__(init_cfg)
        self.bg_cls_weight = 0
        self.sync_cls_avg_factor = sync_cls_avg_factor
        self.num_query = num_query
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.num_reg_fcs = num_reg_fcs
        self.train_cfg = train_cfg
        self.test_cfg = test_cfg
        self.fp16_enabled = False
        self.loss_cls = _Loss(**loss_cls)
        self.loss_bbox = _Loss(**loss_bbox)
        self.loss_iou = _Loss(**loss_iou)
        self.cls_out_channels = num_classes if self.loss_cls.use_sigmoid else num_classes + 1
        self.act_cfg = transformer.get("act_cfg", dict(type="ReLU", inplace=True))
        self.activate = nn.ReLU(inplace=True)
        self.positional_encoding = build_from_cfg(positional_encoding, POSITIONAL_ENCODING)
        self.transformer = build_from_cfg(transformer, TRANSFORMER)
        self.embed_dims = self.transformer.embed_dims
        assert "num_feats" in positional_encoding
        assert positional_encoding["num_feats"] * 2 == self.embed_dims
        self._init_layers()


class FixedDecoderOutputs(nn.Module):
    """Stands in for the transformer in the toy case: returns given decoder outputs and records what the head
    passed in (the head's arithmetic after the transformer is what the goldens pin)."""

    def __init__(self, outputs=None, num_layers=3, embed_dims=256):
        super().__init__()
        self.outputs = outputs
        self.decoder = types.SimpleNamespace(num_layers=num_layers)
        self.embed_dims = embed_dims
        self.seen = {}

    def init_weights(self):
        pass

    def forward(self, mlvl_feats, bev_queries, object_query_embed, bev_h, bev_w, grid_length=None, bev_pos=None,
                reg_branches=None, cls_branches=None, img_metas=None, prev_bev=None):
        self.seen = dict(bev_pos=bev_pos, object_query_embed=object_query_embed, grid_length=grid_length)
        return self.outputs


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference_head():
    """(BEVFormerHead, BEVFormerHead_GroupDETR, NMSFreeCoder, util module) of the reference, unmodified."""
    mmcv_stub.load_reference_decoder()
    PT = mmcv_stub.load_reference_transformer()
    v2 = mmcv_stub.load_reference_transformer_v2().module
    for cls in (PT, v2.PerceptionTransformerV2, FixedDecoderOutputs):
        TRANSFORMER.register_module(name=cls.__name__, module=cls)
    POSITIONAL_ENCODING.register_module(name="LearnedPositionalEncoding", module=LearnedPositionalEncoding)
    sys.modules["mmcv.cnn"].bias_init_with_prob = bias_init_with_prob
    util = _load("_bevf_ref_bbox_util", os.path.join(PLUGIN, "core", "bbox", "util.py"))
    extra = {
        "mmdet": mmcv_stub._mod("mmdet"),
        "mmdet.core": mmcv_stub._mod("mmdet.core", multi_apply=multi_apply, reduce_mean=reduce_mean),
        "mmdet.core.bbox": mmcv_stub._mod("mmdet.core.bbox", BaseBBoxCoder=BaseBBoxCoder),
        "mmdet.core.bbox.builder": mmcv_stub._mod("mmdet.core.bbox.builder", BBOX_CODERS=BBOX_CODERS),
        "mmdet.models": mmcv_stub._mod("mmdet.models", HEADS=HEADS),
        "mmdet.models.utils": mmcv_stub._mod("mmdet.models.utils"),
        "mmdet.models.utils.transformer": mmcv_stub._mod("mmdet.models.utils.transformer",
                                                         inverse_sigmoid=inverse_sigmoid),
        "mmdet.models.dense_heads": mmcv_stub._mod("mmdet.models.dense_heads", DETRHead=DETRHead),
        "mmdet3d": mmcv_stub._mod("mmdet3d"), "mmdet3d.core": mmcv_stub._mod("mmdet3d.core"),
        "mmdet3d.core.bbox": mmcv_stub._mod("mmdet3d.core.bbox"),
        "mmdet3d.core.bbox.coders": mmcv_stub._mod(
            "mmdet3d.core.bbox.coders", build_bbox_coder=lambda cfg: build_from_cfg(cfg, BBOX_CODERS)),
        "projects.mmdet3d_plugin.core": mmcv_stub._mod("projects.mmdet3d_plugin.core"),
        "projects.mmdet3d_plugin.core.bbox": mmcv_stub._mod("projects.mmdet3d_plugin.core.bbox"),
        "projects.mmdet3d_plugin.core.bbox.util": util,
    }
    saved = {k: sys.modules.get(k) for k in extra}
    sys.modules.update(extra)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            coder = _load("_bevf_ref_nms_free_coder", os.path.join(PLUGIN, "core", "bbox", "coders",
                                                                   "nms_free_coder.py"))
            head = _load("_bevf_ref_bevformer_head", os.path.join(PLUGIN, "bevformer", "dense_heads",
                                                                  "bevformer_head.py"))
    finally:
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    return head.BEVFormerHead, head.BEVFormerHead_GroupDETR, coder.NMSFreeCoder, util


def toy_head_cfg(refine, outputs):
    return dict(num_query=ho.HEAD_NQ, num_classes=ho.HEAD_NCLS, in_channels=256, sync_cls_avg_factor=True,
                with_box_refine=refine, as_two_stage=False, bev_h=4, bev_w=5,
                transformer=dict(type="FixedDecoderOutputs", outputs=outputs, num_layers=ho.HEAD_L),
                bbox_coder=dict(type="NMSFreeCoder", post_center_range=ho.POST_CENTER_RANGE, pc_range=ho.PC_RANGE,
                                max_num=100, num_classes=ho.HEAD_NCLS),
                positional_encoding=dict(type="LearnedPositionalEncoding", num_feats=128, row_num_embed=4,
                                         col_num_embed=5),
                loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
                loss_bbox=dict(type="L1Loss", loss_weight=0.25), loss_iou=dict(type="GIoULoss", loss_weight=0.0))


def _decoded(ret, prefix):
    """get_bboxes' per-sample lists concatenated, with the per-sample counts."""
    return {f"{prefix}_bboxes": np.concatenate([r[0].detach().numpy() for r in ret]),
            f"{prefix}_scores": np.concatenate([r[1].detach().numpy() for r in ret]),
            f"{prefix}_labels": np.concatenate([r[2].numpy() for r in ret]),
            f"{prefix}_num": np.array([len(r[1]) for r in ret])}


def head_toy():
    Head, _, _, _ = load_reference_head()
    hs, ref0, refs = ho.head_case_inputs()
    out = {}
    for refine in (True, False):
        tag = "refine" if refine else "shared"
        for dt, name in ((torch.float64, "fp64"), (torch.float32, "fp32")):
            inputs = [t.to(dt).clone() for t in (hs, ref0, refs)]
            if dt == torch.float64 and refine:
                inputs[0].requires_grad_(True)
            head = Head(**copy.deepcopy(toy_head_cfg(refine, None)))
            state = ho.branch_state(refine)
            missing = set(head.state_dict()) - set(state)
            assert all(not k.startswith(("cls_branches", "reg_branches")) for k in missing)
            head.load_state_dict(state, strict=False)
            head = head.to(dt).eval()
            head.transformer.outputs = (torch.zeros(20, ho.HEAD_BS, 256, dtype=dt), inputs[0], inputs[1], inputs[2])
            feats = [torch.zeros(ho.HEAD_BS, 1, 1, 1, 1, dtype=dt)]
            res = head(feats, None)
            cls, box = res["all_cls_scores"], res["all_bbox_preds"]
            out[f"{tag}_{name}_cls"] = cls.detach().numpy()
            out[f"{tag}_{name}_box"] = box.detach().numpy()
            metas = [dict(box_type_3d=lambda b, code_size: b) for _ in range(ho.HEAD_BS)]
            with torch.no_grad():
                ret = head.get_bboxes({k: (v.detach() if torch.is_tensor(v) else v) for k, v in res.items()}, metas)
            out.update(_decoded(ret, f"{tag}_{name}_dec"))
            if inputs[0].requires_grad:
                g = torch.Generator().manual_seed(44000)
                pc = torch.randn(cls.shape, generator=g, dtype=dt)
                pb = torch.randn(box.shape, generator=g, dtype=dt)
                ((cls * pc).sum() + (box * pb).sum()).backward()
                out["grad_hs"] = inputs[0].grad.numpy()
                out["grad_cls0_w0"] = head.cls_branches[0][0].weight.grad.numpy()
                out["grad_reg2_b4"] = head.reg_branches[2][4].bias.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "head_toy.npz"), **out)
    print("head_toy:", {k: v.shape for k, v in out.items() if k.endswith(("cls", "num", "grad_hs"))})


def head_keys():
    Head, HeadG, _, _ = load_reference_head()
    from tests.test_group_attention_cpu import load_reference_group_attention
    mmcv_stub.ATTENTION.register_module(name="GroupMultiheadAttention", module=load_reference_group_attention(),
                                        force=True)
    out = {}
    for name, path in (("tiny", "bevformer/bevformer_tiny.py"), ("small", "bevformer/bevformer_small.py"),
                       ("base", "bevformer/bevformer_base.py"), ("v2", "bevformerv2/bevformerv2-r50-t1-24ep.py")):
        cfg = config.load_config(os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs", path))
        hcfg = copy.deepcopy(cfg["model"]["pts_bbox_head"])
        typ = hcfg.pop("type")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            head = (HeadG if typ == "BEVFormerHead_GroupDETR" else Head)(**hcfg)
        out[name] = np.array(sorted(head.state_dict()))
        out[name + "_config"] = np.array(path)
        # the config's own pts_bbox_head dict, so that a checkout without the reference tree builds the same head
        out[name + "_pts_bbox_head"] = np.array(json.dumps(cfg["model"]["pts_bbox_head"]))
        print(f"head keys {name}: {len(out[name])}")
    np.savez_compressed(os.path.join(OUT, "head_keys.npz"), **out)


def nms_decode():
    _, _, Coder, _ = load_reference_head()
    for name, (thr, _, _) in ho.NMS_CASES.items():
        cls, box = ho.nms_case_inputs(name)
        out = {}
        for dt, tag in ((torch.float64, "fp64"), (torch.float32, "fp32")):
            coder = Coder(pc_range=ho.PC_RANGE, post_center_range=list(ho.POST_CENTER_RANGE), max_num=100,
                          score_threshold=thr, num_classes=10)
            res = coder.decode(dict(all_cls_scores=cls.to(dt)[None], all_bbox_preds=box.to(dt)[None]))
            out.update(_decoded([(r["bboxes"], r["scores"], r["labels"]) for r in res], tag))
        np.savez_compressed(os.path.join(OUT, f"ref_nms_decode_{name}.npz"), **out)
        print(f"ref_nms_decode_{name}: kept {out['fp64_num'].tolist()} of 100")


if __name__ == "__main__":
    if not mmcv_stub.reference_available():
        raise SystemExit("needs a reference checkout (set BEVF_REFERENCE_ROOT)")
    torch.manual_seed(0)
    head_toy()
    nms_decode()
    head_keys()
    for f in sorted(os.listdir(OUT)):
        if f.startswith(("head_", "ref_nms_decode_")):
            assert os.path.getsize(os.path.join(OUT, f)) < 1 << 20, f
