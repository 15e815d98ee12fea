"""Reads the reference's python config files (projects/configs/bevformer/*.py) without mmcv and
builds the encoder they describe.  The files are ``exec``-ed as mmcv's ``Config.fromfile`` does;
``_base_`` entries only carry dataset / runtime settings, which the encoder does not read."""
from __future__ import annotations

import copy
import os

from .registry import HEADS, build_from_cfg, build_transformer_layer_sequence


def load_config(path: str) -> dict:
    ns: dict = {"__file__": os.path.abspath(path)}
    with open(path) as f:
        exec(compile(f.read(), path, "exec"), ns)  # noqa: S102 - a config file the user names
    return {k: v for k, v in ns.items() if not k.startswith("__")}


def encoder_cfg_from_config(cfg: dict) -> dict:
    """``model.pts_bbox_head.transformer.encoder`` (bevformer_base.py:78-105)."""
    return copy.deepcopy(cfg["model"]["pts_bbox_head"]["transformer"]["encoder"])


def build_encoder(cfg_or_path):
    """Accepts a config file path, a full config dict, or the encoder dict itself."""
    cfg = load_config(cfg_or_path) if isinstance(cfg_or_path, str) else cfg_or_path
    if "model" in cfg:
        cfg = encoder_cfg_from_config(cfg)
    return build_transformer_layer_sequence(copy.deepcopy(cfg))


def head_cfg_from_config(cfg: dict) -> dict:
    """``model.pts_bbox_head`` with the detector's ``train_cfg.pts`` / ``test_cfg.pts`` added, as mmdet3d's
    MVXTwoStageDetector passes them to the head."""
    model = cfg["model"]
    head = copy.deepcopy(model["pts_bbox_head"])
    for key in ("train_cfg", "test_cfg"):
        sub = model.get(key)
        head.setdefault(key, copy.deepcopy(sub.get("pts")) if isinstance(sub, dict) else None)
    return head


def build_head(cfg_or_path):
    """BEVFormerHead / BEVFormerHead_GroupDETR (bevformer_b200.plugin.head) from a config file path, a full config
    dict, or the ``pts_bbox_head`` dict itself; the transformer inside is this package's."""
    from . import head as _head  # noqa: F401 - registers the head classes
    cfg = load_config(cfg_or_path) if isinstance(cfg_or_path, str) else cfg_or_path
    if "model" in cfg:
        cfg = head_cfg_from_config(cfg)
    return build_from_cfg(copy.deepcopy(cfg), HEADS)
