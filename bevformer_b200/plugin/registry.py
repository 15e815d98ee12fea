"""Registry surface the reference configs are built through (SURVEY.md §8b).

When mmcv is importable (a real BEVFormer checkout) the classes register into mmcv's own
ATTENTION / TRANSFORMER_LAYER / TRANSFORMER_LAYER_SEQUENCE / FEEDFORWARD_NETWORK registries, so
``build_transformer_layer_sequence(cfg)`` finds them under the reference's type names.  Without
mmcv (this image) an API-compatible local registry is used.
"""
from __future__ import annotations

import copy

try:  # pragma: no cover - mmcv is absent from the build image
    import mmcv as _mmcv
    if getattr(_mmcv, "_bevf_stub", False):
        # the test oracle's stand-in for mmcv (oracle/mmcv_stub.py) holds the REFERENCE classes: the
        # product must never register into it, whatever the import order of a test session
        raise ImportError("oracle stub, not mmcv")
    from mmcv.cnn.bricks.registry import (ATTENTION, FEEDFORWARD_NETWORK, TRANSFORMER_LAYER,
                                          TRANSFORMER_LAYER_SEQUENCE)
    from mmcv.utils import build_from_cfg
    HAVE_MMCV = True
except Exception:  # noqa: BLE001
    HAVE_MMCV = False

    class Registry:
        def __init__(self, name):
            self.name = name
            self.module_dict = {}

        def register_module(self, name=None, force=False, module=None):
            def deco(cls):
                key = name or cls.__name__
                if key in self.module_dict and not force and self.module_dict[key] is not cls:
                    raise KeyError(f"{key} is already registered in {self.name}")
                self.module_dict[key] = cls
                return cls
            return deco(module) if module is not None else deco

        def get(self, key):
            return self.module_dict.get(key)

        def build(self, cfg, **default_args):
            return build_from_cfg(cfg, self, default_args or None)

    def build_from_cfg(cfg, registry, default_args=None):
        if not isinstance(cfg, dict) or "type" not in cfg:
            raise KeyError("cfg must be a dict with a 'type' key")
        args = copy.deepcopy(dict(cfg))
        for k, v in (default_args or {}).items():
            args.setdefault(k, v)
        typ = args.pop("type")
        cls = registry.get(typ) if isinstance(typ, str) else typ
        if cls is None:
            raise KeyError(f"{typ} is not in the {registry.name} registry")
        return cls(**args)

    ATTENTION = Registry("attention")
    FEEDFORWARD_NETWORK = Registry("feed-forward Network")
    TRANSFORMER_LAYER = Registry("transformerLayer")
    TRANSFORMER_LAYER_SEQUENCE = Registry("transformer-layers sequence")


# PerceptionTransformer registers in mmdet's TRANSFORMER registry (modules/transformer.py:26)
try:  # pragma: no cover - mmdet is absent from the build image
    from mmdet.models.utils.builder import TRANSFORMER
except Exception:  # noqa: BLE001
    if HAVE_MMCV:
        from mmcv.utils import Registry as _MmcvRegistry
        TRANSFORMER = _MmcvRegistry("Transformer")
    else:
        TRANSFORMER = Registry("Transformer")


# BEVFormerHead / NMSFreeCoder / LearnedPositionalEncoding register where the reference's classes do: mmdet's HEADS
# (dense_heads/bevformer_head.py:16), mmdet's BBOX_CODERS (core/bbox/coders/nms_free_coder.py:9) and mmcv's
# POSITIONAL_ENCODING (mmdet 2.14 models/utils/positional_encoding.py)
def _registry(import_name, attr, name):
    try:  # pragma: no cover - mmdet / mmcv are absent from the build image
        if not HAVE_MMCV:
            raise ImportError(import_name)
        import importlib
        return getattr(importlib.import_module(import_name), attr)
    except Exception:  # noqa: BLE001
        if HAVE_MMCV:
            from mmcv.utils import Registry as _MmcvRegistry
            return _MmcvRegistry(name)
        return Registry(name)


HEADS = _registry("mmdet.models.builder", "HEADS", "head")
BBOX_CODERS = _registry("mmdet.core.bbox.builder", "BBOX_CODERS", "bbox_coder")
POSITIONAL_ENCODING = _registry("mmcv.cnn.bricks.registry", "POSITIONAL_ENCODING", "position encoding")
# ModulatedDeformConv2dPack registers as 'DCNv2' where mmcv's own class does (mmcv/ops/modulated_deform_conv.py), and
# replaces it there: mmdet's ResNet builds its dcn convs through mmcv.cnn's build_conv_layer
CONV_LAYERS = _registry("mmcv.cnn.bricks.registry", "CONV_LAYERS", "conv layer")


def _register(registry, cls, name=None):
    """Register without tripping over a name mmcv (or an earlier import) already holds."""
    try:
        registry.register_module(name=name, module=cls)
    except (KeyError, TypeError):
        try:
            registry.register_module(name=name, force=True, module=cls)
        except Exception:  # noqa: BLE001
            pass
    return cls


if not HAVE_MMCV:     # what mmcv.cnn.bricks.conv registers
    import torch.nn as _nn
    for _name, _cls in (("Conv1d", _nn.Conv1d), ("Conv2d", _nn.Conv2d), ("Conv3d", _nn.Conv3d), ("Conv", _nn.Conv2d)):
        CONV_LAYERS.register_module(name=_name, module=_cls)


def build_conv_layer(cfg, *args, **kwargs):
    """mmcv.cnn.build_conv_layer: the CONV_LAYERS class named by cfg['type'] (cfg None: nn.Conv2d), built with
    ``*args, **kwargs`` plus the rest of cfg."""
    if cfg is None:
        cfg_ = dict(type="Conv2d")
    else:
        if not isinstance(cfg, dict):
            raise TypeError("cfg must be a dict")
        if "type" not in cfg:
            raise KeyError('the cfg dict must contain the key "type"')
        cfg_ = dict(cfg)
    layer_type = cfg_.pop("type")
    conv_layer = CONV_LAYERS.get(layer_type)
    if conv_layer is None:
        raise KeyError(f"Unrecognized conv type {layer_type}")
    return conv_layer(*args, **kwargs, **cfg_)


def build_attention(cfg, default_args=None):
    return build_from_cfg(cfg, ATTENTION, default_args)


def build_feedforward_network(cfg, default_args=None):
    return build_from_cfg(cfg, FEEDFORWARD_NETWORK, default_args)


def build_transformer_layer(cfg, default_args=None):
    return build_from_cfg(cfg, TRANSFORMER_LAYER, default_args)


def build_transformer_layer_sequence(cfg, default_args=None):
    if cfg is None:
        return None
    return build_from_cfg(cfg, TRANSFORMER_LAYER_SEQUENCE, default_args)
