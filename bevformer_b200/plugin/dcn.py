"""Modulated deformable convolution (DCNv2) modules: drop-ins for mmcv's ModulatedDeformConv2d and
ModulatedDeformConv2dPack (mmcv-full 1.4.0 mmcv/ops/modulated_deform_conv.py), the ``dcn=dict(type='DCNv2', ...)``
convolutions of the ResNet-101-DCN backbone (projects/configs/bevformer/bevformer_base.py:43-53).

Same constructor arguments, parameter names, initialisers and state-dict migration as mmcv's classes; the op is
``ops.modulated_deform_conv2d`` (csrc/dcn.cu around the library's GEMMs).  The Pack module registers in CONV_LAYERS as
'DCNv2' (plugin/registry.py).
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.utils import _pair, _single

from .. import ops, precision
from .registry import CONV_LAYERS, _register


class ModulatedDeformConv2d(nn.Module):
    """out = modulated_deform_conv2d(x, offset, mask, weight, bias, ...) with offset / mask supplied by the caller."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deform_groups=1, bias=True):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = _pair(stride)
        self.padding = _pair(padding)
        self.dilation = _pair(dilation)
        self.groups = groups
        self.deform_groups = deform_groups
        # enable compatibility with nn.Conv2d
        self.transposed = False
        self.output_padding = _single(0)
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self.init_weights()

    def init_weights(self):
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.zero_()

    def _conv(self, x, offset, mask):
        return ops.modulated_deform_conv2d(x, offset, mask, self.weight, self.bias, self.stride, self.padding,
                                           self.dilation, self.groups, self.deform_groups)

    @precision.entry("x", "offset", "mask")
    def forward(self, x, offset, mask):
        return self._conv(x, offset, mask)


class ModulatedDeformConv2dPack(ModulatedDeformConv2d):
    """ModulatedDeformConv2d that predicts its own offset and mask with ``conv_offset`` (zero-initialised, so a fresh
    module starts as a plain convolution with mask 0.5): o1, o2, m = chunk(conv_offset(x), 3, 1),
    offset = cat(o1, o2), mask = sigmoid(m)."""

    _version = 2

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deform_groups * 3 * self.kernel_size[0] *
                                     self.kernel_size[1], kernel_size=self.kernel_size, stride=self.stride,
                                     padding=self.padding, dilation=self.dilation, bias=True)
        self.init_weights()

    def init_weights(self):
        super().init_weights()
        if hasattr(self, "conv_offset"):
            self.conv_offset.weight.data.zero_()
            self.conv_offset.bias.data.zero_()

    @precision.entry("x")
    def forward(self, x):
        # conv_offset runs on cuDNN in x's dtype (the entry point has switched autocast off for the body)
        w, b = self.conv_offset.weight, self.conv_offset.bias
        out = F.conv2d(x, w.to(x.dtype), b.to(x.dtype), self.conv_offset.stride, self.conv_offset.padding,
                       self.conv_offset.dilation)
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        return self._conv(x, offset, torch.sigmoid(mask))

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        version = local_metadata.get("version", None)
        if version is None or version < 2:
            _adopt_offset_keys(state_dict, prefix)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)


def _adopt_offset_keys(state_dict, prefix):
    """Checkpoints of the original DCNv2 (such as the configs' r101_dcn_fcos3d_pretrain.pth) hold the offset conv as
    ``<name>_offset.*`` beside the module: rename them to ``<name>.conv_offset.*``."""
    for p in ("weight", "bias"):
        old, new = prefix[:-1] + "_offset." + p, prefix + "conv_offset." + p
        if new not in state_dict and old in state_dict:
            state_dict[new] = state_dict.pop(old)


def _parent_pre_hook(module, state_dict, prefix, *args):
    for name, child in module._modules.items():
        if isinstance(child, ModulatedDeformConv2dPack):
            _adopt_offset_keys(state_dict, prefix + name + ".")


def _on_submodule(module, name, submodule):
    """The ``<name>_offset.*`` keys are the PARENT's (they do not start with ``<name>.``), and torch hands a child only
    the keys under its own prefix: the parent of every Pack module renames them before its children load."""
    if isinstance(submodule, ModulatedDeformConv2dPack) and not getattr(module, "_dcn_offset_hook", False):
        module.register_load_state_dict_pre_hook(_parent_pre_hook)
        object.__setattr__(module, "_dcn_offset_hook", True)


torch.nn.modules.module.register_module_module_registration_hook(_on_submodule)
_register(CONV_LAYERS, ModulatedDeformConv2dPack, "DCNv2")
