"""CustomMSDeformableAttention on the CUDA kernels: the decoder's cross-attention from object queries
into the BEV map, third call site of the sampler after TSA and SCA.

Drop-in for the reference class of the same name
(projects/mmdet3d_plugin/bevformer/modules/decoder.py:132-345): same registry name, constructor
arguments, parameter names / shapes / initialisers, forward signature and return convention.  Around it:
``DetectionTransformerDecoder`` (decoder.py:52-129, the reference-point refinement loop) and the two
third-party classes its config names -- mmdet's ``DetrTransformerDecoderLayer`` and mmcv's
``MultiheadAttention`` wrapper (mmcv-full==1.4.0 semantics) -- so that the decoder dict of
projects/configs/bevformer/*.py builds unchanged (SURVEY.md §8 f2).

The shapes here are small (900 queries, one 200x200 level, 4 points): the value projection over the
40 000 BEV cells is the only part with real work -- it and the other projections run on the wgmma
GEMM, the gather on the sampler kernel.  What sits between the library calls is fused too, because at these
sizes a decoder layer is bound by launches: the sampling-point prep runs on the TSA prep kernels with one
frame (``bevf_query_prep_*``), the reference-point refinement is one kernel (``bevf_refine_points``) and the
object-query self-attention runs on the attention kernel.
"""
from __future__ import annotations

import torch
import torch.nn as nn

import copy
import warnings

from .. import ops, precision
from .linear import linear, linear_fp32_out, query_sampling_head
from .registry import (ATTENTION, HAVE_MMCV, TRANSFORMER_LAYER, TRANSFORMER_LAYER_SEQUENCE, _register,
                       build_transformer_layer)
from .temporal_self_attention import _check_head_dim, ring_offsets_


class CustomMSDeformableAttention(nn.Module):
    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64,
                 dropout=0.1, batch_first=False, norm_cfg=None, init_cfg=None):
        super().__init__()
        _check_head_dim(embed_dims, num_heads)
        self.init_cfg = init_cfg
        self.norm_cfg = norm_cfg
        self.dropout = nn.Dropout(dropout)
        self.batch_first = batch_first
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weights()

    def init_weights(self):
        """decoder.py:209-228: zero offset/attention weights, ring bias, xavier projections."""
        nn.init.zeros_(self.sampling_offsets.weight)
        ring_offsets_(self.sampling_offsets.bias, self.num_heads, self.num_levels, self.num_points)
        nn.init.zeros_(self.attention_weights.weight)
        nn.init.zeros_(self.attention_weights.bias)
        for lin in (self.value_proj, self.output_proj):
            nn.init.xavier_uniform_(lin.weight)
            nn.init.zeros_(lin.bias)
        self._is_init = True

    @precision.entry("query", "key", "value", "identity", "query_pos")
    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, flag="decoder", **kwargs):
        """query (num_query, bs, C) (or batch-first), value (num_key, bs, C), reference_points
        (bs, num_query, num_levels, 2 | 4).  Returns dropout(output_proj(sampled)) + identity in the
        caller's layout (decoder.py:233-345)."""
        if value is None:
            value = query
        if identity is None:
            identity = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query = query.permute(1, 0, 2)
            value = value.permute(1, 0, 2)
        bs, nq, _ = query.shape
        nv = value.shape[1]
        m, l, p = self.num_heads, self.num_levels, self.num_points
        ss = torch.as_tensor(spatial_shapes).to(device=query.device, dtype=torch.int64)
        lsi = torch.as_tensor(level_start_index).to(device=query.device, dtype=torch.int64)
        if ss.shape[0] != l:
            raise AssertionError("spatial_shapes does not have num_levels rows")
        # (the reference also asserts sum(h*w) == num_value, a host sync per call: the sampler's
        #  argument check covers it without one)

        v = linear(value, self.value_proj.weight, self.value_proj.bias)
        if key_padding_mask is not None:
            v = v.masked_fill(key_padding_mask[..., None], 0.0)
        v = v.reshape(bs, nv, m, -1)
        w = torch.cat([self.sampling_offsets.weight, self.attention_weights.weight], 0)
        b = torch.cat([self.sampling_offsets.bias, self.attention_weights.bias], 0)
        if reference_points.shape[-1] == 2 and query.is_cuda:
            # the offsets|logits head and the softmax / offset / (W, H) + reference point prep (:300-330) as one
            # node: the TSA prep kernels with one frame
            ref = reference_points.reshape(bs, nq, l, 2).float().contiguous()
            loc, att = query_sampling_head(query, w, b, ref, ss.contiguous(), bs, nq, m, l, p)
            if reference_points.requires_grad and torch.is_grad_enabled():
                # the prep reads the reference points as a constant; their gradient (grad_loc summed over heads
                # and points, what the reference's broadcast add gives them) flows through this zero-valued term
                d = reference_points.reshape(bs, nq, l, 2).float()
                loc = loc + (d - d.detach())[:, :, None, :, None, :]
            out = ops.MultiScaleDeformableAttnFunction_fp32.apply(v, ss, lsi, loc, att, self.im2col_step)
            out = linear(out.to(query.dtype), self.output_proj.weight, self.output_proj.bias)
            if not self.batch_first:
                out = out.permute(1, 0, 2)
            return self.dropout(out) + identity
        raw = linear_fp32_out(query, w, b)                                   # (bs, nq, m*l*p*3) fp32
        n_off = m * l * p * 2
        off = raw[..., :n_off].reshape(bs, nq, m, l, p, 2)
        att = raw[..., n_off:].reshape(bs, nq, m, l * p).softmax(-1).reshape(bs, nq, m, l, p)
        rp = reference_points.float()
        if rp.shape[-1] == 2:
            norm = torch.stack([ss[..., 1], ss[..., 0]], -1).to(torch.float32)
            loc = rp[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
        elif rp.shape[-1] == 4:
            loc = rp[:, :, None, :, None, :2] + off / p * rp[:, :, None, :, None, 2:] * 0.5
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, "
                             f"but get {rp.shape[-1]} instead.")
        out = ops.MultiScaleDeformableAttnFunction_fp32.apply(v, ss, lsi, loc.contiguous(),
                                                              att.contiguous(), self.im2col_step)
        out = linear(out.to(query.dtype), self.output_proj.weight, self.output_proj.bias)
        if not self.batch_first:
            out = out.permute(1, 0, 2)
        return self.dropout(out) + identity


_register(ATTENTION, CustomMSDeformableAttention)


def inverse_sigmoid(x, eps=1e-5):
    """decoder.py:31-49."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


class _KernelAttention(nn.Module):
    """The attention-kernel route shared by mmcv's ``MultiheadAttention`` wrapper and ``GroupMultiheadAttention``
    (both keep their ``nn.MultiheadAttention`` as ``self.attn``): 16-bit CUDA inputs with head_dim 32 and no masks
    run the in-projection on the wgmma GEMM (one GEMM over the [W_q; W_k] rows when query and key are the same
    tensor), ``ops.GroupAttention`` (Philox dropout in training) and the out-projection on the GEMM."""

    def _kernel_ok(self, query, key, attn_mask, key_padding_mask, groups):
        a = self.attn
        return (query.is_cuda and query.dtype in ops.TC_DTYPES and key.dtype == query.dtype
                and attn_mask is None and key_padding_mask is None
                and self.embed_dims == self.num_heads * 32 and a._qkv_same_embed_dim and a.bias_k is None
                and not a.add_zero_attn and not a.batch_first and (groups == 1 or key.shape[0] == query.shape[0]))

    def _forward_kernel(self, qin, kin, value, shared, groups):
        a, C = self.attn, self.embed_dims
        w, b = a.in_proj_weight, a.in_proj_bias
        bq = (lambda lo, hi: None) if b is None else (lambda lo, hi: b[lo:hi])
        v = linear(value, w[2 * C:], bq(2 * C, 3 * C))
        drop = a.dropout if self.training else 0.0
        scale = float(C // self.num_heads) ** -0.5
        if shared:
            qk = linear(qin, w[:2 * C], bq(0, 2 * C))
            out = ops.GroupAttention.apply(qk, None, v, self.num_heads, groups, scale, drop)
        else:
            q = linear(qin, w[:C], bq(0, C))
            k = linear(kin, w[C:2 * C], bq(C, 2 * C))
            out = ops.GroupAttention.apply(q, k, v, self.num_heads, groups, scale, drop)
        return linear(out, a.out_proj.weight, a.out_proj.bias)


class MultiheadAttention(_KernelAttention):
    """mmcv's wrapper around nn.MultiheadAttention (mmcv/cnn/bricks/transformer.py, 1.4.0): positional
    encodings added to query / key, optional batch-first layout, ``identity + dropout_layer(proj_drop(attn))``.
    The object-query self-attention of the decoder (900 queries): on the attention kernel with ``groups = 1``
    (_KernelAttention) for 16-bit CUDA inputs, head_dim 32 and no masks; fp32 and masked calls keep
    ``nn.MultiheadAttention``."""

    def __init__(self, embed_dims, num_heads, attn_drop=0.0, proj_drop=0.0,
                 dropout_layer=dict(type="Dropout", drop_prob=0.0), init_cfg=None, batch_first=False, **kwargs):
        super().__init__()
        if "dropout" in kwargs:                      # deprecated spelling the BEVFormer configs still use
            attn_drop = kwargs["dropout"]
            dropout_layer = dict(dropout_layer or dict(type="Dropout"), drop_prob=kwargs.pop("dropout"))
        self.init_cfg = init_cfg
        self.embed_dims, self.num_heads, self.batch_first = embed_dims, num_heads, batch_first
        self.attn = nn.MultiheadAttention(embed_dims, num_heads, attn_drop, **kwargs)
        self.proj_drop = nn.Dropout(proj_drop)
        dl = dict(dropout_layer) if dropout_layer else None
        self.dropout_layer = nn.Dropout(dl.get("drop_prob", 0.0)) if dl and dl.get("type", "Dropout") == "Dropout" \
            else nn.Identity()

    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_pos=None,
                attn_mask=None, key_padding_mask=None, **kwargs):
        if key is None:
            key = query
        if value is None:
            value = key
        if identity is None:
            identity = query
        if key_pos is None and query_pos is not None and query_pos.shape == key.shape:
            key_pos = query_pos
        shared = key is query and key_pos is query_pos       # self-attention: Q and K projected by one GEMM
        if query_pos is not None:
            query = query + query_pos
        if shared:
            key = query
        elif key_pos is not None:
            key = key + key_pos
        if self.batch_first:
            query, key, value = query.transpose(0, 1), key.transpose(0, 1), value.transpose(0, 1)
        if self._kernel_ok(query, key, attn_mask, key_padding_mask, 1):
            out = self._forward_kernel(query, key, value, shared, 1)
        else:
            out = self.attn(query=query, key=key, value=value, attn_mask=attn_mask,
                            key_padding_mask=key_padding_mask)[0]
        if self.batch_first:
            out = out.transpose(0, 1)
        return identity + self.dropout_layer(self.proj_drop(out))


_GROUP_DROPOUT_DEFAULT = dict(type="Dropout", drop_prob=0.)


class GroupMultiheadAttention(_KernelAttention):
    """Group DETR's decoder self-attention (group_attention.py:18-162): mmcv's MultiheadAttention wrapper whose
    ``num_query`` queries split, in training only, into ``group`` equal slices that attend only within their own
    slice.  The BEVFormerV2 configs train 11 groups of 900 queries (9900) and evaluate one group.

    Same registry name, constructor arguments, parameters (an ``nn.MultiheadAttention`` as ``self.attn`` holds
    ``in_proj_weight/bias`` and ``out_proj``) and forward contract as the reference.  16-bit CUDA inputs with
    head_dim 32 and no masks run the in-projection on the wgmma GEMM (one GEMM over the [W_q; W_k] rows when query
    and key are the same tensor), the grouped attention kernel (``ops.GroupAttention``) and the out-projection on
    the GEMM.  fp32 inputs, masks and other head sizes take the reference arithmetic on torch.

    One deviation: with the deprecated ``dropout`` kwarg the reference writes ``drop_prob`` into ``dropout_layer``
    in place, and so into its shared default dict, which then leaks into every later instance built without
    ``dropout_layer``.  Here a dict the caller passes is updated in place as there, the default is not shared."""

    def __init__(self, embed_dims, num_heads, attn_drop=0., proj_drop=0., group=1,
                 dropout_layer=_GROUP_DROPOUT_DEFAULT, init_cfg=None, batch_first=False, **kwargs):
        super().__init__()
        if dropout_layer is _GROUP_DROPOUT_DEFAULT:
            dropout_layer = dict(dropout_layer)
        if "dropout" in kwargs:
            warnings.warn("The arguments `dropout` in MultiheadAttention has been deprecated, now you can "
                          "separately set `attn_drop`(float), proj_drop(float), and `dropout_layer`(dict) ",
                          DeprecationWarning)
            attn_drop = kwargs["dropout"]
            dropout_layer["drop_prob"] = kwargs.pop("dropout")
        self.init_cfg = init_cfg
        self.embed_dims, self.num_heads, self.group, self.batch_first = embed_dims, num_heads, group, batch_first
        self.attn = nn.MultiheadAttention(embed_dims, num_heads, attn_drop, **kwargs)
        self.proj_drop = nn.Dropout(proj_drop)
        if dropout_layer and dropout_layer.get("type", "Dropout") != "Dropout":
            raise NotImplementedError(f"GroupMultiheadAttention: dropout_layer type {dropout_layer['type']!r} is not "
                                      "supported (only 'Dropout')")
        self.dropout_layer = nn.Dropout(dropout_layer.get("drop_prob", 0.0)) if dropout_layer else nn.Identity()

    @precision.entry("query", "key", "value", "identity", "query_pos", "key_pos")
    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_pos=None,
                attn_mask=None, key_padding_mask=None, **kwargs):
        """query (num_query, bs, C) (or batch-first); returns identity + dropout_layer(proj_drop(attn)) in the same
        layout (group_attention.py:117-162)."""
        if "residual" in kwargs:               # mmcv's deprecated_api_warning({'residual': 'identity'})
            warnings.warn("'residual' is deprecated in MultiheadAttention, please use 'identity' instead",
                          DeprecationWarning)
            identity = kwargs.pop("residual")
        if key is None:
            key = query
        if value is None:
            value = key
        if identity is None:
            identity = query
        if key_pos is None and query_pos is not None:
            if query_pos.shape == key.shape:
                key_pos = query_pos
            else:
                warnings.warn(f"position encoding of key is missing in {self.__class__.__name__}.")
        shared = key is query and key_pos is query_pos       # self-attention: Q and K projected by one GEMM
        qin = query if query_pos is None else query + query_pos
        kin = qin if shared else (key if key_pos is None else key + key_pos)
        if self.batch_first:
            qin, kin, value = qin.transpose(0, 1), kin.transpose(0, 1), value.transpose(0, 1)
        nq, bs = qin.shape[0], qin.shape[1]
        groups = self.group if self.training else 1
        if self.training and (self.group <= 0 or nq % self.group):
            raise RuntimeError(f"GroupMultiheadAttention: {nq} queries do not split into {self.group} equal groups")
        if self._kernel_ok(qin, kin, attn_mask, key_padding_mask, groups):
            out = self._forward_kernel(qin, kin, value, shared, groups)
        else:
            out = self._forward_torch(qin, kin, value, attn_mask, key_padding_mask, nq, bs)
        if self.batch_first:
            out = out.transpose(0, 1)
        return identity + self.dropout_layer(self.proj_drop(out))

    def _forward_torch(self, query, key, value, attn_mask, key_padding_mask, nq, bs):
        """The reference's arithmetic: groups moved to the batch axis around nn.MultiheadAttention."""
        if self.training:
            query = torch.cat(query.split(nq // self.group, dim=0), dim=1)
            key = torch.cat(key.split(nq // self.group, dim=0), dim=1)
            value = torch.cat(value.split(nq // self.group, dim=0), dim=1)
        out = self.attn(query=query, key=key, value=value, attn_mask=attn_mask, key_padding_mask=key_padding_mask)[0]
        if self.training:
            out = torch.cat(out.split(bs, dim=1), dim=0)
        return out


def _decoder_layer_cls():
    from .encoder import MyCustomBaseTransformerLayer

    class DetrTransformerDecoderLayer(MyCustomBaseTransformerLayer):
        """mmdet's DETR decoder layer (mmdet/models/utils/transformer.py, 2.14): mmcv's BaseTransformerLayer
        with sequence-first tensors and the six-step order (self_attn, norm, cross_attn, norm, ffn, norm)."""

        def __init__(self, attn_cfgs, feedforward_channels, ffn_dropout=0.0, operation_order=None,
                     act_cfg=dict(type="ReLU", inplace=True), norm_cfg=dict(type="LN"), ffn_num_fcs=2, **kwargs):
            kwargs.setdefault("batch_first", False)
            super().__init__(attn_cfgs=attn_cfgs, feedforward_channels=feedforward_channels,
                             ffn_dropout=ffn_dropout, operation_order=operation_order, act_cfg=act_cfg,
                             norm_cfg=norm_cfg, ffn_num_fcs=ffn_num_fcs, **kwargs)
            assert len(self.operation_order) == 6
            assert set(self.operation_order) == {"self_attn", "norm", "cross_attn", "ffn"}

    return DetrTransformerDecoderLayer


def _run_branch(branch, x):
    """A head branch (the caller's module) on a decoder output.  Inside an entry point autocast is off; a 16-bit
    output meeting an fp32 branch then runs the branch under autocast in that dtype, as the caller's autocast
    would have."""
    p = next(branch.parameters(), None)
    if x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and p is not None and p.dtype != x.dtype:
        with torch.autocast(device_type="cuda", dtype=x.dtype):
            return branch(x)
    return branch(x)


class DetectionTransformerDecoder(nn.Module):
    """The DETR3D-style decoder (decoder.py:52-129): ``num_layers`` decoder layers; after each, the
    layer's regression branch refines the (x, y, z) reference points in inverse-sigmoid space and the
    refined points are detached before the next layer.  Also plays mmcv's TransformerLayerSequence
    (deep-copies the layer config ``num_layers`` times into ``self.layers``)."""

    def __init__(self, *args, transformerlayers=None, num_layers=None, return_intermediate=False,
                 init_cfg=None, **kwargs):
        super().__init__()
        if args:
            transformerlayers = args[0]
            num_layers = args[1] if len(args) > 1 else num_layers
        if isinstance(transformerlayers, dict):
            transformerlayers = [copy.deepcopy(transformerlayers) for _ in range(num_layers)]
        assert isinstance(transformerlayers, (list, tuple)) and len(transformerlayers) == num_layers
        self.init_cfg = init_cfg
        self.num_layers = num_layers
        self.layers = nn.ModuleList(build_transformer_layer(c) for c in transformerlayers)
        self.embed_dims = self.layers[0].embed_dims
        self.pre_norm = self.layers[0].pre_norm
        self.return_intermediate = return_intermediate
        self.fp16_enabled = False

    def forward(self, query, *args, reference_points=None, reg_branches=None, key_padding_mask=None, **kwargs):
        """query (num_query, bs, C); reference_points (bs, num_query, 3) in [0, 1].  Returns
        (stack of layer outputs, stack of reference points) with return_intermediate, else the last pair."""
        output = query
        intermediate, intermediate_reference_points = [], []
        ref2d = None            # the refinement kernel's fp32 (bs, nq, 1, 2) copy of reference_points[..., :2]
        for lid, layer in enumerate(self.layers):
            reference_points_input = reference_points[..., :2].unsqueeze(2) if ref2d is None else ref2d
            output = layer(output, *args, reference_points=reference_points_input,
                           key_padding_mask=key_padding_mask, **kwargs)
            output = output.permute(1, 0, 2)
            if reg_branches is not None:
                tmp = _run_branch(reg_branches[lid], output)
                assert reference_points.shape[-1] == 3
                if tmp.is_cuda and tmp.dtype == reference_points.dtype:
                    # one kernel for the zeros_like / two inverse_sigmoid / slice assignments / sigmoid below
                    reference_points, ref2d = ops.refine_points(tmp.detach(), reference_points.detach())
                else:
                    new_reference_points = torch.zeros_like(reference_points)
                    new_reference_points[..., :2] = tmp[..., :2] + inverse_sigmoid(reference_points[..., :2])
                    new_reference_points[..., 2:3] = tmp[..., 4:5] + inverse_sigmoid(reference_points[..., 2:3])
                    reference_points = new_reference_points.sigmoid().detach()
            output = output.permute(1, 0, 2)
            if self.return_intermediate:
                intermediate.append(output)
                intermediate_reference_points.append(reference_points)
        if self.return_intermediate:
            return torch.stack(intermediate), torch.stack(intermediate_reference_points)
        return output, reference_points


DetrTransformerDecoderLayer = _decoder_layer_cls()
if not HAVE_MMCV:      # with a real mmcv / mmdet these two names keep their own classes
    _register(ATTENTION, MultiheadAttention)
    _register(TRANSFORMER_LAYER, DetrTransformerDecoderLayer)
_register(TRANSFORMER_LAYER_SEQUENCE, DetectionTransformerDecoder)
_register(ATTENTION, GroupMultiheadAttention)
