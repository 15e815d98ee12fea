"""BEVFormerEncoder / BEVFormerLayer / MyCustomBaseTransformerLayer / FFN on the CUDA kernels.

Drop-ins for projects/mmdet3d_plugin/bevformer/modules/encoder.py:24-406 and
custom_base_transformer_layer.py:37-260, plus the two mmcv classes those files instantiate from the
config (``FFN`` and ``TransformerLayerSequence``; mmcv-full==1.4.0 semantics as in SURVEY.md
Appendix B).  Parameter names follow the reference ``state_dict``:
``layers.{i}.attentions.{0,1}.*``, ``layers.{i}.ffns.0.layers.0.0.*``, ``layers.{i}.ffns.0.layers.1.*``,
``layers.{i}.norms.{0,1,2}.*``.

Per layer the reference issues ~60 launches (GEMMs, element-wise ops, copies, the op); here a layer
is: one stacked offsets|logits projection + value/output projections per attention, one prep
kernel, one sampler launch, one combine (SCA), and a fused dropout-residual-LayerNorm kernel after
each of the three blocks.
"""
from __future__ import annotations

import copy
import os
import warnings
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from .. import ops, precision
from .linear import linear, linear_relu_dropout, shared_input_projections
from .registry import (FEEDFORWARD_NETWORK, HAVE_MMCV, TRANSFORMER_LAYER, TRANSFORMER_LAYER_SEQUENCE, _register,
                       build_attention, build_feedforward_network, build_transformer_layer)
from .spatial_cross_attention import ScaPlan, SpatialCrossAttention
from .temporal_self_attention import TemporalSelfAttention

_OPS = ("self_attn", "norm", "ffn", "cross_attn")


class _DropPath(nn.Module):
    """mmcv's DropPath (stochastic depth per sample), for FFN(dropout_layer=dict(type='DropPath'))."""

    def __init__(self, drop_prob=0.1):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1.0 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        return x / keep * mask


def _build_dropout(cfg):
    if not cfg:
        return nn.Identity()
    cfg = dict(cfg)
    typ = cfg.pop("type", "Dropout")
    if typ == "Dropout":
        return nn.Dropout(cfg.get("drop_prob", cfg.get("p", 0.5)), inplace=cfg.get("inplace", False))
    if typ == "DropPath":
        return _DropPath(cfg.get("drop_prob", 0.1))
    raise KeyError(f"unsupported dropout_layer type {typ}")


class FFN(nn.Module):
    """mmcv's FFN: ``identity + Dropout(Linear(Dropout(act(Linear(x)))))`` with the module tree
    ``layers = Sequential(Sequential(Linear, act, Dropout), ..., Linear, Dropout)`` so that the
    checkpoint keys ``layers.0.0.*`` / ``layers.1.*`` line up."""

    def __init__(self, embed_dims=256, feedforward_channels=1024, num_fcs=2,
                 act_cfg=dict(type="ReLU", inplace=True), ffn_drop=0.0, dropout_layer=None,
                 add_identity=True, init_cfg=None, **kwargs):
        super().__init__()
        if num_fcs < 2:
            raise AssertionError(f"num_fcs should be no less than 2. got {num_fcs}.")
        act = (act_cfg or {}).get("type", "ReLU")
        if act not in ("ReLU", "GELU"):
            raise KeyError(f"unsupported FFN activation {act}")
        self.embed_dims, self.feedforward_channels, self.num_fcs = embed_dims, feedforward_channels, num_fcs
        self.act_type = act
        blocks, width = [], embed_dims
        for _ in range(num_fcs - 1):
            blocks.append(nn.Sequential(nn.Linear(width, feedforward_channels),
                                        nn.ReLU(inplace=True) if act == "ReLU" else nn.GELU(),
                                        nn.Dropout(ffn_drop)))
            width = feedforward_channels
        blocks += [nn.Linear(feedforward_channels, embed_dims), nn.Dropout(ffn_drop)]
        self.layers = nn.Sequential(*blocks)
        self.dropout_layer = _build_dropout(dropout_layer)      # mmcv: build_dropout(cfg) or Identity
        self.add_identity = add_identity

    def transform(self, x):
        """The stack without the identity add (hidden dropout included, final dropout not)."""
        h = x
        for blk in list(self.layers)[: self.num_fcs - 1]:
            if self.act_type == "ReLU":
                p = blk[2].p if blk[2].training else 0.0
                h = linear_relu_dropout(h, blk[0].weight, blk[0].bias, p)
            else:
                h = blk[2](blk[1](linear(h, blk[0].weight, blk[0].bias)))
        last = self.layers[self.num_fcs - 1]
        return linear(h, last.weight, last.bias)

    @precision.entry("x", "identity")
    def forward(self, x, identity=None):
        out = self.layers[self.num_fcs](self.transform(x))
        if not self.add_identity:
            return self.dropout_layer(out)
        return (x if identity is None else identity) + self.dropout_layer(out)


if not HAVE_MMCV:
    # local registry only: in a real mmcv checkout 'FFN' stays mmcv's own class (the detection decoder
    # builds its FFNs from the same registry); BEVFormer layers build THIS class directly, see
    # MyCustomBaseTransformerLayer.__init__
    _register(FEEDFORWARD_NETWORK, FFN, name="FFN")


def _fused_norm(norm: nn.LayerNorm, x, residual, dropout: Optional[nn.Dropout] = None, pos=None,
                twin: bool = False):
    """LayerNorm(dropout(x) + residual) in one kernel (fp32 statistics; the dropout of the block
    that produced x is applied inside, active only in training mode).  With ``pos`` the kernel also
    emits y + pos and the call returns (y, y + pos); with ``twin`` it returns (y, alias of y) so that the
    next block and its residual connection receive separate gradients (summed inside the backward kernel
    instead of by autograd).  Shapes the kernel does not cover (embed_dims other than 256 / 512) take the
    unfused CUDA ops instead."""
    if x.dtype not in (torch.float32, torch.bfloat16, torch.float16) or x.shape[-1] not in (256, 512):
        h = x if dropout is None else dropout(x)
        y = norm(h if residual is None else h + residual)
        if pos is None and twin:
            return y, y
        return y if pos is None else (y, y + pos)
    p = dropout.p if (dropout is not None and dropout.training) else 0.0
    return ops.LayerNormResidual.apply(x.contiguous(), residual, norm.weight, norm.bias, norm.eps, p, pos,
                                       twin and pos is None)


class MyCustomBaseTransformerLayer(nn.Module):
    """Builds ``attentions`` / ``ffns`` / ``norms`` from config dicts and runs them in
    ``operation_order`` (custom_base_transformer_layer.py:72-260)."""

    def __init__(self, attn_cfgs=None, ffn_cfgs=None, operation_order=None,
                 norm_cfg=dict(type="LN"), init_cfg=None, batch_first=True, **kwargs):
        super().__init__()
        ffn_cfgs = dict(type="FFN", embed_dims=256, feedforward_channels=1024, num_fcs=2, ffn_drop=0.0,
                        act_cfg=dict(type="ReLU", inplace=True)) if ffn_cfgs is None else copy.deepcopy(ffn_cfgs)
        legacy = dict(feedforward_channels="feedforward_channels", ffn_dropout="ffn_drop",
                      ffn_num_fcs="num_fcs")
        for old, new in legacy.items():                       # deprecated kwargs the configs still use
            if old in kwargs:
                ffn_cfgs[new] = kwargs[old]
        if "act_cfg" in kwargs and isinstance(ffn_cfgs, dict):
            ffn_cfgs.setdefault("act_cfg", kwargs["act_cfg"])
        operation_order = tuple(operation_order)
        if not set(operation_order) <= set(_OPS):
            raise AssertionError(f"operation_order of {type(self).__name__} may only contain {_OPS}")
        self.init_cfg = init_cfg
        self.batch_first = batch_first
        self.operation_order = operation_order
        self.norm_cfg = norm_cfg
        self.pre_norm = operation_order[0] == "norm"
        self.num_attn = operation_order.count("self_attn") + operation_order.count("cross_attn")
        if isinstance(attn_cfgs, dict):
            attn_cfgs = [copy.deepcopy(attn_cfgs) for _ in range(self.num_attn)]
        else:
            attn_cfgs = [copy.deepcopy(c) for c in attn_cfgs]
            if len(attn_cfgs) != self.num_attn:
                raise AssertionError(f"{len(attn_cfgs)} attention configs for {self.num_attn} attention "
                                     f"operations in {operation_order}")
        self.attentions = nn.ModuleList()
        names = [n for n in operation_order if n in ("self_attn", "cross_attn")]
        for cfg, name in zip(attn_cfgs, names):
            if "batch_first" in cfg:
                assert self.batch_first == cfg["batch_first"]
            else:
                cfg["batch_first"] = self.batch_first
            att = build_attention(cfg)
            att.operation_name = name
            self.attentions.append(att)
        self.embed_dims = self.attentions[0].embed_dims

        n_ffn = operation_order.count("ffn")
        if isinstance(ffn_cfgs, dict):
            ffn_cfgs = [copy.deepcopy(ffn_cfgs) for _ in range(n_ffn)]
        assert len(ffn_cfgs) == n_ffn
        self.ffns = nn.ModuleList()
        for cfg in ffn_cfgs:
            cfg = dict(cfg)
            cfg.setdefault("embed_dims", self.embed_dims)
            assert cfg["embed_dims"] == self.embed_dims
            if cfg.get("type", "FFN") == "FFN":       # the kernels' FFN, whatever mmcv registered as 'FFN'
                cfg.pop("type", None)
                self.ffns.append(FFN(**cfg))
            else:
                self.ffns.append(build_feedforward_network(cfg))

        if (norm_cfg or {}).get("type", "LN") != "LN":
            raise KeyError("only LayerNorm ('LN') is supported")
        self.norms = nn.ModuleList(
            nn.LayerNorm(self.embed_dims, eps=(norm_cfg or {}).get("eps", 1e-5))
            for _ in range(operation_order.count("norm")))

    def _attn_masks(self, attn_masks):
        if attn_masks is None:
            return [None] * self.num_attn
        if isinstance(attn_masks, torch.Tensor):
            warnings.warn(f"Use same attn_mask in all attentions in {type(self).__name__} ")
            return [copy.deepcopy(attn_masks) for _ in range(self.num_attn)]
        assert len(attn_masks) == self.num_attn
        return attn_masks

    def forward(self, query, key=None, value=None, query_pos=None, key_pos=None, attn_masks=None,
                query_key_padding_mask=None, key_padding_mask=None, **kwargs):
        masks = self._attn_masks(attn_masks)
        ni = ai = fi = 0
        identity = query
        for op in self.operation_order:
            if op == "self_attn":
                query = self.attentions[ai](query, query, query, identity if self.pre_norm else None,
                                            query_pos=query_pos, key_pos=query_pos,
                                            attn_mask=masks[ai],
                                            key_padding_mask=query_key_padding_mask, **kwargs)
                ai += 1
                identity = query
            elif op == "cross_attn":
                query = self.attentions[ai](query, key, value, identity if self.pre_norm else None,
                                            query_pos=query_pos, key_pos=key_pos, attn_mask=masks[ai],
                                            key_padding_mask=key_padding_mask, **kwargs)
                ai += 1
                identity = query
            elif op == "norm":
                query = _fused_norm(self.norms[ni], query, None) if query.is_cuda else self.norms[ni](query)
                ni += 1
            else:
                query = self.ffns[fi](query, identity if self.pre_norm else None)
                fi += 1
        return query


class BEVFormerLayer(MyCustomBaseTransformerLayer):
    """One encoder layer: temporal self-attention, spatial cross-attention, FFN, each followed by a
    LayerNorm (encoder.py:242-406).  When a block is directly followed by ``norm`` (the post-norm
    order every shipped config uses) its dropout + identity add are folded into the LayerNorm
    kernel; any other order runs through the blocks' public forwards."""

    def __init__(self, attn_cfgs, feedforward_channels, ffn_dropout=0.0, operation_order=None,
                 act_cfg=dict(type="ReLU", inplace=True), norm_cfg=dict(type="LN"), ffn_num_fcs=2,
                 **kwargs):
        super().__init__(attn_cfgs=attn_cfgs, feedforward_channels=feedforward_channels,
                         ffn_dropout=ffn_dropout, operation_order=operation_order, act_cfg=act_cfg,
                         norm_cfg=norm_cfg, ffn_num_fcs=ffn_num_fcs, **kwargs)
        self.fp16_enabled = False
        assert len(self.operation_order) == 6
        assert set(self.operation_order) == {"self_attn", "norm", "cross_attn", "ffn"}

    def forward(self, query, key=None, value=None, bev_pos=None, query_pos=None, key_pos=None,
                attn_masks=None, query_key_padding_mask=None, key_padding_mask=None, ref_2d=None,
                ref_3d=None, bev_h=None, bev_w=None, reference_points_cam=None, mask=None,
                spatial_shapes=None, level_start_index=None, prev_bev=None, **kwargs):
        masks = self._attn_masks(attn_masks)
        order = self.operation_order
        ni = ai = fi = 0
        identity = query
        # encoder-internal: {"q_in": query + bev_pos computed by the previous layer's last LayerNorm,
        # "emit": write this layer's output + bev_pos there for the next layer}
        carry = kwargs.pop("pos_carry", None)
        q_in0 = carry.pop("q_in", None) if carry is not None else None     # valid for THIS layer's input only
        tsa_ss = kwargs.pop("tsa_spatial_shapes", None)
        tsa_lsi = kwargs.pop("tsa_level_start_index", None)
        if tsa_ss is None:                                    # (the reference rebuilds these per call)
            tsa_ss = torch.tensor([[bev_h, bev_w]], device=query.device)
            tsa_lsi = torch.tensor([0], device=query.device)
        i = 0
        resid = None      # alias of `query` for the next fused block's residual connection (see _fused_norm)
        while i < len(order):
            op = order[i]
            fuse = (not self.pre_norm) and i + 1 < len(order) and order[i + 1] == "norm" and query.is_cuda
            # the norm closing this block feeds another block + its residual: ask for the alias pair
            twin = (fuse and i + 2 < len(order) and order[i + 2] in ("cross_attn", "ffn")
                    and torch.is_grad_enabled())
            res_in, resid = (query if resid is None else resid), None
            if op == "self_attn":
                att = self.attentions[ai]
                if fuse and isinstance(att, TemporalSelfAttention) and att.batch_first:
                    q_in = q_in0 if i == 0 else None
                    pre = att.attend(query, prev_bev, bev_pos, query_key_padding_mask, ref_2d,
                                     tsa_ss, tsa_lsi, q_in=q_in,
                                     bev_hw=None if bev_h is None else (bev_h, bev_w),
                                     value_pre=kwargs.get("tsa_value_pre"),
                                     prev_no_grad=bool(kwargs.get("tsa_prev_no_grad", False)))
                    query = _fused_norm(self.norms[ni], pre, res_in, att.dropout, twin=twin)
                    if twin:
                        query, resid = query
                    ni += 1
                    i += 1
                else:
                    query = att(query, prev_bev, prev_bev, identity if self.pre_norm else None,
                                query_pos=bev_pos, key_pos=bev_pos, attn_mask=masks[ai],
                                key_padding_mask=query_key_padding_mask, reference_points=ref_2d,
                                spatial_shapes=tsa_ss, level_start_index=tsa_lsi, **kwargs)
                ai += 1
                identity = query
            elif op == "cross_attn":
                att = self.attentions[ai]
                if fuse and isinstance(att, SpatialCrossAttention) and query_pos is None:
                    pre = att.attend(query, value if value is not None else key, reference_points_cam,
                                     kwargs.get("bev_mask"), spatial_shapes, level_start_index,
                                     kwargs.get("sca_plan"), kwargs.get("level_hw_host"),
                                     kwargs.get("sca_value_pre"))
                    query = _fused_norm(self.norms[ni], pre, res_in, att.dropout, twin=twin)
                    if twin:
                        query, resid = query
                    ni += 1
                    i += 1
                else:
                    query = att(query, key, value, identity if self.pre_norm else None,
                                query_pos=query_pos, key_pos=key_pos, reference_points=ref_3d,
                                reference_points_cam=reference_points_cam, mask=mask,
                                attn_mask=masks[ai], key_padding_mask=key_padding_mask,
                                spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                                **kwargs)
                ai += 1
                identity = query
            elif op == "ffn":
                ffn = self.ffns[fi]
                if (fuse and isinstance(ffn, FFN) and ffn.add_identity
                        and isinstance(ffn.dropout_layer, nn.Identity)):
                    emit = (carry is not None and carry.get("emit") and i + 2 == len(order)
                            and bev_pos is not None and bev_pos.dtype == query.dtype)
                    out = _fused_norm(self.norms[ni], ffn.transform(query), res_in,
                                      ffn.layers[ffn.num_fcs], bev_pos if emit else None,
                                      twin=twin and not emit)
                    if emit:
                        query, carry["q_in"] = out
                    elif twin:
                        query, resid = out
                    else:
                        query = out
                    ni += 1
                    i += 1
                else:
                    query = ffn(query, identity if self.pre_norm else None)
                fi += 1
            else:   # a norm that is not fused with the block before it
                query = _fused_norm(self.norms[ni], query, None) if query.is_cuda else self.norms[ni](query)
                ni += 1
            i += 1
        return query


def key_padding_free(kwargs) -> bool:
    """No key-padding mask in play (the shared value projections skip the per-layer masked_fill)."""
    return kwargs.get("key_padding_mask") is None and kwargs.get("query_key_padding_mask") is None


class BEVFormerEncoder(nn.Module):
    """The stack of BEVFormerLayers plus the once-per-forward geometry (encoder.py:24-239).
    Also stands in for mmcv's TransformerLayerSequence (deep-copies the layer config num_layers
    times into ``self.layers``)."""

    def __init__(self, *args, transformerlayers=None, num_layers=None, pc_range=None,
                 num_points_in_pillar=4, return_intermediate=False, dataset_type="nuscenes",
                 init_cfg=None, **kwargs):
        super().__init__()
        if args:   # positional (transformerlayers, num_layers) as TransformerLayerSequence allows
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
        self.num_points_in_pillar = num_points_in_pillar
        self.pc_range = pc_range
        self.fp16_enabled = False

    # ---- geometry --------------------------------------------------------------------------------
    @staticmethod
    def get_reference_points(H, W, Z=8, num_points_in_pillar=4, dim="3d", bs=1, device="cuda",
                             dtype=torch.float):
        """Pillar anchors (bs, D, H*W, 3) for dim='3d', BEV grid (bs, H*W, 1, 2) for '2d', both
        normalised to [0, 1] with q = i*W + j (encoder.py:46-85)."""
        xs = torch.linspace(0.5, W - 0.5, W, dtype=dtype, device=device) / W
        ys = torch.linspace(0.5, H - 0.5, H, dtype=dtype, device=device) / H
        if dim == "3d":
            zs = torch.linspace(0.5, Z - 0.5, num_points_in_pillar, dtype=dtype, device=device) / Z
            d = num_points_in_pillar
            pts = torch.stack([xs.view(1, 1, W).expand(d, H, W), ys.view(1, H, 1).expand(d, H, W),
                               zs.view(d, 1, 1).expand(d, H, W)], -1)
            return pts.reshape(1, d, H * W, 3).repeat(bs, 1, 1, 1)
        if dim == "2d":
            grid = torch.stack([xs.view(1, W).expand(H, W), ys.view(H, 1).expand(H, W)], -1)
            return grid.reshape(1, H * W, 1, 2).repeat(bs, 1, 1, 1)
        raise ValueError(dim)

    def point_sampling(self, reference_points, pc_range, img_metas):
        """Generic projection of arbitrary reference points (encoder.py:88-149), kept for API
        compatibility; ``forward`` uses the fused kernel for the canonical pillar grid."""
        l2i = reference_points.new_tensor(np.asarray([m["lidar2img"] for m in img_metas])).float()
        ext = [pc_range[3] - pc_range[0], pc_range[4] - pc_range[1], pc_range[5] - pc_range[2]]
        pts = torch.stack([reference_points[..., k] * ext[k] + pc_range[k] for k in range(3)], -1)
        pts = torch.cat([pts, torch.ones_like(pts[..., :1])], -1).float()       # (B, D, Nq, 4)
        b, d, nq = pts.shape[:3]
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            cam = torch.matmul(l2i.view(1, b, -1, 1, 4, 4),
                               pts.permute(1, 0, 2, 3).reshape(d, b, 1, nq, 4, 1)).squeeze(-1)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
        cam = cam.permute(2, 1, 3, 0, 4)                                        # (cam, B, Nq, D, 4)
        eps = 1e-5
        depth = cam[..., 2:3]
        xy = cam[..., :2] / torch.clamp(depth, min=eps)
        h, w = img_metas[0]["img_shape"][0][0], img_metas[0]["img_shape"][0][1]
        xy = torch.stack([xy[..., 0] / w, xy[..., 1] / h], -1)
        mask = ((depth > eps) & (xy[..., 1:2] > 0.0) & (xy[..., 1:2] < 1.0)
                & (xy[..., 0:1] < 1.0) & (xy[..., 0:1] > 0.0)).squeeze(-1)
        return xy, mask

    def _camera_geometry(self, bs, bev_h, bev_w, img_metas, device, lidar2img=None, raw_mask=False):
        """reference_points_cam (cam, bs, Nq, D, 2) f32 and bev_mask (cam, bs, Nq, D) through the fused
        projection kernel (replaces get_reference_points('3d') + point_sampling).  ``lidar2img``: an
        already-resident (bs, cam, 4, 4) f32 device tensor (what a CUDA-graph-captured step reads, refreshed
        by the caller every frame); otherwise the matrices are copied from ``img_metas``."""
        if lidar2img is None:
            l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in img_metas], dtype=np.float32))
            l2i = l2i.to(device, non_blocking=True).contiguous()                # (B, cam, 4, 4)
        else:
            l2i = lidar2img.to(device=device, dtype=torch.float32).contiguous()
        z_extent = self.pc_range[5] - self.pc_range[2]
        z_norm = (torch.linspace(0.5, z_extent - 0.5, self.num_points_in_pillar) / z_extent).tolist()
        h, w = img_metas[0]["img_shape"][0][0], img_metas[0]["img_shape"][0][1]   # quirk 10
        return ops.point_sampling(l2i, self.pc_range, z_norm, h, w, bev_h, bev_w, raw_mask=raw_mask)

    def prepare(self, img_metas, bev_h, bev_w, device, lidar2img=None) -> ScaPlan:
        """Everything of a forward that depends only on the camera rig: pillar projection, in-view mask,
        the (camera, query) pair plan -- all on the device.  The first call for a BEV size synchronises
        ONCE to size the pair list (capacity = pairs found + 15 %); every later call, and every call made
        while a CUDA graph is being captured, is sync-free.  ``forward`` calls this itself unless a plan
        is passed as ``sca_plan=``."""
        device = torch.device(device)
        bs = len(img_metas)
        ref_cam, mask = self._camera_geometry(bs, bev_h, bev_w, img_metas, device, lidar2img, raw_mask=True)
        cache = self.__dict__.setdefault("_plan_cache", {})
        key = (bev_h, bev_w, str(device))
        if key not in cache:
            cache[key] = dict(qorder=ScaPlan.tile_order(bev_h, bev_w, device), capacity=None, last=None)
        ent = cache[key]
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:                  # (event queries are not allowed while a capture is active)
            self._poll_plan(ent)
        if ent["capacity"] is None:
            if capturing:
                raise RuntimeError("BEVFormerEncoder: run one eager forward (or prepare()) before capturing a "
                                   "CUDA graph, so that the SCA pair list can be sized")
            found = int((mask[:, 0] != 0).any(-1).sum())            # the one calibration sync
            ent["capacity"] = max(256, -(-int(found * 1.15 + 64) // 256) * 256)
        plan = ScaPlan.build_device(mask, ref_cam, ent["qorder"], ent["capacity"])
        if not capturing:
            # overflow is checked WITHOUT blocking: the counters travel to pinned memory behind an event
            # and are looked at by the next prepare() / check_plan()
            host = torch.empty(2, dtype=torch.int32, pin_memory=True)
            host.copy_(plan.counters, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(device))
            ent["last"] = (ev, host)
        return plan

    @staticmethod
    def _poll_plan(ent, wait=False):
        last = ent.get("last")
        if last is None:
            return
        ev, host = last
        if wait:
            ev.synchronize()
        if not ev.query():
            return
        ent["last"] = None
        found, over = int(host[0]), int(host[1])
        if over:
            cap = ent["capacity"]
            ent["capacity"] = max(256, -(-int(found * 1.15 + 64) // 256) * 256)
            raise RuntimeError(f"BEVFormerEncoder: the camera rig put {found} (camera, query) pairs in view, more "
                               f"than the pair-list capacity {cap}; the previous forward dropped the excess. "
                               f"Capacity is now {ent['capacity']}: re-run the step (re-capture a captured graph)")

    def check_plan(self, plan: Optional[ScaPlan] = None) -> Optional[int]:
        """Blocking check of the pair-list capacity (tests, end of an epoch, after graph replays): raises
        if a forward overflowed; returns the pair count of ``plan`` when one is given."""
        for ent in self.__dict__.get("_plan_cache", {}).values():
            self._poll_plan(ent, wait=True)
        if plan is not None and plan.counters is not None:
            found, over = (int(v) for v in plan.counters.tolist())
            if over:
                raise RuntimeError(f"SCA pair list overflow: {found} pairs > capacity {plan.num_pairs}")
            return found
        return None

    def enable_grad_arena(self, overlap: bool = False):
        """Opt in to the flat gradient arena (bevformer_b200/arena.py): every parameter gradient of the
        encoder accumulates in one fp32 buffer (one memset per backward pass), is converted once at the end
        of the pass and handed out as views (``p.grad``).  Gradients are then OVERWRITTEN by each backward
        pass.  Call after the module sits on its device / dtype; returns the arena (its ``flat_grad(dtype)``
        is the bucket a data-parallel all-reduce can use directly).  ``overlap``: issue the weight-gradient
        GEMMs on a side stream (they feed nothing but the arena), joined at the end of the backward pass."""
        from ..arena import GradArena
        seen, groups = set(), []
        for mod in self.modules():
            so, aw = getattr(mod, "sampling_offsets", None), getattr(mod, "attention_weights", None)
            if isinstance(so, nn.Linear) and isinstance(aw, nn.Linear):     # projected as one stacked matrix
                for grp in ([so.weight, aw.weight], [so.bias, aw.bias]):
                    if all(id(p) not in seen for p in grp):
                        groups.append(grp)
                        seen.update(id(p) for p in grp)
        for p in self.parameters():
            if id(p) not in seen:
                groups.append([p])
                seen.add(id(p))
        self._grad_arena = GradArena(groups)
        if overlap:
            prio = int(os.environ.get("BEVF_SIDE_PRIORITY", "0"))
            self._grad_arena.side_stream = torch.cuda.Stream(self._grad_arena.acc.device, priority=prio)
            ops.AUX_STREAM[torch.device(self._grad_arena.acc.device)] = self._grad_arena.side_stream
        return self._grad_arena

    def _level_shapes_host(self, spatial_shapes):
        """[(h, w), ...] as python ints, for ops.gv_mode_for and the dense sampler backward.  Lists / CPU tensors
        are read directly; a device tensor is read ONCE (one sync, never during a graph capture) and
        remembered by its storage address -- safe to go stale, because the sampler backward re-checks the
        shapes against the device tensor and leaves the levels to the reduction path on a mismatch."""
        if not torch.is_tensor(spatial_shapes):
            return [(int(h), int(w)) for h, w in spatial_shapes]
        if not spatial_shapes.is_cuda:
            return [(int(h), int(w)) for h, w in spatial_shapes.tolist()]
        cache = self.__dict__.setdefault("_ss_host_cache", {})
        key = (spatial_shapes.data_ptr(), tuple(spatial_shapes.shape), str(spatial_shapes.device))
        if key not in cache:
            if torch.cuda.is_current_stream_capturing():
                return None
            cache[key] = [(int(h), int(w)) for h, w in spatial_shapes.tolist()]
        return cache[key]

    def _constants(self, bev_h, bev_w, bs, dev):
        """Small device tensors that never change for a BEV size (built once: creating a tensor from
        Python numbers is a pageable host copy, which a stream capture does not allow)."""
        key = (bev_h, bev_w, bs, str(dev))
        cache = self.__dict__.setdefault("_const_cache", {})
        if key not in cache:
            ref_2d = self.get_reference_points(bev_h, bev_w, dim="2d", bs=bs, device=dev,
                                               dtype=torch.float32)
            cache[key] = (ref_2d, torch.tensor([[bev_h, bev_w]], device=dev, dtype=torch.int64),
                          torch.zeros(1, device=dev, dtype=torch.int64))
        return cache[key]

    # ---- forward ---------------------------------------------------------------------------------
    @precision.entry("bev_query", "key", "value", "bev_pos", "prev_bev")
    def forward(self, bev_query, key, value, *args, bev_h=None, bev_w=None, bev_pos=None,
                spatial_shapes=None, level_start_index=None, valid_ratios=None, prev_bev=None,
                shift=0.0, **kwargs):
        """bev_query / bev_pos / prev_bev (Nq, bs, C); key = value (num_cams, S, bs, C);
        returns (bs, Nq, C), or (num_layers, bs, Nq, C) with return_intermediate
        (same contract as encoder.py:151-239).  Under autocast, or with ``fp16_enabled``, the activations are
        cast once to the compute dtype (bevformer_b200.precision) and the result is returned in it."""
        bs = bev_query.size(1)
        dev, dtype = bev_query.device, bev_query.dtype
        ref_2d, tsa_ss, tsa_lsi = self._constants(bev_h, bev_w, bs, dev)
        plan = kwargs.pop("sca_plan", None)
        l2i_dev = kwargs.pop("lidar2img", None)        # optional device-resident (bs, cam, 4, 4) matrices
        bev_mask = None
        if plan is None:
            if dev.type != "cuda":
                raise RuntimeError("BEVFormerEncoder: inputs must be CUDA tensors (bevformer_b200 has no CPU path)")
            plan = self.prepare(kwargs["img_metas"], bev_h, bev_w, dev, l2i_dev)
        ref_cam = plan.ref_cam
        if self.training and dev.type == "cuda":
            ops.advance_seed(dev)                 # new dropout masks this step (also under graph replay)

        shift = torch.as_tensor(shift, device=dev, dtype=torch.float32)
        shift_ref = ref_2d + (shift[:, None, None, :] if shift.dim() == 2 else shift)   # quirk 9
        query = bev_query.permute(1, 0, 2)
        pos = bev_pos.permute(1, 0, 2)
        nq = query.shape[1]
        if prev_bev is not None:   # quirk 8: the queue pairs prev_bev with the LAYER-0 input query
            queue = torch.stack([prev_bev.permute(1, 0, 2), query], 1).reshape(bs * 2, nq, -1)
            hybrid = torch.stack([shift_ref, ref_2d], 1).reshape(bs * 2, nq, 1, 2)
        else:
            queue = None
            hybrid = torch.stack([ref_2d, ref_2d], 1).reshape(bs * 2, nq, 1, 2)
        hybrid = hybrid.contiguous()
        hw_host = kwargs.pop("level_hw_host", None) or self._level_shapes_host(spatial_shapes)
        ss = torch.as_tensor(spatial_shapes).to(device=dev, dtype=torch.int64).contiguous()
        lsi = torch.as_tensor(level_start_index).to(device=dev, dtype=torch.int64).contiguous()

        # Every layer projects the SAME camera features (SCA value_proj) and the SAME BEV queue (TSA
        # value_proj): all of those projections are issued here as one autograd node per shared input, whose
        # backward chains the input gradients through the GEMM epilogue (plugin/linear.py)
        sca_pre = tsa_pre = None
        fusable = [l for l in self.layers if isinstance(l, BEVFormerLayer) and not l.pre_norm
                   and len(l.attentions) == 2 and isinstance(l.attentions[0], TemporalSelfAttention)
                   and isinstance(l.attentions[1], SpatialCrossAttention)]
        if (len(fusable) == len(self.layers) and dev.type == "cuda" and dtype in ops.TC_DTYPES
                and key_padding_free(kwargs) and value is not None):
            ncam, s_len, c = value.shape[0], value.shape[1], value.shape[3]
            feats = value.permute(2, 0, 1, 3).reshape(bs * ncam, s_len, c)
            sca_pre = shared_input_projections(
                feats, [(l.attentions[1].deformable_attention.value_proj.weight,
                         l.attentions[1].deformable_attention.value_proj.bias) for l in self.layers])
            if queue is not None:
                tsa_pre = shared_input_projections(
                    queue, [(l.attentions[0].value_proj.weight, l.attentions[0].value_proj.bias)
                            for l in self.layers])
        prev_no_grad = prev_bev is not None and bs == 1 and not prev_bev.requires_grad

        inter = []
        # the last LayerNorm of layer i also writes (output + bev_pos), the query the temporal
        # self-attention of layer i+1 starts from: no separate add forward, and the two gradients of
        # the output are summed inside the LayerNorm backward kernel
        carry = {} if (dev.type == "cuda" and not self.pre_norm) else None
        for li, layer in enumerate(self.layers):
            if carry is not None:
                carry["emit"] = li + 1 < len(self.layers) and isinstance(layer, BEVFormerLayer)
                if not isinstance(layer, BEVFormerLayer):
                    carry.pop("q_in", None)
            extra = dict(pos_carry=carry) if isinstance(layer, BEVFormerLayer) else {}
            if sca_pre is not None:
                extra["sca_value_pre"] = sca_pre[li]
            if tsa_pre is not None:
                extra["tsa_value_pre"] = tsa_pre[li]
            if isinstance(layer, BEVFormerLayer):
                extra["tsa_prev_no_grad"] = prev_no_grad
            query = layer(query, key, value, *args, bev_pos=pos, ref_2d=hybrid, ref_3d=None,
                          bev_h=bev_h, bev_w=bev_w, spatial_shapes=ss, level_start_index=lsi,
                          reference_points_cam=ref_cam, bev_mask=bev_mask, prev_bev=queue,
                          sca_plan=plan, level_hw_host=hw_host, tsa_spatial_shapes=tsa_ss,
                          tsa_level_start_index=tsa_lsi,
                          **extra, **kwargs)
            if self.return_intermediate:
                inter.append(query)
        return torch.stack(inter) if self.return_intermediate else query


_register(TRANSFORMER_LAYER, MyCustomBaseTransformerLayer)
_register(TRANSFORMER_LAYER, BEVFormerLayer)
_register(TRANSFORMER_LAYER_SEQUENCE, BEVFormerEncoder)
