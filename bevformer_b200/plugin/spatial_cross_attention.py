"""SpatialCrossAttention / MSDeformableAttention3D on the CUDA kernels.

Drop-ins for the reference classes of the same names
(projects/mmdet3d_plugin/bevformer/modules/spatial_cross_attention.py:31-175 and :178-399): same
registry names, constructor arguments, parameter names/shapes, forward signatures.

What changes is the execution plan.  The reference finds the queries each camera sees with
``nonzero()`` (a host sync per layer), copies them into zero-padded ``(bs, num_cams, max_len, C)``
tensors with Python loops, runs the op on the padded batch and scatters back (:138-172).  Here a
``ScaPlan`` -- the compact list of in-view (camera, query) pairs -- is built once per encoder
forward (one sync, or none when the caller passes a cached plan); per layer the sampling offsets
and attention logits are produced for every BEV query exactly once (they do not depend on the
camera), and the sampler runs over the pair list in a single launch with no padding rows.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from .. import ops, precision
from .linear import _use_tc as use_tc, linear, sca_head_sampler, sca_sampling_head, stacked_head
from .registry import ATTENTION, _register, build_attention
from .temporal_self_attention import _check_head_dim, ring_offsets_


@dataclass
class ScaPlan:
    """In-view (camera, query) pairs of one encoder forward, camera-major then query-ascending
    (the order of the reference's per-camera index lists)."""
    pair_cam: torch.Tensor      # (R,) int32
    pair_q: torch.Tensor        # (R,) int32
    pair_of: torch.Tensor       # (ncam, Nq) int32: pair row of (cam, q) or -1
    inv_count: torch.Tensor     # (bs, Nq) f32: 1 / max(1, #cameras seeing q)   (per batch item)
    row_map: torch.Tensor       # (bs*R,) int32: value map (b*ncam + cam) of every sampler row
    ref_cam: torch.Tensor       # (ncam, bs, Nq, D, 2) f32
    num_pairs: int              # rows of the pair list (== its capacity for a device-built plan)
    counters: Optional[torch.Tensor] = None   # device-built plans: int32 [pairs found, overflow flag]
    map_range: Optional[torch.Tensor] = None  # (bs*ncam, 2) int32: [first, end) sampler rows of every value map

    @staticmethod
    def build(bev_mask: torch.Tensor, reference_points_cam: torch.Tensor, bev_hw=None,
              tile: int = 8) -> "ScaPlan":
        """bev_mask (ncam, bs, Nq, D) bool.  Quirk 1 (SURVEY.md App. D): the pair list comes from
        batch item 0's mask for every batch item (:139), the divisor from each item's own mask
        (:169-171).  With ``bev_hw`` the pairs of each camera are ordered in tile x tile BEV patches
        (row-major inside a patch) instead of plain row-major: the sampler's CTAs then work on compact
        patches whose image footprints overlap in L1.  The order is immaterial to the result (the
        combine step gathers through ``pair_of``)."""
        ncam, bs, nq, _ = bev_mask.shape
        seen = bev_mask.any(-1)                                 # (ncam, bs, Nq)
        hit0 = seen[:, 0]
        nz = hit0.nonzero()                                     # the one host sync (sizes the lists)
        r = int(nz.shape[0])
        if bev_hw is not None and tile > 1 and os.environ.get("BEVF_SCA_TILE", "1") != "0":
            h, w = bev_hw
            qi, qj = nz[:, 1] // w, nz[:, 1] % w
            tiles_x = (w + tile - 1) // tile
            key = ((nz[:, 0] * ((h + tile - 1) // tile) + qi // tile) * tiles_x + qj // tile) * (tile * tile) \
                + (qi % tile) * tile + qj % tile
            nz = nz[torch.argsort(key)]
        pair_cam = nz[:, 0].to(torch.int32).contiguous()
        pair_q = nz[:, 1].to(torch.int32).contiguous()
        pair_of = torch.full((ncam, nq), -1, dtype=torch.int32, device=bev_mask.device)
        pair_of[pair_cam.long(), pair_q.long()] = torch.arange(r, dtype=torch.int32, device=bev_mask.device)
        inv_count = 1.0 / seen.sum(0).clamp(min=1).to(torch.float32)
        row_map = (torch.arange(bs, device=bev_mask.device, dtype=torch.int32)[:, None] * ncam
                   + pair_cam[None, :]).reshape(-1).contiguous()
        per_cam = torch.bincount(pair_cam.long(), minlength=ncam)
        ends = per_cam.cumsum(0)
        rng = torch.stack([ends - per_cam, ends], 1)                                  # (ncam, 2)
        map_range = (rng[None] + (torch.arange(bs, device=rng.device) * r)[:, None, None]).reshape(-1, 2)
        return ScaPlan(pair_cam, pair_q, pair_of, inv_count.contiguous(), row_map,
                       reference_points_cam.float().contiguous(), r, None,
                       map_range.to(torch.int32).contiguous())


    @staticmethod
    def tile_order(bev_h: int, bev_w: int, device, tile: int = 8) -> torch.Tensor:
        """(Nq,) int32: the BEV queries in tile x tile patches (row-major inside a patch) -- the order of
        the queries inside each camera's pair list.  Depends on the BEV size only."""
        qi = torch.arange(bev_h, device=device).view(bev_h, 1).expand(bev_h, bev_w).reshape(-1)
        qj = torch.arange(bev_w, device=device).view(1, bev_w).expand(bev_h, bev_w).reshape(-1)
        tiles_x = (bev_w + tile - 1) // tile
        key = ((qi // tile) * tiles_x + qj // tile) * (tile * tile) + (qi % tile) * tile + qj % tile
        return torch.argsort(key, stable=True).to(torch.int32).contiguous()

    @staticmethod
    def build_device(mask_u8: torch.Tensor, reference_points_cam: torch.Tensor, qorder, capacity: int) -> "ScaPlan":
        """Same plan as ``build`` (same pairs, same order when ``qorder`` is the tile order), produced by
        three small kernels with NO host synchronisation: the lists have a fixed ``capacity`` and unused
        rows are marked -1, which every row-list kernel skips.  Capturable in a CUDA graph; replaying the
        graph with a new lidar2img rebuilds the list for that frame.  ``counters`` = [pairs found, overflow]
        stays on the device -- see BEVFormerEncoder.check_plan()."""
        t = ops.sca_plan_build(mask_u8, qorder, capacity)
        return ScaPlan(t["pair_cam"], t["pair_q"], t["pair_of"], t["inv_count"], t["row_map"],
                       reference_points_cam.float().contiguous(), int(capacity), t["counters"], t["map_range"])


class MSDeformableAttention3D(nn.Module):
    """Holder of SCA's per-camera deformable-attention parameters (value_proj, sampling_offsets,
    attention_weights; no output_proj -- it lives in SpatialCrossAttention, :67,221) and, for
    callers that use it on its own, the reference's dense forward."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=8, im2col_step=64,
                 dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__()
        _check_head_dim(embed_dims, num_heads)
        self.init_cfg = init_cfg
        self.norm_cfg = norm_cfg
        self.batch_first = batch_first
        self.output_proj = None
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weights()

    def init_weights(self):
        nn.init.zeros_(self.sampling_offsets.weight)
        ring_offsets_(self.sampling_offsets.bias, self.num_heads, self.num_levels, self.num_points)
        nn.init.zeros_(self.attention_weights.weight)
        nn.init.zeros_(self.attention_weights.bias)
        nn.init.xavier_uniform_(self.value_proj.weight)
        nn.init.zeros_(self.value_proj.bias)
        self._is_init = True

    def head_weights(self, x):
        """sampling_offsets and attention_weights stacked into one projection (applied to ``x``)."""
        ws, bs_ = (self.sampling_offsets.weight, self.attention_weights.weight), \
                  (self.sampling_offsets.bias, self.attention_weights.bias)
        return stacked_head(ws, bs_, x)

    @precision.entry("query", "key", "value", "identity", "query_pos")
    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, **kwargs):
        """Dense form (:273-399): query (bs, Nq, C), value (bs, S, C), reference_points
        (bs, Nq, D, 2) -> (bs, Nq, C); no identity add, no output projection."""
        if value is None:
            value = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, nq, _ = query.shape
        nv = value.shape[1]
        m, l, p = self.num_heads, self.num_levels, self.num_points
        if reference_points.shape[-1] == 4:
            raise AssertionError("box-form reference points are not supported here")   # :374-375
        if reference_points.shape[-1] != 2:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, "
                             f"but get {reference_points.shape[-1]} instead.")
        v = linear(value, self.value_proj.weight, self.value_proj.bias)
        if key_padding_mask is not None:
            v = v.masked_fill(key_padding_mask[..., None], 0.0)
        v = v.view(bs, nv, m, -1)
        w, b = self.head_weights(query)
        ss = torch.as_tensor(spatial_shapes).to(device=query.device, dtype=torch.int64)
        lsi = torch.as_tensor(level_start_index).to(device=query.device, dtype=torch.int64)
        d = reference_points.shape[2]
        # every (batch, query) row is its own "pair" of a one-camera plan
        dev = query.device
        ref = reference_points.reshape(1, bs, nq, d, 2).float().contiguous()
        pair_q = torch.arange(nq, device=dev, dtype=torch.int32)
        pair_cam = torch.zeros(nq, device=dev, dtype=torch.int32)
        pair_of = pair_q.view(1, nq).contiguous()
        loc, attn = sca_sampling_head(query, w, b, ref, pair_q, pair_cam, pair_of, ss.contiguous(),
                                      bs, nq, m, l, p)
        out = ops.MultiScaleDeformableAttnFunction_fp32.apply(
            v, ss, lsi, loc.view(bs, nq, m, l, p, 2), attn.view(bs, nq, m, l, p), self.im2col_step)
        return out if self.batch_first else out.permute(1, 0, 2)


class SpatialCrossAttention(nn.Module):
    """Each BEV query gathers from the cameras that see its pillar (reference :31-175)."""

    def __init__(self, embed_dims=256, num_cams=6, pc_range=None, dropout=0.1, init_cfg=None,
                 batch_first=False,
                 deformable_attention=dict(type="MSDeformableAttention3D", embed_dims=256,
                                           num_levels=4),
                 **kwargs):
        super().__init__()
        self.init_cfg = init_cfg
        self.dropout = nn.Dropout(dropout)
        self.pc_range = pc_range
        self.fp16_enabled = False
        self.deformable_attention = build_attention(deformable_attention)
        self.embed_dims = embed_dims
        self.num_cams = num_cams
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.batch_first = batch_first
        self.init_weight()

    def init_weight(self):
        nn.init.xavier_uniform_(self.output_proj.weight)
        nn.init.zeros_(self.output_proj.bias)

    def _fused_prep(self, query, w, v, gv_mode, dense) -> bool:
        """Whether the sampler computes the sampling points itself (plugin/linear.py::sca_head_sampler): the 16-bit
        tensor-core head, 8 heads of 32 channels and 32 samples per head, the mixed grad_value accumulation with a
        host pyramid that matches the value maps, and outside deterministic mode (its fixed-point backward reads loc /
        attn)."""
        da = self.deformable_attention
        return (isinstance(gv_mode, tuple) and dense is not None and not ops.deterministic()
                and da.num_heads == 8 and v.shape[-1] == 32 and da.num_levels * da.num_points == 32
                and use_tc(query, w) and sum(h * w_ for h, w_ in gv_mode[1]) == v.shape[1])

    def attend(self, query, value, reference_points_cam, bev_mask, spatial_shapes,
               level_start_index, plan: Optional[ScaPlan] = None, level_hw_host=None, value_pre=None):
        """Everything up to and including output_proj, WITHOUT dropout / residual.
        query (bs, Nq, C); value (num_cams, S, bs, C).  ``level_hw_host``: [(h, w), ...] python ints of
        the pyramid, when the caller knows them without a device read: the sampler backward then picks
        its grad_value accumulation per level (ops.gv_mode_for) and hands the coarse levels to the dense kernel.  ``value_pre``: value_proj(value) already computed
        by the encoder for all layers at once (plugin/linear.py::shared_input_projections)."""
        da = self.deformable_attention
        bs, nq, c = query.shape
        ncam, s = value.shape[0], value.shape[1]
        m, l, p = da.num_heads, da.num_levels, da.num_points
        if plan is None:
            plan = ScaPlan.build(bev_mask, reference_points_cam)
        d = plan.ref_cam.shape[3]
        ss = torch.as_tensor(spatial_shapes).to(device=query.device, dtype=torch.int64).contiguous()
        lsi = torch.as_tensor(level_start_index).to(device=query.device, dtype=torch.int64).contiguous()
        if int(s) <= 0 or p % d != 0:
            raise AssertionError("num_points must be a multiple of the pillar anchors")   # :369
        # offsets / logits once per BEV query: they do not depend on the camera (:338-341)
        w, b = da.head_weights(query)
        # value_proj over every camera's feature pyramid (:334), batch-major like the reference
        if value_pre is None:
            feats = value.permute(2, 0, 1, 3).reshape(bs * ncam, s, c)
            value_pre = linear(feats, da.value_proj.weight, da.value_proj.bias)
        if getattr(value_pre, "_bevf_ready", None) is not None:       # produced on the second stream
            torch.cuda.current_stream(value_pre.device).wait_event(value_pre._bevf_ready)
        v = value_pre.view(bs * ncam, s, m, -1)
        if hasattr(value_pre, "_bevf_early"):
            v._bevf_early = value_pre._bevf_early
        dense = None
        if level_hw_host is not None and plan.map_range is not None and len(level_hw_host) == l:
            dense = (level_hw_host, plan.map_range)
        # grad_value of the fine pyramid levels accumulated in scaled fp16, the coarse ones in fp32 (ops.gv_mode_for),
        # those in between in replicated scaled-fp16 copies (ops.gv_replicas_for)
        gv_mode = None
        if level_hw_host is not None and len(level_hw_host) == l and v.dtype == torch.bfloat16:
            rows_per_map = plan.row_map.numel() / max(1, bs * ncam)
            gv_mode = ops.gv_mode_for(rows_per_map, p, level_hw_host)
            if isinstance(gv_mode, tuple):
                gv_mode = gv_mode + (ops.gv_replicas_for(rows_per_map, p, level_hw_host),)
        if self._fused_prep(query, w, v, gv_mode, dense):
            # the sampling-point prep inside the sampler kernels: loc / attn never go through memory
            fuse = (plan.ref_cam, plan.pair_q, plan.pair_cam, plan.pair_of, plan.row_map, ss, lsi, bs, nq,
                    gv_mode[1], gv_mode[2], plan.map_range, gv_mode[3])
            out = sca_head_sampler(query, w, b, v, fuse)                                      # (bs*R, C)
        else:
            loc, attn = sca_sampling_head(query, w, b, plan.ref_cam, plan.pair_q, plan.pair_cam,
                                          plan.pair_of, ss, bs, nq, m, l, p)
            out = ops.SamplerRows.apply(v, loc, attn, plan.row_map, ss, lsi, None, dense, gv_mode)   # (bs*R, C)
        slots = ops.ScaCombine.apply(out, plan.pair_of, plan.pair_q, plan.inv_count, bs, nq)
        return linear(slots, self.output_proj.weight, self.output_proj.bias)

    @precision.entry("query", "key", "value", "residual", "query_pos")
    def forward(self, query, key, value, residual=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, reference_points_cam=None,
                bev_mask=None, level_start_index=None, flag="encoder", **kwargs):
        """Same contract as the reference forward (:76-175): (bs, Nq, C) in, (bs, Nq, C) out =
        dropout(output_proj(camera-mean of sampled features)) + residual."""
        if key is None:
            key = query
        if value is None:
            value = key
        inp_residual = query if residual is None else residual
        if query_pos is not None:
            query = query + query_pos
        out = self.attend(query, value, reference_points_cam, bev_mask, spatial_shapes,
                          level_start_index, kwargs.get("sca_plan"))
        return self.dropout(out) + inp_residual


_register(ATTENTION, MSDeformableAttention3D)
_register(ATTENTION, SpatialCrossAttention)
