"""TemporalSelfAttention on the CUDA kernels.

Drop-in for the reference class of the same name
(projects/mmdet3d_plugin/bevformer/modules/temporal_self_attention.py:25-272): same registry name,
constructor arguments and defaults, parameter names/shapes (so published checkpoints load), forward
signature and return convention.  The arithmetic is re-organised around three launches of
``libbevformer_b200.so`` (sampling-point prep, sampler, and -- in the layer -- residual+LayerNorm)
bracketed by the dense projections of ``plugin/linear.py``.
"""
from __future__ import annotations

import math
import os
import warnings

import torch
import torch.nn as nn

from .. import ops, precision
from .linear import linear, linear_fp32_out, stacked_head, tsa_sampling_head
from .registry import ATTENTION, _register


def ring_offsets_(bias: torch.Tensor, num_heads: int, groups: int, num_points: int) -> None:
    """Fill a sampling_offsets bias with the reference initialiser: head m looks along angle
    2*pi*m/num_heads (scaled so the larger component is 1), point i sits at radius i+1
    (temporal_self_attention.py:109-122, spatial_cross_attention.py:255-267)."""
    ang = torch.arange(num_heads, dtype=torch.float32) * (2.0 * math.pi / num_heads)
    unit = torch.stack([ang.cos(), ang.sin()], -1)
    unit = unit / unit.abs().max(-1, keepdim=True)[0]
    radius = torch.arange(1, num_points + 1, dtype=torch.float32).view(1, 1, num_points, 1)
    grid = unit.view(num_heads, 1, 1, 2) * radius
    with torch.no_grad():
        bias.copy_(grid.expand(num_heads, groups, num_points, 2).reshape(-1))


def _check_head_dim(embed_dims: int, num_heads: int) -> int:
    if embed_dims % num_heads != 0:
        raise ValueError(f"embed_dims must be divisible by num_heads, "
                         f"but got {embed_dims} and {num_heads}")
    d = embed_dims // num_heads
    if d & (d - 1):
        warnings.warn("head dimension is not a power of two; the sampler falls back to its "
                      "generic (slower) kernel unless head_dim == 32")
    return d


class TemporalSelfAttention(nn.Module):
    """Deformable self-attention over the 2-frame BEV queue [previous BEV, current BEV]."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, num_bev_queue=2,
                 im2col_step=64, dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__()
        _check_head_dim(embed_dims, num_heads)
        self.init_cfg = init_cfg
        self.norm_cfg = norm_cfg
        self.batch_first = batch_first
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.num_bev_queue = num_bev_queue
        self.dropout = nn.Dropout(dropout)
        q = num_bev_queue
        self.sampling_offsets = nn.Linear(embed_dims * q, q * num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims * q, q * num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weights()

    def init_weights(self):
        nn.init.zeros_(self.sampling_offsets.weight)
        ring_offsets_(self.sampling_offsets.bias, self.num_heads,
                      self.num_levels * self.num_bev_queue, self.num_points)
        nn.init.zeros_(self.attention_weights.weight)
        nn.init.zeros_(self.attention_weights.bias)
        for lin in (self.value_proj, self.output_proj):
            nn.init.xavier_uniform_(lin.weight)
            nn.init.zeros_(lin.bias)
        self._is_init = True

    # -------------------------------------------------------------------------------------------
    def attend(self, query, value=None, query_pos=None, key_padding_mask=None,
               reference_points=None, spatial_shapes=None, level_start_index=None, q_in=None,
               bev_hw=None, value_pre=None, prev_no_grad=False):
        """Everything up to and including output_proj, batch-first, WITHOUT dropout / identity.
        query (bs, Nq, C); value (bs*2, Nq, C) stacked [prev, cur] or None; ``q_in`` = query +
        query_pos when the caller already has it (the encoder's previous LayerNorm emits it)."""
        assert self.num_bev_queue == 2
        bs, nq, c = query.shape
        if value is None:   # first frame: the queue is the current BEV twice (:177-180)
            value = torch.stack([query, query], 1).reshape(bs * 2, nq, c)
        nv = value.shape[1]
        if q_in is None:
            q_in = query if query_pos is None else query + query_pos
        # quirk 6: the first bs rows of the stacked queue, whatever they are for bs > 1 (:197).
        # prev_no_grad: those rows are the detached history BEV (bs == 1, prev_bev without grad): cutting the
        # edge here spares the backward a zero-filled (2, Nq, C) gradient, a copy into it and an add
        head = value[:bs].detach() if prev_no_grad else value[:bs]
        q_cat = torch.cat([head, q_in], -1)
        v = value_pre if value_pre is not None else linear(value, self.value_proj.weight, self.value_proj.bias)
        if getattr(v, "_bevf_ready", None) is not None:               # produced on the second stream
            torch.cuda.current_stream(v.device).wait_event(v._bevf_ready)
        if key_padding_mask is not None:
            v = v.masked_fill(key_padding_mask[..., None], 0.0)
        early = getattr(v, "_bevf_early", None)
        v = v.reshape(bs * 2, nv, self.num_heads, -1)
        if early is not None and key_padding_mask is None:
            v._bevf_early = early
        ws, bs_ = (self.sampling_offsets.weight, self.attention_weights.weight), \
                  (self.sampling_offsets.bias, self.attention_weights.bias)
        w, b = stacked_head(ws, bs_, q_cat)

        ss = torch.as_tensor(spatial_shapes).to(device=query.device, dtype=torch.int64)
        lsi = torch.as_tensor(level_start_index).to(device=query.device, dtype=torch.int64)
        if reference_points.shape[-1] == 2:
            ref = reference_points.reshape(bs * 2, nq, self.num_levels, 2).float().contiguous()
            lp = self.num_levels * self.num_points
            if (self.num_heads == 8 and lp in (2, 4, 8, 16, 32) and nv == nq
                    and os.environ.get("BEVF_TSA_INTERLEAVE", "1") != "0"):
                # interleaved rows (b, q, frame): the sampler writes (bs*Nq, 2C) and the mean over the
                # two frames (:257-265) is folded into the output projection as [W | W] / 2 -- no
                # reduction kernel forward, no scatter of the gradient to the two frames backward
                loc, attn = tsa_sampling_head(q_cat, w, b, ref, ss.contiguous(), bs, nq, self.num_heads,
                                              self.num_levels, self.num_points, True)
                order = None
                if bev_hw is not None and bev_hw[0] * bev_hw[1] == nq:
                    order = self._group_order(bs, int(bev_hw[0]), int(bev_hw[1]), query.device)
                # grad_value of the BEV maps accumulated in scaled fp16 when a (pixel, head) collects few contributions
                # (4 * num_points at nv == nq: 16 at base) -- ops.gv_mode_for; single level: its size is nv, no host shapes
                gv_mode = None
                if self.num_levels == 1 and v.dtype == torch.bfloat16:
                    gv_mode = ops.gv_mode_for(float(nq), self.num_points, [(1, int(nv))])
                out = ops.SamplerRows.apply(v, loc, attn, self._frame_map(bs, nq, query.device), ss, lsi,
                                            order, None, gv_mode)
                w2 = torch.cat([self.output_proj.weight, self.output_proj.weight], 1) * 0.5
                return linear(out.view(bs, nq, 2 * c), w2, self.output_proj.bias)
            loc, attn = tsa_sampling_head(q_cat, w, b, ref, ss.contiguous(), bs, nq, self.num_heads,
                                          self.num_levels, self.num_points)
        elif reference_points.shape[-1] == 4:
            raw = linear_fp32_out(q_cat, w, b).reshape(bs * nq, -1)
            loc, attn = self._box_points(raw, reference_points, bs, nq)
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, "
                             f"but get {reference_points.shape[-1]} instead.")
        out = ops.MultiScaleDeformableAttnFunction_fp32.apply(v, ss, lsi, loc, attn, self.im2col_step)
        # average of the two frames (:257-265): (a + b) / 2 with the exact factor 1/2 folded into the
        # projection weights, so the reduction is one add instead of a strided mean kernel
        out = out.view(bs, 2, nq, c)
        pair_sum = out[:, 0] + out[:, 1]
        return linear(pair_sum, self.output_proj.weight * 0.5, self.output_proj.bias)

    def _frame_map(self, bs, nq, device):
        """value-map index (b*2 + frame) of every interleaved sampler row; cached per shape."""
        key = (bs, nq, str(device))
        cache = self.__dict__.setdefault("_frame_map_cache", {})
        if key not in cache:
            r = torch.arange(bs * nq * 2, device=device, dtype=torch.int32)
            cache[key] = ((r // (2 * nq)) * 2 + (r % 2)).contiguous()
        return cache[key]

    def _group_order(self, bs, h, w, device, tile=8):
        """Permutation of the interleaved sampler rows (b, q, frame) in which 64 consecutive entries are
        one 8x8 BEV tile of one frame: the rows whose grad_value contributions the backward merges
        before they reach L2 (bevf_msda_rows_backward_ordered).  Cached per shape."""
        key = ("order", bs, h, w, str(device))
        cache = self.__dict__.setdefault("_frame_map_cache", {})
        if key not in cache:
            qi = torch.arange(h, device=device).view(h, 1).expand(h, w)
            qj = torch.arange(w, device=device).view(1, w).expand(h, w)
            tiles_x = (w + tile - 1) // tile
            tkey = ((qi // tile) * tiles_x + qj // tile) * (tile * tile) + (qi % tile) * tile + qj % tile
            q_sorted = torch.argsort(tkey.reshape(-1), stable=True)                # queries in tile order
            tile_of = (tkey.reshape(-1)[q_sorted] // (tile * tile))
            # within a tile: all its queries for frame 0, then for frame 1
            k2 = (tile_of * 2).repeat_interleave(2) + torch.arange(2, device=device).repeat(h * w)
            rows = (q_sorted.repeat_interleave(2) * 2 + torch.arange(2, device=device).repeat(h * w))
            rows = rows[torch.argsort(k2, stable=True)]
            full = (torch.arange(bs, device=device).view(bs, 1) * (2 * h * w) + rows.view(1, -1)).reshape(-1)
            cache[key] = full.to(torch.int32).contiguous()
        return cache[key]

    def _box_points(self, raw, reference_points, bs, nq):
        """(cx, cy, w, h) reference boxes (:231-235); rare path, spelled with tensor ops."""
        m, l, p = self.num_heads, self.num_levels, self.num_points
        n_off = 2 * m * l * p * 2
        off = raw[:, :n_off].view(bs, nq, m, 2, l, p, 2)
        att = raw[:, n_off:].view(bs, nq, m, 2, l * p).softmax(-1).view(bs, nq, m, 2, l, p)
        off = off.permute(0, 3, 1, 2, 4, 5, 6).reshape(bs * 2, nq, m, l, p, 2)
        att = att.permute(0, 3, 1, 2, 4, 5).reshape(bs * 2, nq, m, l, p).contiguous()
        rp = reference_points.float()
        loc = rp[:, :, None, :, None, :2] + off / p * rp[:, :, None, :, None, 2:] * 0.5
        return loc.contiguous(), att

    @precision.entry("query", "key", "value", "identity", "query_pos")
    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, flag="decoder", **kwargs):
        """Same contract as the reference forward (:128-272): returns dropout(attn) + identity in
        the caller's layout ((bs, Nq, C) when batch_first)."""
        if identity is None:
            identity = query
        if not self.batch_first:
            if value is None:
                raise AssertionError("value=None requires batch_first")   # :178
            query = query.permute(1, 0, 2)
            value = value.permute(1, 0, 2)
            if query_pos is not None:
                query_pos = query_pos.permute(1, 0, 2)
        out = self.attend(query, value, query_pos, key_padding_mask, reference_points,
                          spatial_shapes, level_start_index)
        if not self.batch_first:
            out = out.permute(1, 0, 2)
        return self.dropout(out) + identity


_register(ATTENTION, TemporalSelfAttention)
