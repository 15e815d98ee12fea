"""PerceptionTransformer on the CUDA encoder and decoder.

Drop-in for the reference class of the same name (projects/mmdet3d_plugin/bevformer/modules/transformer.py:26-289):
same constructor arguments, parameter names (``level_embeds``, ``cams_embeds``, ``reference_points``,
``can_bus_mlp.*``, ``encoder.*``, ``decoder.*``), ``get_bev_features`` and ``forward`` signatures and return values.
``forward`` is ``get_bev_features`` followed by the object-query decoder (plugin/decoder.py), the same tail as
PerceptionTransformerV2; built without a ``decoder`` dict the module is the BEV encoder alone and ``forward``
raises ``NotImplementedError``.

What changes underneath: the five tensor passes that build the encoder's key/value tensor become one
kernel per pyramid level (``bevf_flatten_feats``), and the encoder is ``plugin.encoder.BEVFormerEncoder``.
The once-per-frame host arithmetic (ego-motion shift, CAN-bus MLP on an 18-vector, torchvision's
nearest-neighbour rotation of prev_bev) stays as the reference wrote it when the metas carry ``can_bus``;
with ``can_bus=`` passed as a (bs, 18) float64 CUDA tensor the same block runs in two kernels on the device
(``bevf_ego_motion``, ``bevf_rotate_bev``) and the frame has no host arithmetic left.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .. import ops, precision
from .linear import linear
from .registry import TRANSFORMER, _register, build_transformer_layer_sequence


class PerceptionTransformer(nn.Module):
    def __init__(self, num_feature_levels=4, num_cams=6, two_stage_num_proposals=300, encoder=None,
                 decoder=None, embed_dims=256, rotate_prev_bev=True, use_shift=True, use_can_bus=True,
                 can_bus_norm=True, use_cams_embeds=True, rotate_center=[100, 100], init_cfg=None,
                 **kwargs):
        super().__init__()
        self.init_cfg = init_cfg
        self.encoder = build_transformer_layer_sequence(encoder)
        self.decoder = build_transformer_layer_sequence(decoder)
        self.decoder_cfg = decoder
        self.embed_dims = embed_dims
        self.num_feature_levels = num_feature_levels
        self.num_cams = num_cams
        self.fp16_enabled = False
        self.rotate_prev_bev = rotate_prev_bev
        self.use_shift = use_shift
        self.use_can_bus = use_can_bus
        self.can_bus_norm = can_bus_norm
        self.use_cams_embeds = use_cams_embeds
        self.two_stage_num_proposals = two_stage_num_proposals
        self.rotate_center = rotate_center
        self.init_layers()
        self.init_weights()

    def init_layers(self):
        c = self.embed_dims
        self.level_embeds = nn.Parameter(torch.empty(self.num_feature_levels, c))
        self.cams_embeds = nn.Parameter(torch.empty(self.num_cams, c))
        self.reference_points = nn.Linear(c, 3)
        self.can_bus_mlp = nn.Sequential(nn.Linear(18, c // 2), nn.ReLU(inplace=True),
                                         nn.Linear(c // 2, c), nn.ReLU(inplace=True))
        if self.can_bus_norm:
            self.can_bus_mlp.add_module("norm", nn.LayerNorm(c))

    def init_weights(self):
        """transformer.py:86-101: xavier for matrices, the attention modules' own initialisers,
        N(0,1) embeddings."""
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            init = getattr(m, "init_weight", None) or (getattr(m, "init_weights", None) if m is not self else None)
            if init is not None and type(m).__name__ in ("MSDeformableAttention3D", "TemporalSelfAttention",
                                                         "CustomMSDeformableAttention"):
                init()
        nn.init.normal_(self.level_embeds)
        nn.init.normal_(self.cams_embeds)
        nn.init.xavier_uniform_(self.reference_points.weight)
        nn.init.zeros_(self.reference_points.bias)
        for m in self.can_bus_mlp:
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)

    # ---------------------------------------------------------------------------------------------
    def _shift(self, img_metas, bev_h, bev_w, grid_length):
        """Ego-motion shift in normalised BEV units, float64 on the host exactly like the reference
        (transformer.py:122-140)."""
        dx = np.array([m["can_bus"][0] for m in img_metas])
        dy = np.array([m["can_bus"][1] for m in img_metas])
        ego = np.array([m["can_bus"][-2] / np.pi * 180 for m in img_metas])
        length = np.sqrt(dx ** 2 + dy ** 2)
        bev_angle = ego - np.arctan2(dy, dx) / np.pi * 180
        sy = length * np.cos(bev_angle / 180 * np.pi) / grid_length[0] / bev_h
        sx = length * np.sin(bev_angle / 180 * np.pi) / grid_length[1] / bev_w
        return np.stack([sx * self.use_shift, sy * self.use_shift], -1)

    def _rotate_prev(self, prev_bev, img_metas, bev_h, bev_w):
        """prev_bev (Nq, bs, C) rotated by each sample's yaw delta (transformer.py:142-153).  Unlike
        the reference, the caller's tensor is left untouched (the result is a new tensor), and the
        sampling grid is always built in fp32: torchvision builds it in the image's dtype, and a
        bf16 / fp16 grid (8-11 mantissa bits for coordinates up to +-100) picks wrong source cells for
        the nearest-neighbour lookup.  The values themselves are copied, so the result is exact."""
        from torchvision.transforms.functional import rotate
        out = torch.empty_like(prev_bev)
        for i in range(prev_bev.shape[1]):
            img = prev_bev[:, i].reshape(bev_h, bev_w, -1).permute(2, 0, 1)
            img = rotate(img.float(), img_metas[i]["can_bus"][-1], center=self.rotate_center)
            out[:, i] = img.permute(1, 2, 0).reshape(bev_h * bev_w, -1).to(out.dtype)
        return out

    def get_bev_features(self, mlvl_feats, bev_queries, bev_h, bev_w, grid_length=[0.512, 0.512],
                         bev_pos=None, prev_bev=None, **kwargs):
        """mlvl_feats: per level (bs, num_cams, C, h, w); bev_queries (Nq, C); bev_pos
        (bs, C, bev_h, bev_w); prev_bev (bs, Nq, C) / (Nq, bs, C) / None; kwargs carry ``img_metas``.
        Optional ``can_bus=`` (bs, 18) float64 CUDA and ``lidar2img=`` (bs, num_cams, 4, 4) float32 CUDA replace the
        metas' entries of the same names and select the device path (``_get_bev_features_device``): same result
        (shift within one fp32 ulp, rotation cells equal except where the source coordinate sits on a rounding
        boundary), no host synchronisation, prev_bev without gradient only.
        Returns bev_embed (bs, Nq, C) in the compute dtype: the autocast dtype, fp16 with ``fp16_enabled``
        (what mmcv's auto_fp16 gives), else the features' dtype (bevformer_b200.precision)."""
        dt, amp_off = precision.entered(self, mlvl_feats[0])
        with amp_off:
            return self._get_bev_features(precision.cast(list(mlvl_feats), dt), bev_queries, bev_h, bev_w, dt,
                                          grid_length, bev_pos, prev_bev, **kwargs)

    def _get_bev_features_device(self, mlvl_feats, bev_queries, bev_h, bev_w, dt, grid_length, bev_pos, prev_bev,
                                 can_bus, ego_state=None, ego_mode=ops.EGO_DELTAS, **kwargs):
        """The frame with its ego-motion block on the device (selected by ``can_bus=`` being a CUDA tensor):
        shift, rotation operand and CAN-bus MLP input come from ``bevf_ego_motion``, prev_bev is rotated by
        ``bevf_rotate_bev``; no numpy, no ``new_tensor``, no torchvision, no host synchronisation -- with
        ``lidar2img=`` a device tensor too, the call can be captured in a CUDA graph.  ``img_metas`` is read for
        ``img_shape`` only and may be omitted once a call has seen it.  ``ego_state`` / ``ego_mode``: BEVStream's
        device-side ``prev_frame_info`` (ops.ego_motion)."""
        if not mlvl_feats[0].is_cuda:
            raise RuntimeError("PerceptionTransformer.get_bev_features: CUDA tensors required "
                               "(bevformer_b200 has no CPU path)")
        if prev_bev is not None and prev_bev.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("PerceptionTransformer.get_bev_features: the device path (can_bus= as a CUDA tensor) "
                               "takes prev_bev without gradient; for a gradient through the rotated prev_bev use "
                               "the host path (can_bus in img_metas, no can_bus= argument)")
        bs = mlvl_feats[0].size(0)
        dev = mlvl_feats[0].device
        can_bus = can_bus.to(torch.float64).reshape(bs, 18).contiguous()
        static = self.__dict__.setdefault("_static_cache", {})
        if kwargs.get("img_metas") is None:
            if ("img_shape", bs) not in static:
                raise RuntimeError("PerceptionTransformer.get_bev_features: img_metas (for img_shape) is needed on the "
                                   "first call")
            kwargs["img_metas"] = static["img_shape", bs]
        else:
            static["img_shape", bs] = [dict(img_shape=kwargs["img_metas"][0]["img_shape"])] * bs
        shapes = tuple(tuple(f.shape[-2:]) for f in mlvl_feats)
        if (shapes, str(dev)) not in static:           # small constant tensors: built once (a pageable host copy)
            ss = torch.as_tensor(shapes, dtype=torch.long, device=dev)
            static[shapes, str(dev)] = (ss, torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1])))
        spatial_shapes, level_start_index = static[shapes, str(dev)]

        shift, rot, mlp_in = ops.ego_motion(can_bus, bev_h, bev_w, grid_length, self.rotate_center, self.use_shift,
                                            bev_queries.dtype, ego_state, ego_mode)
        if prev_bev is not None:
            if self.rotate_prev_bev:
                prev_bev = ops.rotate_bev(prev_bev.detach(), rot, bev_h, bev_w, dt)
            elif prev_bev.shape[1] == bev_h * bev_w:
                prev_bev = prev_bev.permute(1, 0, 2)
        bev_queries = bev_queries.unsqueeze(1).repeat(1, bs, 1)
        bev_pos = bev_pos.flatten(2).permute(2, 0, 1)
        bev_queries = bev_queries + self.can_bus_mlp(mlp_in)[None, :, :] * self.use_can_bus
        bev_queries, bev_pos, prev_bev = (precision.cast(t, dt) for t in (bev_queries, bev_pos, prev_bev))
        feat_flatten = ops.FlattenFeats.apply(self.cams_embeds if self.use_cams_embeds else None,
                                              self.level_embeds, *mlvl_feats)
        return self.encoder(bev_queries, feat_flatten, feat_flatten, bev_h=bev_h, bev_w=bev_w, bev_pos=bev_pos,
                            spatial_shapes=spatial_shapes, level_start_index=level_start_index, prev_bev=prev_bev,
                            shift=shift, level_hw_host=[tuple(int(v) for v in s) for s in shapes], **kwargs)

    def _get_bev_features(self, mlvl_feats, bev_queries, bev_h, bev_w, dt, grid_length, bev_pos, prev_bev,
                          **kwargs):
        can_bus = kwargs.pop("can_bus", None)
        if torch.is_tensor(can_bus) and can_bus.is_cuda:
            return self._get_bev_features_device(mlvl_feats, bev_queries, bev_h, bev_w, dt, grid_length, bev_pos,
                                                 prev_bev, can_bus, **kwargs)
        if can_bus is not None:
            raise RuntimeError("PerceptionTransformer.get_bev_features: can_bus= must be a CUDA tensor (bs, 18); "
                               "host values belong in img_metas[i]['can_bus']")
        img_metas = kwargs["img_metas"]
        bs = mlvl_feats[0].size(0)
        bev_queries = bev_queries.unsqueeze(1).repeat(1, bs, 1)
        bev_pos = bev_pos.flatten(2).permute(2, 0, 1)
        shift = bev_queries.new_tensor(self._shift(img_metas, bev_h, bev_w, grid_length))
        if prev_bev is not None:
            if prev_bev.shape[1] == bev_h * bev_w:
                prev_bev = prev_bev.permute(1, 0, 2)
            if self.rotate_prev_bev:
                prev_bev = self._rotate_prev(prev_bev, img_metas, bev_h, bev_w)
        can_bus = bev_queries.new_tensor([m["can_bus"] for m in img_metas])
        can_bus = self.can_bus_mlp(can_bus)[None, :, :]
        bev_queries = bev_queries + can_bus * self.use_can_bus
        # (the can_bus MLP above runs in its parameters' dtype; the encoder from here on in the compute dtype)
        bev_queries, bev_pos, prev_bev = (precision.cast(t, dt) for t in (bev_queries, bev_pos, prev_bev))

        shapes = [tuple(f.shape[-2:]) for f in mlvl_feats]
        if mlvl_feats[0].is_cuda:
            feat_flatten = ops.FlattenFeats.apply(self.cams_embeds if self.use_cams_embeds else None,
                                                  self.level_embeds, *mlvl_feats)
        else:
            raise RuntimeError("PerceptionTransformer.get_bev_features: CUDA tensors required "
                               "(bevformer_b200 has no CPU path)")
        spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=bev_pos.device)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)),
                                       spatial_shapes.prod(1).cumsum(0)[:-1]))
        return self.encoder(bev_queries, feat_flatten, feat_flatten, bev_h=bev_h, bev_w=bev_w,
                            bev_pos=bev_pos, spatial_shapes=spatial_shapes,
                            level_start_index=level_start_index, prev_bev=prev_bev, shift=shift,
                            **kwargs)

    def forward(self, mlvl_feats, bev_queries, object_query_embed=None, bev_h=None, bev_w=None,
                grid_length=[0.512, 0.512], bev_pos=None, reg_branches=None, cls_branches=None, prev_bev=None,
                **kwargs):
        """transformer.py:202-289: ``get_bev_features`` (with every keyword it takes, the device-path ``can_bus=`` /
        ``lidar2img=`` / ``ego_state=`` / ``ego_mode=`` included), then the decoder over ``object_query_embed``
        (num_query, 2C) = [query_pos | query].  Returns (bev_embed (Nq, bs, C), inter_states, init_reference_out,
        inter_references_out) in the compute dtype.  On the device path the call neither synchronises nor copies
        from host memory, so it can be captured in a CUDA graph (BEVStream)."""
        if self.decoder is None:
            raise NotImplementedError(
                "bevformer_b200.PerceptionTransformer was built without a decoder dict: it is the BEV encoder "
                "(get_bev_features) alone")
        dec_kwargs = {k: v for k, v in kwargs.items() if k not in _BEV_ONLY_KWARGS}
        bev_embed = self.get_bev_features(mlvl_feats, bev_queries, bev_h, bev_w, grid_length=grid_length,
                                          bev_pos=bev_pos, prev_bev=prev_bev, **kwargs)
        return _decode(self, bev_embed, object_query_embed, bev_h, bev_w, reg_branches, cls_branches, **dec_kwargs)


# get_bev_features' device-path arguments: the decoder layers do not see them
_BEV_ONLY_KWARGS = ("can_bus", "lidar2img", "ego_state", "ego_mode")


def _level_tensors(module, bev_h, bev_w, device):
    """The decoder's one-level spatial_shapes / level_start_index as device tensors, built once per (shape,
    device): a fresh ``torch.tensor`` per call is a pageable host copy, which a CUDA graph cannot capture."""
    cache = module.__dict__.setdefault("_decoder_levels", {})
    key = (int(bev_h), int(bev_w), str(device))
    if key not in cache:
        cache[key] = (torch.tensor([[bev_h, bev_w]], device=device), torch.tensor([0], device=device))
    return cache[key]


@precision.entry("bev_embed", "object_query_embed")
def _decode(module, bev_embed, object_query_embed, bev_h, bev_w, reg_branches=None, cls_branches=None, **kwargs):
    """The object-query half of PerceptionTransformer.forward (transformer.py:262-289) and
    PerceptionTransformerV2.forward (transformerV2.py:329-353): split of ``object_query_embed`` into position and
    content, initial reference points (Linear + sigmoid), the decoder over ``bev_embed`` (bs, Nq, C).  Returns
    (bev_embed (Nq, bs, C), inter_states, init_reference_out, inter_references_out)."""
    bs = bev_embed.shape[0]
    query_pos, query = torch.split(object_query_embed, module.embed_dims, dim=1)
    query_pos = query_pos.unsqueeze(0).expand(bs, -1, -1)
    query = query.unsqueeze(0).expand(bs, -1, -1)
    rp = module.reference_points
    reference_points = linear(query_pos, rp.weight, rp.bias).sigmoid()
    init_reference_out = reference_points
    query = query.permute(1, 0, 2)
    query_pos = query_pos.permute(1, 0, 2)
    bev_embed = bev_embed.permute(1, 0, 2)
    spatial_shapes, level_start_index = _level_tensors(module, bev_h, bev_w, query.device)
    inter_states, inter_references = module.decoder(
        query=query, key=None, value=bev_embed, query_pos=query_pos, reference_points=reference_points,
        reg_branches=reg_branches, cls_branches=cls_branches, spatial_shapes=spatial_shapes,
        level_start_index=level_start_index, **kwargs)
    return bev_embed, inter_states, init_reference_out, inter_references


class PerceptionTransformerBEVEncoder(nn.Module):
    """BEVFormerV2's wrapper around the same encoder (modules/transformerV2.py:54-174): camera / level
    embeddings + flatten, then the encoder WITHOUT temporal input (prev_bev=None, zero shift), then --
    only when the data pipeline applied a global BEV augmentation -- a resampling of the result onto the
    augmented grid.  Same constructor arguments, parameter names and forward signature."""

    def __init__(self, num_feature_levels=4, num_cams=6, two_stage_num_proposals=300, encoder=None,
                 embed_dims=256, use_cams_embeds=True, rotate_center=[100, 100], init_cfg=None, **kwargs):
        super().__init__()
        self.init_cfg = init_cfg
        self.encoder = build_transformer_layer_sequence(encoder)
        self.embed_dims = embed_dims
        self.num_feature_levels = num_feature_levels
        self.num_cams = num_cams
        self.fp16_enabled = False
        self.use_cams_embeds = use_cams_embeds
        self.two_stage_num_proposals = two_stage_num_proposals
        self.rotate_center = rotate_center
        self.level_embeds = nn.Parameter(torch.empty(num_feature_levels, embed_dims))
        if use_cams_embeds:
            self.cams_embeds = nn.Parameter(torch.empty(num_cams, embed_dims))
        self.init_weights()

    def init_weights(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if type(m).__name__ in ("MSDeformableAttention3D", "TemporalSelfAttention",
                                    "CustomMSDeformableAttention"):
                (getattr(m, "init_weight", None) or m.init_weights)()
        nn.init.normal_(self.level_embeds)
        if self.use_cams_embeds:
            nn.init.normal_(self.cams_embeds)

    @precision.entry("mlvl_feats", "bev_queries", "bev_pos")
    def forward(self, mlvl_feats, bev_queries, bev_h, bev_w, grid_length=[0.512, 0.512], bev_pos=None,
                prev_bev=None, **kwargs):
        """Returns the BEV features (bs, bev_h*bev_w, C) in the compute dtype (bevformer_b200.precision);
        ``prev_bev`` is accepted and ignored, as in the reference (:97-141).  Also the encoder half of
        PerceptionTransformerV2."""
        if not mlvl_feats[0].is_cuda:
            raise RuntimeError("PerceptionTransformerBEVEncoder: CUDA tensors required "
                               "(bevformer_b200 has no CPU path)")
        bs = mlvl_feats[0].size(0)
        bev_queries = bev_queries.unsqueeze(1).repeat(1, bs, 1)
        bev_pos = bev_pos.flatten(2).permute(2, 0, 1)
        feat_flatten = ops.FlattenFeats.apply(self.cams_embeds if self.use_cams_embeds else None,
                                              self.level_embeds, *mlvl_feats)
        spatial_shapes = torch.as_tensor([tuple(f.shape[-2:]) for f in mlvl_feats], dtype=torch.long,
                                         device=bev_pos.device)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)),
                                       spatial_shapes.prod(1).cumsum(0)[:-1]))
        bev_embed = self.encoder(bev_queries, feat_flatten, feat_flatten, bev_h=bev_h, bev_w=bev_w,
                                 bev_pos=bev_pos, spatial_shapes=spatial_shapes,
                                 level_start_index=level_start_index, prev_bev=None,
                                 shift=bev_queries.new_tensor([0, 0]).unsqueeze(0), **kwargs)
        return self._align_to_augmentation(bev_embed, kwargs["img_metas"], bs, bev_h, bev_w)

    @staticmethod
    def _align_to_augmentation(bev, img_metas, bs, bev_h, bev_w):
        """transformerV2.py:142-174: with a GlobalRotScaleTransImage augmentation that only moved the
        ground truth, the BEV map is resampled through the 2x2 part of the augmentation matrix (bilinear
        grid_sample); with the augmentation applied to the images too it is only re-laid-out; without it
        the encoder output is returned as is.  Once per training sample, tensor ops as in the reference."""
        aug = img_metas[0].get("aug_param", {}) if isinstance(img_metas[0], dict) else {}
        if "GlobalRotScaleTransImage_param" not in aug:
            return bev
        _rot, _scale, _fx, _fy, bda_mat, only_gt = aug["GlobalRotScaleTransImage_param"]
        img = bev.reshape(bs, bev_h, bev_w, -1).permute(0, 3, 1, 2)
        if only_gt:
            ys = torch.linspace(0.5, bev_h - 0.5, bev_h, dtype=bev.dtype, device=bev.device) / bev_h
            xs = torch.linspace(0.5, bev_w - 0.5, bev_w, dtype=bev.dtype, device=bev.device) / bev_w
            ref_y, ref_x = torch.meshgrid(ys, xs, indexing="ij")
            grid = (torch.stack((ref_x, ref_y), -1) * 2.0 - 1.0).unsqueeze(0).unsqueeze(-1)
            mat = torch.as_tensor(bda_mat)[:2, :2].to(grid).view(1, 1, 1, 2, 2)
            grid = torch.matmul(mat, grid).squeeze(-1)
            img = torch.nn.functional.grid_sample(img, grid.expand(bs, -1, -1, -1), align_corners=False)
        return img.reshape(bs, -1, bev_h * bev_w).permute(0, 2, 1)


class _BasicBlock(nn.Module):
    """mmdet's ResNet BasicBlock (mmdet/models/backbones/resnet.py, 2.14): conv3x3 - norm - ReLU - conv3x3 -
    norm, + identity (or downsample(x)), ReLU; parameter names conv1 / bn1 / conv2 / bn2 / downsample."""

    def __init__(self, inplanes, planes, norm, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride=1, padding=1, bias=False)
        self.bn1 = norm(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False)
        self.bn2 = norm(planes)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        identity = x if self.downsample is None else self.downsample(x)
        out = self.relu(self.bn1(self.conv1(x)))
        return self.relu(self.bn2(self.conv2(out)) + identity)


class ResNetFusion(nn.Module):
    """BEVFormerV2's temporal fusion (modules/transformerV2.py:16-51): the BEV maps of the configured
    frames are concatenated along channels, run through ``num_layer`` ResNet basic blocks and projected back
    to ``out_channels`` with Linear + LayerNorm.  Dense 3x3 convolutions over a 200x200 map: cuDNN work,
    outside the sampler hot path; kept so that the V2 configs build and run through this package."""

    def __init__(self, in_channels, out_channels, inter_channels, num_layer, norm_cfg=dict(type="SyncBN"),
                 with_cp=False):
        super().__init__()
        typ = (norm_cfg or {}).get("type", "BN")
        if typ not in ("BN", "BN2d", "SyncBN"):
            raise KeyError(f"ResNetFusion: unsupported norm {typ}")
        norm = nn.SyncBatchNorm if typ == "SyncBN" else nn.BatchNorm2d
        layers = []
        self.inter_channels = inter_channels
        for i in range(num_layer):
            if i == 0 and inter_channels != in_channels:
                down = nn.Sequential(nn.Conv2d(in_channels, inter_channels, 3, stride=1, padding=1, bias=False),
                                     norm(inter_channels))
                layers.append(_BasicBlock(in_channels, inter_channels, norm, down))
            else:
                layers.append(_BasicBlock(in_channels if i == 0 else inter_channels, inter_channels, norm))
        self.layers = nn.Sequential(*layers)
        self.layer_norm = nn.Sequential(nn.Linear(inter_channels, out_channels), nn.LayerNorm(out_channels))
        self.with_cp = with_cp

    def forward(self, x):
        x = torch.cat(x, 1).contiguous()                      # (bs, frames * C, bev_h, bev_w)
        for layer in self.layers:
            if self.with_cp and x.requires_grad:
                x = torch.utils.checkpoint.checkpoint(layer, x)
            else:
                x = layer(x)
        x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)      # nchw -> n (hw) c
        return self.layer_norm(x)


class PerceptionTransformerV2(PerceptionTransformerBEVEncoder):
    """BEVFormerV2's transformer (modules/transformerV2.py:177-353): the BEV encoder of this package, the
    optional multi-frame ResNetFusion, and the object-query decoder (plugin/decoder.py).  Same constructor
    arguments, parameter names and forward contract as the reference class."""

    def __init__(self, num_feature_levels=4, num_cams=6, two_stage_num_proposals=300, encoder=None,
                 embed_dims=256, use_cams_embeds=True, rotate_center=[100, 100], frames=(0,), decoder=None,
                 num_fusion=3, inter_channels=None, **kwargs):
        super().__init__(num_feature_levels, num_cams, two_stage_num_proposals, encoder, embed_dims,
                         use_cams_embeds, rotate_center, **kwargs)
        self.decoder = build_transformer_layer_sequence(decoder)
        self.reference_points = nn.Linear(self.embed_dims, 3)
        self.frames = frames
        if len(self.frames) > 1:
            self.fusion = ResNetFusion(len(self.frames) * self.embed_dims, self.embed_dims,
                                       inter_channels if inter_channels is not None
                                       else len(self.frames) * self.embed_dims, num_fusion)
        self.init_weights()

    def init_weights(self):
        if not hasattr(self, "reference_points"):
            return                                             # base-class constructor call
        super().init_weights()
        nn.init.xavier_uniform_(self.reference_points.weight)
        nn.init.zeros_(self.reference_points.bias)

    def get_bev_features(self, mlvl_feats, bev_queries, bev_h, bev_w, grid_length=[0.512, 0.512],
                         bev_pos=None, prev_bev=None, **kwargs):
        return super().forward(mlvl_feats, bev_queries, bev_h, bev_w, grid_length, bev_pos, prev_bev, **kwargs)

    def forward(self, mlvl_feats, bev_queries, object_query_embed, bev_h, bev_w, grid_length=[0.512, 0.512],
                bev_pos=None, reg_branches=None, cls_branches=None, prev_bev=None, **kwargs):
        """Returns (bev_embed (Nq, bs, C), inter_states, init_reference_out, inter_references_out)
        (transformerV2.py:243-353).  ``prev_bev``: with several frames, the list of the other frames' BEV
        maps with None at the current frame's slot (and at missing frames, filled from a neighbour)."""
        bev_embed = self.get_bev_features(mlvl_feats, bev_queries, bev_h, bev_w, grid_length=grid_length,
                                          bev_pos=bev_pos, prev_bev=None, **kwargs)
        if len(self.frames) > 1:
            cur = list(self.frames).index(0)
            assert prev_bev[cur] is None and len(prev_bev) == len(self.frames)
            prev_bev[cur] = bev_embed
            for i in range(1, cur + 1):                         # missing earlier frames <- the next one
                if prev_bev[cur - i] is None:
                    prev_bev[cur - i] = prev_bev[cur - i + 1].detach()
            for i in range(cur + 1, len(self.frames)):          # missing later frames <- the previous one
                if prev_bev[i] is None:
                    prev_bev[i] = prev_bev[i - 1].detach()
            maps = [x.reshape(x.shape[0], bev_h, bev_w, x.shape[-1]).permute(0, 3, 1, 2).contiguous()
                    for x in prev_bev]
            bev_embed = self.fusion(maps)
        return _decode(self, bev_embed, object_query_embed, bev_h, bev_w, reg_branches, cls_branches, **kwargs)


def patch_reference(cls):
    """Install this module's ``get_bev_features`` on the reference's own PerceptionTransformer class
    (which keeps its decoder ``forward``): ``patch_reference(PerceptionTransformer)`` once at import
    time of a BEVFormer checkout.  Parameter / attribute names are the reference's, so nothing else
    changes; the encoder inside is whatever the config built (the drop-in BEVFormerEncoder)."""
    for name in ("get_bev_features", "_get_bev_features", "_get_bev_features_device", "_shift", "_rotate_prev"):
        setattr(cls, name, getattr(PerceptionTransformer, name))
    return cls


_register(TRANSFORMER, PerceptionTransformer)
_register(TRANSFORMER, PerceptionTransformerBEVEncoder)
_register(TRANSFORMER, PerceptionTransformerV2)
