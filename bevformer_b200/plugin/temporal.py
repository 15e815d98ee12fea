"""Temporal plumbing around the BEV encoder: the history-BEV recurrence of training and the streaming
state of video inference.

Reference: ``BEVFormer.obtain_history_bev`` (projects/mmdet3d_plugin/bevformer/detectors/bevformer.py:158-177)
runs the encoder over the ``queue_length - 1`` earlier frames without gradients (3 extra encoder passes per
training step at base) and ``BEVFormer.forward_test`` (:236-269, state initialised at :59-64) carries
``prev_frame_info`` from frame to frame.  Both reach the encoder through
``pts_bbox_head(..., only_bev=True)`` -> ``transformer.get_bev_features`` (dense_heads/bevformer_head.py);
here they call ``PerceptionTransformer.get_bev_features`` of this package directly: the detector and head
classes themselves (backbone, FPN, query embeddings, losses) are outside the hot path.  Given the head's object
query embedding (and regression branches), ``BEVStream`` runs the whole transformer per frame instead --
``PerceptionTransformer.forward``, encoder and decoder, as forward_test does through the head (:263-268).

Both take the per-frame CAN-bus vectors and camera matrices either from the metas (host path: numpy + torchvision
once per frame, as the reference) or as CUDA tensors ``can_bus=`` / ``lidar2img=`` (device path: two kernels, no
host synchronisation, and for ``BEVStream`` an optional captured mode that replays one CUDA graph per frame).
"""
from __future__ import annotations

import copy
from typing import List, Optional, Sequence

import numpy as np
import torch

from .. import ops


def _on_device(can_bus) -> bool:
    return torch.is_tensor(can_bus) and can_bus.is_cuda


# a detection frame's outputs, in the order the captured mode keeps its static buffers (the BEV first)
_DET_KEYS = ("bev_embed", "all_cls_scores", "all_bbox_preds", "bboxes", "scores", "labels", "num")


class _DetFrame:
    """A frame through a detection head (plugin.head.BEVFormerHead): ``head.forward`` in eval mode -- the head
    builds its own BEV queries, positional encoding and object queries -- then the coder's ``decode_device``."""

    def __init__(self, head):
        self.head = head

    def __call__(self, mlvl_feats, prev_bev=None, img_metas=None, grid_length=None, bev_pos=None, **device_kwargs):
        was_training = self.head.training
        self.head.eval()
        try:
            out = self.head(mlvl_feats, img_metas, prev_bev=prev_bev, **device_kwargs)
        finally:
            self.head.train(was_training)
        dec = self.head.bbox_coder.decode_device(out)
        return {k: out[k] if k in out else dec[k] for k in _DET_KEYS}


def _bev_of(res):
    """The BEV of a frame's result: the tensor itself, a transformer 4-tuple's first entry, a detection dict's
    ``bev_embed``."""
    if torch.is_tensor(res):
        return res
    return res["bev_embed"] if isinstance(res, dict) else res[0]


def obtain_history_bev(transformer, feats_queue: Sequence[torch.Tensor], img_metas_list, bev_queries,
                       bev_h: int, bev_w: int, bev_pos, grid_length=(0.512, 0.512), can_bus=None,
                       lidar2img=None) -> Optional[torch.Tensor]:
    """The no-grad recurrence over the history frames (bevformer.py:158-177).

    feats_queue   per pyramid level (bs, len_queue, num_cams, C, h, w) -- what ``extract_feat(img,
                  len_queue=len_queue)`` returns (:150-156)
    img_metas_list  per sample, indexable by frame: ``img_metas_list[b][i]`` is frame i's meta dict with
                  ``prev_bev_exists`` / ``can_bus`` / ``lidar2img`` / ``img_shape`` (:169-171)
    can_bus       optional (bs, len_queue, 18) float64 CUDA tensor of the frames' CAN-bus DELTAS (what the metas
                  hold in training): selects the device path of ``get_bev_features`` for every frame; the metas
                  are then read for ``prev_bev_exists`` (a host flag: it decides which kernels run) and
                  ``img_shape`` only
    lidar2img     optional (bs, len_queue, num_cams, 4, 4) float32 CUDA tensor, used instead of the metas' matrices
    Returns the BEV of the last history frame (bs, Nq, C), or None for an empty queue.  The transformer
    is put in eval mode for the loop and returned to the mode it was in (the reference calls
    ``self.train()`` unconditionally, :176)."""
    was_training = transformer.training
    transformer.eval()
    try:
        with torch.no_grad():
            prev_bev = None
            len_queue = feats_queue[0].shape[1]
            for i in range(len_queue):
                img_metas = [each[i] for each in img_metas_list]
                if not img_metas[0]["prev_bev_exists"]:               # :170-171, sample 0 decides for the batch
                    prev_bev = None
                img_feats = [lvl[:, i] for lvl in feats_queue]
                extra = {}
                if can_bus is not None:
                    extra["can_bus"] = can_bus[:, i]
                if lidar2img is not None:
                    extra["lidar2img"] = lidar2img[:, i]
                prev_bev = transformer.get_bev_features(img_feats, bev_queries, bev_h, bev_w,
                                                        grid_length=list(grid_length), bev_pos=bev_pos,
                                                        prev_bev=prev_bev, img_metas=img_metas, **extra)
            return prev_bev
    finally:
        transformer.train(was_training)


class BEVStream:
    """Streaming inference state: the previous frame's BEV, ego position and heading
    (``prev_frame_info``, bevformer.py:59-64) and the per-frame update of forward_test (:236-269):
    a new scene (or ``video_test_mode=False``) drops the history; CAN-bus position / angle are turned into
    deltas against the previous frame before the encoder sees them, zeros on a scene's first frame.

    Three ways to run a frame, chosen by what ``step`` is given:
      * host path     the metas carry ABSOLUTE ``can_bus``; position / angle live in ``prev_frame_info`` as numpy;
      * device path   ``can_bus=`` (bs, 18) float64 and ``lidar2img=`` (bs, num_cams, 4, 4) float32 CUDA tensors;
                      position / angle / "has history" live in a 40-byte device block (``ops.ego_state``) that
                      ``bevf_ego_motion`` reads and advances; the step never synchronises with the host;
      * captured      after ``capture(...)``: the device path recorded as two CUDA graphs (first frame of a scene,
                      continuation); ``step`` replays the one the scene token selects.
    With ``object_query_embed`` (num_query, 2C) given -- to ``step``, or to ``capture`` for the captured mode -- a
    frame is the whole transformer (``transformer.forward``: encoder, then the object-query decoder with
    ``reg_branches`` / ``cls_branches``) and returns its 4-tuple (bev_embed (Nq, bs, C), inter_states,
    init_reference_out, inter_references_out); bev_embed becomes the next frame's prev_bev.  Without it a frame is
    ``get_bev_features`` and returns the BEV alone.
    With ``head`` (plugin.head.BEVFormerHead, whose transformer is this stream's) a frame is ``head.forward`` plus
    its coder's ``decode_device`` and returns ``dict(bev_embed, all_cls_scores, all_bbox_preds, bboxes, scores, labels,
    num)`` (the decode's fixed-capacity tensors: no host synchronisation); ``bev_queries`` / ``bev_pos`` /
    ``grid_length`` are then the head's own and the arguments of those names are not read.
    ``prev_frame_info["scene_token"]`` and ``["prev_bev"]`` are shared by the three; do not mix the host path with
    the other two inside one scene (each keeps its own previous position / angle)."""

    def __init__(self, transformer, video_test_mode: bool = True):
        self.transformer = transformer
        self.video_test_mode = video_test_mode
        self.ego_state = None            # device-side prev_pos / prev_angle / has-history (created on first use)
        self.static = None               # captured mode: {"feats": [...], "can_bus": ..., "lidar2img": ...}
        self._graphs = None
        self.reset()

    def reset(self) -> None:
        self.prev_frame_info = {"prev_bev": None, "scene_token": None, "prev_pos": 0, "prev_angle": 0}
        if self.ego_state is not None:
            self.ego_state.zero_()

    @torch.no_grad()
    def step(self, mlvl_feats: Optional[List[torch.Tensor]], img_metas: List[dict], bev_queries=None, bev_h: int = None,
             bev_w: int = None, bev_pos=None, grid_length=(0.512, 0.512), can_bus=None, lidar2img=None,
             object_query_embed=None, reg_branches=None, cls_branches=None, head=None):
        """One frame: mlvl_feats per level (bs, num_cams, C, h, w), img_metas one dict per sample with
        ABSOLUTE ``can_bus`` and a ``scene_token``.  Returns this frame's BEV (bs, Nq, C), which also becomes
        the next frame's ``prev_bev``.  The caller's metas are not modified (the reference edits them in
        place, :254-261; the values the encoder sees are the same).

        Device path: ``can_bus=`` holds the ABSOLUTE CAN-bus vectors on the device (the metas' ``can_bus`` is not
        read; ``scene_token`` and ``img_shape`` are).  Captured mode: only ``img_metas[0]["scene_token"]`` is read;
        tensors passed for ``mlvl_feats`` / ``can_bus`` / ``lidar2img`` are copied into the static buffers, ``None``
        means the caller has filled ``self.static`` itself.  The BEV returned in captured mode is the static
        output buffer: it is OVERWRITTEN by the next ``step`` (clone it to keep it).

        ``object_query_embed`` / ``reg_branches`` / ``cls_branches``: run the whole transformer and return its 4-tuple
        (in captured mode, what ``capture`` was given decides, and these are ignored)."""
        if self._graphs is not None:
            return self._step_captured(mlvl_feats, img_metas, can_bus, lidar2img)
        if head is not None:
            head = _DetFrame(head)
        elif object_query_embed is not None:
            head = (object_query_embed, reg_branches, cls_branches)
        info = self.prev_frame_info
        if img_metas[0].get("scene_token") != info["scene_token"]:
            info["prev_bev"] = None                                  # :243-245
        info["scene_token"] = img_metas[0].get("scene_token")
        if not self.video_test_mode:
            info["prev_bev"] = None                                  # :249-251
        if _on_device(can_bus):
            res = self._frame(mlvl_feats, img_metas, bev_queries, bev_h, bev_w, bev_pos, grid_length, can_bus,
                              lidar2img, info["prev_bev"], head)
            info["prev_bev"] = _bev_of(res)
            return res
        metas = [dict(m) for m in img_metas]
        can_bus = np.array(metas[0]["can_bus"], dtype=np.float64, copy=True)
        tmp_pos, tmp_angle = can_bus[:3].copy(), copy.deepcopy(can_bus[-1])      # :254-255
        if info["prev_bev"] is not None:
            can_bus[:3] -= info["prev_pos"]                          # :257-258
            can_bus[-1] -= info["prev_angle"]
        else:
            can_bus[-1] = 0                                          # :260-261
            can_bus[:3] = 0
        metas[0]["can_bus"] = can_bus
        was_training = self.transformer.training
        self.transformer.eval()
        try:
            res = self._run(head, mlvl_feats, bev_queries, bev_h, bev_w, grid_length=list(grid_length),
                            bev_pos=bev_pos, prev_bev=info["prev_bev"], img_metas=metas)
        finally:
            self.transformer.train(was_training)
        bev = _bev_of(res)
        info["prev_pos"], info["prev_angle"], info["prev_bev"] = tmp_pos, tmp_angle, bev    # :266-268
        return res

    def _run(self, head, mlvl_feats, bev_queries, bev_h, bev_w, **kwargs):
        """get_bev_features, or with ``head`` = (object_query_embed, reg_branches, cls_branches) the whole
        transformer; with a ``_DetFrame`` the detection frame."""
        if head is None:
            return self.transformer.get_bev_features(mlvl_feats, bev_queries, bev_h, bev_w, **kwargs)
        if isinstance(head, _DetFrame):
            return head(mlvl_feats, **kwargs)
        oq, reg, cls = head
        return self.transformer(mlvl_feats, bev_queries, oq, bev_h, bev_w, reg_branches=reg, cls_branches=cls,
                                **kwargs)

    # ---- device path --------------------------------------------------------------------------------------------
    def _frame(self, mlvl_feats, img_metas, bev_queries, bev_h, bev_w, bev_pos, grid_length, can_bus, lidar2img,
               prev_bev, head=None):
        """One device-path frame; the delta step of forward_test (:254-268) happens inside bevf_ego_motion."""
        if self.ego_state is None:
            self.ego_state = ops.ego_state(can_bus.device)
        extra = {} if lidar2img is None else dict(lidar2img=lidar2img)
        was_training = self.transformer.training
        self.transformer.eval()
        try:
            return self._run(head, mlvl_feats, bev_queries, bev_h, bev_w, grid_length=list(grid_length),
                             bev_pos=bev_pos, prev_bev=prev_bev, img_metas=img_metas, can_bus=can_bus,
                             ego_state=self.ego_state,
                             ego_mode=ops.EGO_NEW_SCENE if prev_bev is None else ops.EGO_CONTINUE, **extra)
        finally:
            self.transformer.train(was_training)

    # ---- captured mode ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def capture(self, mlvl_feats: List[torch.Tensor], img_metas: List[dict], bev_queries=None, bev_h: int = None,
                bev_w: int = None, bev_pos=None, grid_length=(0.512, 0.512), *, can_bus, lidar2img,
                object_query_embed=None, reg_branches=None, cls_branches=None, head=None) -> dict:
        """Record the device path for these shapes as two CUDA graphs -- first frame of a scene (no history: the
        temporal self-attention stacks the query with itself) and continuation (prev_bev = the previous output,
        rotated) -- over static input buffers, returned (and kept as ``self.static``): ``{"feats": [per level],
        "can_bus": (bs, 18) f64, "lidar2img": (bs, num_cams, 4, 4) f32}``.  They start as copies of the arguments;
        write each frame's data into them (or pass tensors to ``step``, which copies).  ``bev_queries`` and
        ``bev_pos`` are read in place by every replay.  One eager frame of each kind runs first (it sizes the
        encoder's pair list from the rig given here, + 15 %, which synchronises once); the stream is reset
        afterwards.  A replay cannot report a pair-list overflow (``BEVFormerEncoder.check_plan`` sees eager forwards
        only): before replaying a rig that may put more pairs in view than the captured one, run one eager
        device-path frame with it and ``encoder.check_plan()``, and capture again if that raises.

        With ``object_query_embed`` the graphs record the whole transformer (encoder and decoder; the embedding and
        the branches are read in place by every replay) and ``step`` returns the static 4-tuple of output buffers; with
        ``head`` the graphs record the detection frame and ``step`` returns its dict of static output buffers."""
        if not (_on_device(can_bus) and _on_device(lidar2img)):
            raise RuntimeError("BEVStream.capture: can_bus and lidar2img must be CUDA tensors (the device path)")
        self._graphs = None
        self.static = dict(feats=[f.detach().clone() for f in mlvl_feats],
                           can_bus=can_bus.detach().to(torch.float64).reshape(-1, 18).clone(),
                           lidar2img=lidar2img.detach().to(torch.float32).clone())
        self._cap = dict(img_metas=[dict(img_shape=img_metas[0]["img_shape"]) for _ in img_metas],
                         bev_queries=bev_queries, bev_h=bev_h, bev_w=bev_w, bev_pos=bev_pos, grid_length=grid_length,
                         head=_DetFrame(head) if head is not None else
                         None if object_query_embed is None else (object_query_embed, reg_branches, cls_branches))
        self._record()
        return self.static

    @torch.no_grad()
    def _record(self) -> None:
        c, st = self._cap, self.static
        dev = st["can_bus"].device

        def frame(prev):                                   # the frame's outputs as a tuple, bev first
            res = self._frame(st["feats"], c["img_metas"], c["bev_queries"], c["bev_h"], c["bev_w"], c["bev_pos"],
                              c["grid_length"], st["can_bus"], st["lidar2img"], prev, c["head"])
            if c["head"] is None:
                return (res,)
            return tuple(res[k] for k in _DET_KEYS) if isinstance(res, dict) else tuple(res)

        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):                      # eager warm-up of both kinds of frame
            outs = tuple(t.clone() for t in frame(None))
            frame(outs[0])
        cur.wait_stream(side)
        graphs, pool = {}, None
        for kind in ("first", "cont"):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):
                for o, r in zip(outs, frame(None if kind == "first" else outs[0])):
                    o.copy_(r)
            graphs[kind], pool = g, g.pool()
        if c["head"] is None:
            out = outs[0]
        else:
            out = dict(zip(_DET_KEYS, outs)) if isinstance(c["head"], _DetFrame) else outs
        self._graphs, self._out = graphs, out
        self.reset()

    def _step_captured(self, mlvl_feats, img_metas, can_bus, lidar2img):
        st, info = self.static, self.prev_frame_info
        for src, dst in zip(mlvl_feats or (), st["feats"]):
            if src.data_ptr() != dst.data_ptr():
                dst.copy_(src)
        for src, dst in ((can_bus, st["can_bus"]), (lidar2img, st["lidar2img"])):
            if src is not None and src.data_ptr() != dst.data_ptr():
                dst.copy_(src.reshape(dst.shape))
        token = img_metas[0].get("scene_token")
        first = token != info["scene_token"] or info["prev_bev"] is None or not self.video_test_mode
        info["scene_token"] = token
        self._graphs["first" if first else "cont"].replay()
        info["prev_bev"] = _bev_of(self._out)
        return self._out
