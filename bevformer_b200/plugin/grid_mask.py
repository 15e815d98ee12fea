"""GridMask: drop-in for the detectors' training-time image mask (projects/mmdet3d_plugin/models/utils/grid_mask.py:70-124),
built by BEVFormer and BEVFormerV2 as ``GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=0.7)``
and applied to the current frame's (B*N, 3, H, W) images in ``extract_img_feat``.

The module makes the reference's ``np.random`` calls, with the same arguments in the same order, so a seeded run masks
the same pixels and leaves numpy's global state where the reference leaves it.  The drawn integers travel to the
kernel (``ops.grid_mask``, csrc/grid_mask.cu) as arguments: no mask is built on the host and nothing is copied to the
device, so the call does not synchronise the stream.  The reference's per-image ``Grid`` class, which no pipeline
uses, has no counterpart here.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .. import ops


class GridMask(nn.Module):
    """Same constructor, attributes (use_h, use_w, rotate, offset, ratio, mode, st_prob, prob, l after a masking call,
    fp16_enable) and ``set_prob`` as the reference.  Only rotate = 1 and offset = False, the variant every detector
    builds, are implemented."""

    def __init__(self, use_h, use_w, rotate=1, offset=False, ratio=0.5, mode=0, prob=1.):
        super().__init__()
        if rotate != 1:
            raise NotImplementedError("GridMask: rotate > 1 (a PIL rotation of the mask) is not implemented; the "
                                      "BEVFormer and BEVFormerV2 detectors build rotate=1")
        if offset:
            raise NotImplementedError("GridMask: offset=True is not implemented; the BEVFormer and BEVFormerV2 "
                                      "detectors build offset=False")
        self.use_h = use_h
        self.use_w = use_w
        self.rotate = rotate
        self.offset = offset
        self.ratio = ratio
        self.mode = mode
        self.st_prob = prob
        self.prob = prob
        self.fp16_enable = False

    def set_prob(self, epoch, max_epoch):
        self.prob = self.st_prob * epoch / max_epoch

    def forward(self, x):
        # mmcv's auto_fp16 on the reference's forward: float32 inputs become float16 when fp16_enabled is set
        if getattr(self, "fp16_enabled", False) and isinstance(x, torch.Tensor) and x.dtype == torch.float32:
            x = x.half()
        if self.training and x.is_cuda:
            with torch.cuda.device(x.device):
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("GridMask: a training-mode call cannot be captured in a CUDA graph (every "
                                       "replay would reuse the captured random draws)")
        # the reference's draws and shape handling, in its order (grid_mask.py:86-108)
        if np.random.rand() > self.prob or not self.training:
            return x
        n, c, h, w = x.size()
        x = x.view(-1, h, w)
        d = np.random.randint(2, h)
        self.l = min(max(int(d * self.ratio + 0.5), 1), d - 1)
        st_h = np.random.randint(d)
        st_w = np.random.randint(d)
        np.random.randint(self.rotate)          # the rotation angle: always 0 for rotate=1
        x = ops.grid_mask(x, d, self.l, st_h, st_w, self.use_h, self.use_w, self.mode)
        return x.view(n, c, h, w)
