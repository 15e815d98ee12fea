"""Float64 CPU restatement of the once-per-frame ego-motion block, the yardstick of the device path
(bevf_ego_motion / bevf_rotate_bev).  Test infrastructure only: plain numpy, no kernels.  Each function names the
reference lines or the torchvision function it restates; tests/test_ego_device_cpu.py pins them against the
package's host path and against torchvision itself."""
import math

import numpy as np


def ego_shift(can_bus, bev_h, bev_w, grid_length, use_shift=True):
    """PerceptionTransformer.get_bev_features' shift (modules/transformer.py:122-140): can_bus (bs, 18) float64 ->
    (bs, 2) float64 (shift_x, shift_y) in normalised BEV units."""
    cb = np.asarray(can_bus, dtype=np.float64)
    dx, dy = cb[:, 0], cb[:, 1]
    ego = cb[:, -2] / np.pi * 180
    length = np.sqrt(dx ** 2 + dy ** 2)
    bev_angle = ego - np.arctan2(dy, dx) / np.pi * 180
    sy = length * np.cos(bev_angle / 180 * np.pi) / grid_length[0] / bev_h
    sx = length * np.sin(bev_angle / 180 * np.pi) / grid_length[1] / bev_w
    return np.stack([sx, sy], -1) * float(bool(use_shift))


def stream_deltas(can_bus_seq, new_scene):
    """forward_test's CAN-bus state machine (detectors/bevformer.py:254-268) for sample 0: absolute vectors in,
    the vectors the encoder sees out.  ``new_scene[i]``: frame i has no history (scene change, first frame, or
    video_test_mode off).  Also returns the state after every frame as (prev_pos (3), prev_angle)."""
    out, states = [], []
    prev_pos, prev_angle = np.zeros(3), 0.0
    for cb, fresh in zip(can_bus_seq, new_scene):
        cb = np.array(cb, dtype=np.float64, copy=True)
        tmp_pos, tmp_angle = cb[:3].copy(), float(cb[-1])
        if fresh:
            cb[:3] = 0
            cb[-1] = 0
        else:
            cb[:3] -= prev_pos
            cb[-1] -= prev_angle
        prev_pos, prev_angle = tmp_pos, tmp_angle
        out.append(cb)
        states.append((prev_pos.copy(), prev_angle))
    return out, states


def rotation_matrix(angle, center, bev_h, bev_w):
    """torchvision.transforms.functional.rotate's matrix for an (C, bev_h, bev_w) image: ``center_f = center -
    size / 2`` then ``_get_inverse_affine_matrix(center_f, -angle, [0, 0], 1.0, [0, 0])`` -- six float64."""
    cx, cy = (1.0 * (c - s * 0.5) for c, s in zip(center, [bev_w, bev_h]))
    rot = math.radians(-angle)
    a, b = math.cos(rot), -math.sin(rot)          # (shear 0: cos(0) = 1, tan(0) = 0)
    c, d = math.sin(rot), math.cos(rot)
    m = [d, -b, 0.0, -c, a, 0.0]
    m[2] += m[0] * (-cx) + m[1] * (-cy)
    m[5] += m[3] * (-cx) + m[4] * (-cy)
    m[2] += cx
    m[5] += cy
    return m


def rotation_grid_rows(angle, center, bev_h, bev_w):
    """The matrix as ``_functional_tensor.rotate`` + ``_gen_affine_grid`` use it: rounded to float32, x row divided
    by 0.5 * w and y row by 0.5 * h in float32 -- (6,) float32, the operand bevf_rotate_bev takes."""
    m = np.asarray(rotation_matrix(angle, center, bev_h, bev_w), dtype=np.float64).astype(np.float32)
    div = np.asarray([0.5 * bev_w] * 3 + [0.5 * bev_h] * 3, dtype=np.float32)
    return (m / div).astype(np.float32)


def rotation_source(rows, bev_h, bev_w):
    """Source coordinates of every output cell in float64 from the float32 grid rows: ``_gen_affine_grid``'s base
    grid (-w/2 + 0.5 + j, -h/2 + 0.5 + i, 1) times the rows, then grid_sample's un-normalisation for
    align_corners=False, ((g + 1) * size - 1) / 2.  Returns (src, margin): src (bev_h*bev_w,) int64, the nearest
    cell's flat index (ties to even, as nearbyint) or -1 outside the map; margin, each cell's distance in pixels
    from the nearest rounding boundary k + 0.5 (cells with a small margin may legitimately pick the neighbour)."""
    r = np.asarray(rows, dtype=np.float64)
    j = np.arange(bev_w, dtype=np.float64)[None, :] + 0.5 - bev_w * 0.5
    i = np.arange(bev_h, dtype=np.float64)[:, None] + 0.5 - bev_h * 0.5
    gx = j * r[0] + i * r[1] + r[2]
    gy = j * r[3] + i * r[4] + r[5]
    fx = ((gx + 1) * bev_w - 1) / 2
    fy = ((gy + 1) * bev_h - 1) / 2
    rx, ry = np.rint(fx), np.rint(fy)
    inside = (rx >= 0) & (rx <= bev_w - 1) & (ry >= 0) & (ry <= bev_h - 1)
    src = np.where(inside, ry * bev_w + rx, -1).astype(np.int64).reshape(-1)
    margin = np.minimum(0.5 - np.abs(fx - rx), 0.5 - np.abs(fy - ry)).reshape(-1)
    return src, margin


def check_index_map(got_src, rows, bev_h, bev_w, tol_px=1e-4, max_near=1e-3):
    """The boundary rule: every cell further than ``tol_px`` from a rounding boundary must have picked the
    oracle's source cell; the cells nearer than that must stay below ``max_near`` of the map.  Returns the number
    of near-boundary cells.  1e-4 px is about ten times the float32 error of a coordinate on a 200-cell map
    (torchvision's own float32 grid differs from this float64 one only in cells within 4e-6 px of a boundary);
    a wider band would by plain geometry hold more than 0.1 % of any map (a band of +-t px around the boundaries
    of both axes covers a fraction 4t of the cells)."""
    src, margin = rotation_source(rows, bev_h, bev_w)
    got = np.asarray(got_src).reshape(-1)
    far = margin > tol_px
    bad = np.nonzero(far & (got != src))[0]
    assert bad.size == 0, (bad[:8], got[bad[:8]], src[bad[:8]], margin[bad[:8]])
    near = int((~far).sum())
    assert near < max(1.0, max_near * src.size), (near, src.size)
    return near
