"""Device-resident ego-motion, the part that needs no GPU: the float64 oracle (tests/ego_oracle.py) is pinned
against the package's host path and against torchvision's rotate, and the two new C entry points validate
their arguments before any launch."""
import copy
import types

import numpy as np
import pytest
import torch

from bevformer_b200 import _lib, synthetic as syn
from bevformer_b200.plugin import BEVStream, PerceptionTransformer
from tests import ego_oracle
from tests.golden.make_golden import grid_length_of, sequence_inputs
from tests.test_abi import declared_symbols

ANGLES = [0.0, 0.5, -0.5, 3.0, -37.3, 90.0, 180.0]
SIZES = [(50, 50), (200, 200), (40, 60)]
CENTER = [100, 100]          # the configs' rotate_center for every BEV size, also 50x50


def _host_shift(metas, w, use_shift=True):
    return PerceptionTransformer._shift(types.SimpleNamespace(use_shift=use_shift), metas, w.bev_h, w.bev_w,
                                        grid_length_of(w))


@pytest.mark.parametrize("workload", ["toy", "tiny"])
def test_oracle_shift_equals_host_shift(workload):
    w = syn.WORKLOADS[workload]
    metas = syn.make_perception_inputs(w, bs=2).img_metas + sequence_inputs(w, frames=4)[3]
    cb = np.array([m["can_bus"] for m in metas], dtype=np.float64)
    for use in (True, False):
        assert np.array_equal(ego_oracle.ego_shift(cb, w.bev_h, w.bev_w, grid_length_of(w), use),
                              _host_shift(metas, w, use))
    still = np.zeros((1, 18))                                        # dx = dy = 0: arctan2(0, 0) = 0, length 0
    still[0, -2] = 0.3
    assert np.array_equal(ego_oracle.ego_shift(still, w.bev_h, w.bev_w, grid_length_of(w)), np.zeros((1, 2)))


class _Recorder(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.seen = []

    def get_bev_features(self, feats, bev_queries, bev_h, bev_w, grid_length=None, bev_pos=None, prev_bev=None,
                         img_metas=None):
        self.seen.append(np.array(img_metas[0]["can_bus"], dtype=np.float64).copy())
        return torch.zeros(1, bev_h * bev_w, 4)


def test_oracle_deltas_equal_host_stream():
    """The 4-frame / 2-scene golden sequence, then a reset and the first two frames again."""
    w = syn.WORKLOADS["toy"]
    feats, q, pos, metas = sequence_inputs(w, frames=4)
    rec = _Recorder()
    stream = BEVStream(rec)
    order = [0, 1, 2, 3, None, 0, 1]
    fresh, seq, token = [], [], None
    for i in order:
        if i is None:
            stream.reset()
            token = None
            continue
        stream.step([f[:, i] for f in feats], [metas[i]], q, w.bev_h, w.bev_w, pos)
        fresh.append(metas[i]["scene_token"] != token)
        token = metas[i]["scene_token"]
        seq.append(metas[i]["can_bus"])
    assert fresh == [True, False, False, True, True, False]
    want, states = ego_oracle.stream_deltas(seq, fresh)
    for a, b in zip(rec.seen, want):
        assert np.array_equal(a, b)
    assert np.array_equal(states[-1][0], stream.prev_frame_info["prev_pos"])
    assert states[-1][1] == stream.prev_frame_info["prev_angle"]


@pytest.mark.parametrize("angle", ANGLES)
@pytest.mark.parametrize("size", SIZES)
def test_oracle_matrix_equals_torchvision(angle, size):
    from torchvision.transforms.functional import _get_inverse_affine_matrix
    h, w = size
    center_f = [1.0 * (c - s * 0.5) for c, s in zip(CENTER, [w, h])]
    assert ego_oracle.rotation_matrix(angle, CENTER, h, w) == _get_inverse_affine_matrix(center_f, -angle, [0.0, 0.0],
                                                                                        1.0, [0.0, 0.0])


def _torchvision_sources(angle, h, w, center):
    """Which cell torchvision's rotate copies into every output cell (-1: zero fill), read off an index image."""
    from torchvision.transforms.functional import rotate
    img = (torch.arange(h * w, dtype=torch.float32) + 1).reshape(1, h, w)
    return rotate(img, angle, center=center).reshape(-1).to(torch.int64).numpy() - 1


@pytest.mark.parametrize("angle", ANGLES)
@pytest.mark.parametrize("size", SIZES)
def test_oracle_index_map_equals_torchvision(angle, size):
    h, w = size
    rows = ego_oracle.rotation_grid_rows(angle, CENTER, h, w)
    got = _torchvision_sources(angle, h, w, CENTER)
    ego_oracle.check_index_map(got, rows, h, w)
    if angle == 0.0:                                                 # every first frame, every static ego
        assert np.array_equal(got, np.arange(h * w))
        assert np.array_equal(ego_oracle.rotation_source(rows, h, w)[0], np.arange(h * w))
    else:
        assert (got < 0).any() or angle in (90.0, 180.0)


def test_index_map_rule_rejects_a_wrong_cell():
    h, w = 50, 50
    rows = ego_oracle.rotation_grid_rows(3.0, CENTER, h, w)
    src, margin = ego_oracle.rotation_source(rows, h, w)
    wrong = src.copy()
    k = int(np.argmax(margin))
    wrong[k] = (wrong[k] + 1) % (h * w)
    with pytest.raises(AssertionError):
        ego_oracle.check_index_map(wrong, rows, h, w)


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_entry_points_declared_and_bound():
    for name in ("bevf_ego_motion", "bevf_rotate_bev"):
        assert name in declared_symbols() and name in _lib.SIGNATURES
        assert hasattr(_lib.load(), name)


def _ego(lib, can_bus=64, state=64, mode=0, shift=64, rot=64, out=64, dtype=0, bs=1, h=8, w=8, gh=0.5, gw=0.5):
    return lib.bevf_ego_motion(can_bus, state, mode, shift, rot, out, dtype, bs, h, w, gh, gw, 100.0, 100.0, 1, None)


def _rot(lib, prev=64, in_dtype=0, sq=256, sb=256, rot=64, out=128, out_dtype=0, bs=1, h=8, w=8, c=256):
    return lib.bevf_rotate_bev(prev, in_dtype, sq, sb, rot, out, out_dtype, bs, h, w, c, None)


@pytest.mark.parametrize("call,kwargs,message", [
    (_ego, dict(can_bus=None), "null pointer"),
    (_ego, dict(shift=None), "null pointer"),
    (_ego, dict(rot=None), "null pointer"),
    (_ego, dict(out=None), "null pointer"),
    (_ego, dict(mode=1, state=None), "null pointer"),
    (_ego, dict(mode=2, state=None), "null pointer"),
    (_ego, dict(can_bus=68), "misaligned"),
    (_ego, dict(mode=1, state=68), "misaligned"),
    (_ego, dict(dtype=3), "dtype code"),
    (_ego, dict(dtype=-1), "dtype code"),
    (_ego, dict(mode=3), "history mode"),
    (_ego, dict(h=0), "bad dimension"),
    (_ego, dict(gh=0.0), "grid_length"),
    (_rot, dict(prev=None), "null pointer"),
    (_rot, dict(rot=None), "null pointer"),
    (_rot, dict(out=None), "null pointer"),
    (_rot, dict(prev=72), "16-byte aligned"),
    (_rot, dict(out=136), "16-byte aligned"),
    (_rot, dict(in_dtype=3), "dtype code"),
    (_rot, dict(out_dtype=7), "dtype code"),
    (_rot, dict(c=252), "multiple of 8"),
    (_rot, dict(sq=100), "strides"),
    (_rot, dict(w=0), "bad dimension"),
])
def test_entry_points_reject_bad_arguments(call, kwargs, message):
    lib = _lib.load()
    assert call(lib, **kwargs) != 0
    assert message.encode() in lib.bevf_last_error()
    with pytest.raises(RuntimeError, match=message):
        _lib.check(1, lib)


def test_ops_refuse_cpu_tensors_and_wrong_types():
    from bevformer_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.ego_motion(torch.zeros(1, 18, dtype=torch.float64), 8, 8, (0.5, 0.5), CENTER, True, torch.float32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.rotate_bev(torch.zeros(64, 1, 256), torch.zeros(1, 6), 8, 8)


def test_device_path_needs_a_device_tensor():
    w = syn.WORKLOADS["toy"]
    m = PerceptionTransformer(num_feature_levels=len(w.levels), num_cams=w.num_cams, encoder=syn.encoder_cfg(w),
                              decoder=None, embed_dims=w.embed_dims)
    inp = syn.make_perception_inputs(w, bs=1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        m.get_bev_features(inp.mlvl_feats, inp.bev_queries, w.bev_h, w.bev_w, bev_pos=inp.bev_pos,
                           img_metas=copy.deepcopy(inp.img_metas), can_bus=torch.zeros(1, 18, dtype=torch.float64))
