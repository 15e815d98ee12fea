"""Device-resident ego-motion on the GPU: the two kernels against the float64 oracle and torchvision, the device
path of get_bev_features / obtain_history_bev / BEVStream against the host path and the reference golden data,
the no-host-traffic guarantee, and the captured stream."""
import copy

import numpy as np
import pytest
import torch

from bevformer_b200 import _lib, ops, synthetic as syn
from bevformer_b200.plugin import BEVStream, PerceptionTransformer, obtain_history_bev
from tests import ego_oracle
from tests.golden.make_golden import grid_length_of, sequence_inputs
from tests.util import golden, max_err, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
ANGLES = [0.0, 0.5, -0.5, 3.0, -37.3, 90.0, 180.0]
SIZES = [(50, 50), (200, 200), (40, 60)]
CENTER = [100, 100]


# ---- bevf_rotate_bev ------------------------------------------------------------------------------------------------
def _rotate_case(dtype, batch_first, h, w, angles, out_dtype=None, channels=64):
    from torchvision.transforms.functional import rotate
    bs, nq = len(angles), h * w
    g = torch.Generator().manual_seed(h * w + bs)
    prev = torch.randn(bs, nq, channels, generator=g).to(DEV, dtype)
    if not batch_first:
        prev = prev.permute(1, 0, 2).contiguous()
    rows = np.stack([ego_oracle.rotation_grid_rows(a, CENTER, h, w) for a in angles])
    before = _lib.launch_count()
    out = ops.rotate_bev(prev, torch.as_tensor(rows).to(DEV), h, w, out_dtype)
    assert _lib.launch_count() == before + 1
    assert out.shape == (nq, bs, channels) and out.dtype == (out_dtype or dtype) and out.is_contiguous()
    for b, angle in enumerate(angles):
        mine = prev[b] if batch_first else prev[:, b]
        src, margin = ego_oracle.rotation_source(rows[b], h, w)
        far = torch.as_tensor(margin > 1e-4).to(DEV)
        assert int((~far).sum()) < max(1.0, 1e-3 * nq)
        src_t = torch.as_tensor(src).to(DEV)
        want = torch.where((src_t >= 0)[:, None], mine[src_t.clamp(min=0)], torch.zeros_like(mine)).to(out.dtype)
        got = out[:, b]
        assert torch.equal(got[far], want[far]), (angle, h, w)                     # the oracle's cells, zero fill outside
        img = mine.reshape(h, w, channels).permute(2, 0, 1).float()
        tv = rotate(img, angle, center=CENTER).permute(1, 2, 0).reshape(nq, channels).to(out.dtype)
        assert torch.equal(got[far], tv[far]), (angle, h, w)                       # torchvision on the same device
        if angle == 0.0:
            assert torch.equal(got, mine.to(out.dtype))                            # identity, exactly


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("batch_first", [True, False])
def test_rotate_bev_against_oracle_and_torchvision(dtype, batch_first):
    for h, w in SIZES:
        for k, angle in enumerate(ANGLES):
            _rotate_case(dtype, batch_first, h, w, [angle])
        _rotate_case(dtype, batch_first, h, w, [ANGLES[3], ANGLES[4]])             # bs 2, an angle per sample
        _rotate_case(dtype, batch_first, h, w, [ANGLES[0], ANGLES[5]])


def test_rotate_bev_casts_to_the_compute_dtype_and_takes_256_channels():
    _rotate_case(torch.float32, True, 50, 50, [3.0, -37.3], out_dtype=torch.bfloat16, channels=256)
    _rotate_case(torch.bfloat16, False, 40, 60, [0.5], out_dtype=torch.float32, channels=512)


# ---- bevf_ego_motion ------------------------------------------------------------------------------------------------
def _random_can_bus(n, seed=5):
    g = np.random.default_rng(seed)
    cb = g.standard_normal((n, 18))
    cb[:, :3] *= 3.0
    cb[:, -2] = g.uniform(-np.pi, np.pi, n)
    cb[:, -1] = g.uniform(-180.0, 180.0, n)
    cb[:8, :2] = 0.0                                   # dx = dy = 0: arctan2(0, 0) = 0 and length 0
    cb[8:12, -1] = 0.0                                 # a static heading: the identity rotation
    cb[12:14, -1] = [90.0, 180.0]
    return cb


@pytest.mark.parametrize("size", [(50, 50), (200, 200), (40, 60)])
def test_ego_motion_fp32_against_oracle(size):
    h, w = size
    gl = (0.512 * 200 / h, 0.512 * 200 / w)
    cb = _random_can_bus(300)
    before = _lib.launch_count()
    shift, rot, mlp_in = ops.ego_motion(torch.as_tensor(cb).to(DEV), h, w, gl, CENTER, True, torch.float32)
    assert _lib.launch_count() == before + 1
    want = ego_oracle.ego_shift(cb, h, w, gl).astype(np.float32)
    got = shift.cpu().numpy()
    assert np.all(np.abs(got - want) <= np.spacing(np.abs(want))), np.abs(got - want).max()     # one fp32 ulp
    assert np.array_equal(got[:8], np.zeros((8, 2), dtype=np.float32))
    rows = np.stack([ego_oracle.rotation_grid_rows(a, CENTER, h, w) for a in cb[:, -1]])
    r = rot.cpu().numpy()
    assert np.all(np.abs(r - rows) <= np.spacing(np.abs(rows))) and int((r != rows).sum()) <= 2
    assert np.array_equal(r[8:14], rows[8:14])         # 0, 90, 180 degrees: exactly torchvision's matrix
    assert torch.equal(mlp_in.cpu(), torch.as_tensor(cb).to(torch.float32))
    zero, _, _ = ops.ego_motion(torch.as_tensor(cb).to(DEV), h, w, gl, CENTER, False, torch.float32)
    assert not zero.any()                              # use_shift = False


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ego_motion_rounds_like_new_tensor(dtype):
    """The host path rounds shift and CAN-bus vector to the query dtype (``bev_queries.new_tensor``)."""
    h, w, gl = 50, 50, (2.048, 2.048)
    cb = _random_can_bus(64, seed=6) * 0.25
    shift, _, mlp_in = ops.ego_motion(torch.as_tensor(cb).to(DEV), h, w, gl, CENTER, True, dtype)
    assert shift.dtype == torch.float32 and mlp_in.dtype == dtype
    assert torch.equal(mlp_in.cpu(), torch.as_tensor(cb).to(dtype))
    want = torch.as_tensor(ego_oracle.ego_shift(cb, h, w, gl)).to(dtype).float()
    assert torch.equal(shift.cpu().to(dtype).float(), shift.cpu())                 # representable in the query dtype
    assert bool(((shift.cpu() - want).abs() <= want.abs() * torch.finfo(dtype).eps).all())


def test_ego_motion_stream_state():
    """Five frames, two scenes, a reset in the middle: deltas and state as forward_test keeps them."""
    w = syn.WORKLOADS["toy"]
    metas = sequence_inputs(w, frames=4)[3]
    seq = [np.asarray(metas[i]["can_bus"], dtype=np.float64) for i in (0, 1, 0, 2, 3)]
    fresh = [True, False, True, False, True]           # frame 2 follows a reset, frame 4 opens scene-b
    want, states = ego_oracle.stream_deltas(seq, fresh)
    state = ops.ego_state(DEV)
    gl = grid_length_of(w)
    for i, cb in enumerate(seq):
        if i == 2:
            state.zero_()
        # after the reset the host would ask for a new scene; CONTINUE on an empty state must give zeros too
        mode = ops.EGO_CONTINUE if (not fresh[i] or i == 2) else ops.EGO_NEW_SCENE
        t = torch.as_tensor(cb[None]).to(DEV)
        shift, rot, mlp_in = ops.ego_motion(t, w.bev_h, w.bev_w, gl, CENTER, True, torch.float32, state, mode)
        assert torch.equal(mlp_in.cpu()[0], torch.as_tensor(want[i]).float()), i
        s = ego_oracle.ego_shift(want[i][None], w.bev_h, w.bev_w, gl).astype(np.float32)
        assert np.all(np.abs(shift.cpu().numpy() - s) <= np.spacing(np.abs(s))), i
        rows = ego_oracle.rotation_grid_rows(want[i][-1], CENTER, w.bev_h, w.bev_w)
        assert np.all(np.abs(rot.cpu().numpy()[0] - rows) <= np.spacing(np.abs(rows))), i
        assert np.array_equal(state.view(torch.float64)[:3].cpu().numpy(), states[i][0]), i
        assert float(state.view(torch.float64)[3]) == states[i][1] and int(state[4]) == 1
        assert torch.equal(t.cpu()[0], torch.as_tensor(cb))                        # the input is not edited
    # without a state block the vector is taken as deltas
    _, _, plain = ops.ego_motion(torch.as_tensor(seq[1][None]).to(DEV), w.bev_h, w.bev_w, gl, CENTER, True,
                                 torch.float32)
    assert torch.equal(plain.cpu()[0], torch.as_tensor(seq[1]).float())


# ---- get_bev_features -----------------------------------------------------------------------------------------------
def _transformer(w, dtype, train=False):
    m = PerceptionTransformer(num_feature_levels=len(w.levels), num_cams=w.num_cams, encoder=syn.encoder_cfg(w),
                              decoder=None, embed_dims=w.embed_dims, rotate_center=[w.bev_h // 2, w.bev_w // 2])
    m.load_state_dict(syn.make_perception_state_dict(w))
    return m.to(DEV, dtype).train(train)


def _device_metas(metas):
    """(can_bus (bs, 18) f64, lidar2img (bs, cams, 4, 4) f32) on the device, and metas stripped of both."""
    cb = torch.as_tensor(np.array([m["can_bus"] for m in metas], dtype=np.float64)).to(DEV)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in metas], dtype=np.float32)).to(DEV)
    bare = [{k: v for k, v in m.items() if k not in ("can_bus", "lidar2img")} for m in metas]
    return cb, l2i, bare


GRAD_KEYS = ("can_bus_mlp.0.weight", "can_bus_mlp.norm.bias", "level_embeds",
             "encoder.layers.0.attentions.0.value_proj.weight", "encoder.layers.0.ffns.0.layers.1.weight")


@pytest.mark.parametrize("workload,bs,with_prev", [("toy", 2, True), ("toy", 1, False), ("tiny", 1, True)])
def test_get_bev_features_device_equals_host_fp32(workload, bs, with_prev):
    w = syn.WORKLOADS[workload]
    m = _transformer(w, torch.float32)
    inp = syn.make_perception_inputs(w, bs=bs, with_prev=with_prev, device=DEV)
    cb, l2i, bare = _device_metas(inp.img_metas)
    proj = torch.randn(bs, w.num_query, w.embed_dims, generator=torch.Generator().manual_seed(11)).to(DEV)
    results = []
    for device_path in (False, True):
        q = inp.bev_queries.clone().requires_grad_(True)
        m.zero_grad(set_to_none=True)
        kw = dict(img_metas=bare, can_bus=cb, lidar2img=l2i) if device_path else dict(img_metas=inp.img_metas)
        prev0 = None if inp.prev_bev is None else inp.prev_bev.clone()
        out = m.get_bev_features(inp.mlvl_feats, q, w.bev_h, w.bev_w, grid_length=grid_length_of(w),
                                 bev_pos=inp.bev_pos, prev_bev=inp.prev_bev, **kw)
        if prev0 is not None:
            assert torch.equal(prev0, inp.prev_bev)
        (out * proj).sum().backward()
        params = dict(m.named_parameters())
        results.append((out.detach(), q.grad.clone(), {k: params[k].grad.clone() for k in GRAD_KEYS}))
    (oh, gh, ph), (od, gd, pd) = results
    assert od.shape == (bs, w.num_query, w.embed_dims)
    assert max_err(od, oh) < 1e-3
    assert rel_err(gd, gh) < 1e-3
    for k in GRAD_KEYS:
        assert rel_err(pd[k], ph[k]) < 2e-3, k


@pytest.mark.parametrize("workload,bs,with_prev", [("toy", 2, True), ("toy", 1, False), ("tiny", 1, True)])
def test_get_bev_features_device_equals_host_bf16(workload, bs, with_prev):
    w = syn.WORKLOADS[workload]
    m = _transformer(w, torch.bfloat16)
    inp = syn.make_perception_inputs(w, bs=bs, with_prev=with_prev, device=DEV, dtype=torch.bfloat16)
    cb, l2i, bare = _device_metas(inp.img_metas)
    with torch.no_grad():
        host = m.get_bev_features(inp.mlvl_feats, inp.bev_queries, w.bev_h, w.bev_w, grid_length=grid_length_of(w),
                                  bev_pos=inp.bev_pos, prev_bev=inp.prev_bev, img_metas=inp.img_metas)
        dev = m.get_bev_features(inp.mlvl_feats, inp.bev_queries, w.bev_h, w.bev_w, grid_length=grid_length_of(w),
                                 bev_pos=inp.bev_pos, prev_bev=inp.prev_bev, img_metas=bare, can_bus=cb, lidar2img=l2i)
    assert dev.dtype == torch.bfloat16
    assert rel_err(dev.float(), host.float()) < 6e-2
    if with_prev and workload == "tiny":
        g = golden("perception_tiny")
        assert rel_err(dev.float()[:, g["rows_q"]], g["out_rows"]) < 6e-2


def test_device_path_refuses_prev_bev_with_gradient():
    w = syn.WORKLOADS["toy"]
    m = _transformer(w, torch.float32)
    inp = syn.make_perception_inputs(w, bs=1, with_prev=True, device=DEV)
    cb, l2i, bare = _device_metas(inp.img_metas)
    with pytest.raises(RuntimeError, match="host path"):
        m.get_bev_features(inp.mlvl_feats, inp.bev_queries, w.bev_h, w.bev_w, grid_length=grid_length_of(w),
                           bev_pos=inp.bev_pos, prev_bev=inp.prev_bev.clone().requires_grad_(True), img_metas=bare,
                           can_bus=cb, lidar2img=l2i)


# ---- temporal drivers -----------------------------------------------------------------------------------------------
def _sequence(w, dtype, frames=4):
    feats, q, pos, metas = sequence_inputs(w, frames)
    dfeats = [f.to(DEV, dtype) for f in feats]
    cb, l2i, bare = _device_metas(metas)                   # the frames along dim 0
    return dfeats, q.to(DEV, dtype), pos.to(DEV, dtype), metas, cb, l2i, bare


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_history_and_stream_device_path_against_reference_golden(dtype):
    g = golden("temporal_toy")
    w = syn.WORKLOADS["toy"]
    frames = int(g["meta"][0])
    dfeats, dq, dpos, metas, cb, l2i, bare = _sequence(w, dtype, frames)
    m = _transformer(w, dtype, train=True)
    tol = 1e-3 if dtype == torch.float32 else 6e-2
    deltas = cb[: frames - 1].clone()                      # training: the dataset hands over deltas
    deltas[1:, :3] -= cb[: frames - 2, :3]
    deltas[1:, -1] -= cb[: frames - 2, -1]
    deltas[0, :3] = 0
    deltas[0, -1] = 0
    hist = obtain_history_bev(m, [f[:, : frames - 1] for f in dfeats], [bare[: frames - 1]], dq, w.bev_h, w.bev_w, dpos,
                              grid_length_of(w), can_bus=deltas[None], lidar2img=l2i[None, : frames - 1])
    assert m.training and not hist.requires_grad
    assert rel_err(hist.float().cpu(), g["history"]) < tol
    stream = BEVStream(m)
    for i in range(frames):
        bev = stream.step([f[:, i] for f in dfeats], [bare[i]], dq, w.bev_h, w.bev_w, dpos, grid_length_of(w),
                          can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1])
        assert rel_err(bev.float().cpu(), g[f"stream{i}"]) < tol, i
    fresh = BEVStream(m).step([f[:, frames - 1] for f in dfeats], [bare[frames - 1]], dq, w.bev_h, w.bev_w, dpos,
                              grid_length_of(w), can_bus=cb[frames - 1:], lidar2img=l2i[frames - 1:])
    assert max_err(fresh, bev) == 0.0
    stream.reset()
    assert not stream.ego_state.any() and stream.prev_frame_info["prev_bev"] is None


def test_device_path_has_no_host_traffic():
    """After one warm-up frame (which sizes the pair list) a device-path step and a device-path history pass run
    with host synchronisation forbidden."""
    w = syn.WORKLOADS["toy"]
    dfeats, dq, dpos, metas, cb, l2i, bare = _sequence(w, torch.bfloat16)
    m = _transformer(w, torch.bfloat16)
    stream = BEVStream(m)
    gl = grid_length_of(w)
    stream.step([f[:, 0] for f in dfeats], [bare[0]], dq, w.bev_h, w.bev_w, dpos, gl, can_bus=cb[0:1], lidar2img=l2i[0:1])
    frames = [([f[:, i] for f in dfeats], cb[i:i + 1], l2i[i:i + 1]) for i in range(4)]
    hist_feats, hist_cb, hist_l2i = [f[:, :3] for f in dfeats], cb[None, :3].contiguous(), l2i[None, :3].contiguous()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in (1, 2, 3):                                # continuation, continuation, new scene
            stream.step(frames[i][0], [bare[i]], dq, w.bev_h, w.bev_w, dpos, gl, can_bus=frames[i][1],
                        lidar2img=frames[i][2])
        obtain_history_bev(m, hist_feats, [bare[:3]], dq, w.bev_h, w.bev_w, dpos, gl, can_bus=hist_cb,
                           lidar2img=hist_l2i)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    m.encoder.check_plan()


def _other_rig(l2i):
    """A second camera set-up: the rig yawed by 9 degrees and moved, so other queries are in view."""
    ang = np.deg2rad(9.0)
    rot = np.eye(4)
    rot[:2, :2] = [[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]]
    rot[:3, 3] = [1.5, -0.7, 0.1]
    return (l2i.double() @ torch.as_tensor(rot).to(l2i.device)).float()


def _run_sequence(stream, dfeats, bare, dq, w, dpos, cb, l2i, captured=False):
    outs = []
    for i in range(len(bare)):
        feats_i = [f[:, i] for f in dfeats]
        if captured:
            bev = stream.step(feats_i, [bare[i]], can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1])
        else:
            bev = stream.step(feats_i, [bare[i]], dq, w.bev_h, w.bev_w, dpos, grid_length_of(w), can_bus=cb[i:i + 1],
                              lidar2img=l2i[i:i + 1])
        outs.append(bev.clone())
    return outs


@pytest.mark.parametrize("workload,dtype", [("toy", torch.float32), ("tiny", torch.bfloat16)])
def test_captured_stream_equals_eager_device_path(workload, dtype):
    w = syn.WORKLOADS[workload]
    dfeats, dq, dpos, metas, cb, l2i, bare = _sequence(w, dtype)
    l2i_b = _other_rig(l2i)
    m = _transformer(w, dtype)
    eager_a = _run_sequence(BEVStream(m), dfeats, bare, dq, w, dpos, cb, l2i)
    eager_b = _run_sequence(BEVStream(m), dfeats, bare, dq, w, dpos, cb, l2i_b)
    assert max_err(eager_a[1], eager_b[1]) > 1e-2                                  # the rigs really differ
    stream = BEVStream(m)
    static = stream.capture([f[:, 0] for f in dfeats], [bare[0]], dq, w.bev_h, w.bev_w, dpos, grid_length_of(w),
                            can_bus=cb[0:1], lidar2img=l2i[0:1])
    assert static["can_bus"].shape == (1, 18) and static["lidar2img"].shape == l2i[0:1].shape
    before = _lib.launch_count()
    got_a = _run_sequence(stream, dfeats, bare, dq, w, dpos, cb, l2i, captured=True)
    got_b = _run_sequence(stream, dfeats, bare, dq, w, dpos, cb, l2i_b, captured=True)   # scene-b -> scene-a: new scene
    assert _lib.launch_count() == before                                           # replays, no launches from Python
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(got_a[i], eager_a[i]), i
        assert torch.equal(got_b[i], eager_b[i]), i
    # the returned BEV is the static output buffer
    last = stream.step(None, [bare[3]])
    assert last.data_ptr() == stream.prev_frame_info["prev_bev"].data_ptr()
    m.encoder.check_plan()
    stream.reset()
    again = stream.step([f[:, 0] for f in dfeats], [bare[0]], can_bus=cb[0:1], lidar2img=l2i[0:1])
    assert torch.equal(again, eager_a[0])
