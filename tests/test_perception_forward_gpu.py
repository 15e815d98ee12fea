"""PerceptionTransformer.forward on the GPU: the decoder's fused pieces (sampling-point prep with one frame, reference-
point refinement, self-attention on the attention kernel) against their torch expressions, the whole transformer
against the reference's own golden data, and the whole-frame video stream (no host synchronisation; captured graphs
equal to the eager frames)."""
import copy

import numpy as np
import pytest
import torch

from bevformer_b200 import _lib, ops, synthetic as syn
from bevformer_b200.plugin import BEVStream, PerceptionTransformer
from tests.golden.make_golden import grid_length_of, sequence_inputs, v2_inputs
from tests.util import fixed_projection, golden, max_err, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ulp_err(got, want):
    """max |got - want| in units of want's fp32 spacing (at least the spacing at 2^-10, for values near zero)."""
    want = want.double()
    spacing = torch.clamp(want.abs(), min=2.0 ** -10) * 2.0 ** -23
    return ((got.double() - want).abs() / spacing).max().item()


# ---- bevf_query_prep_* --------------------------------------------------------------------------------------------
def _prep_case(B, Nq, M, L, P, F, seed=0):
    g = torch.Generator().manual_seed(seed)
    raw = (torch.randn(B * Nq, M * F * L * P * 3, generator=g) * 3).to(DEV)
    ref = torch.rand(B * F, Nq, L, 2, generator=g).to(DEV)
    hw = torch.tensor([[13 + 7 * i, 29 - 5 * i] for i in range(L)], dtype=torch.int64, device=DEV)
    gl = torch.randn(B * F, Nq, M, L, P, 2, generator=g).to(DEV)
    ga = torch.randn(B * F, Nq, M, L, P, generator=g).to(DEV)
    return raw, ref, hw, gl, ga


def _decoder_prep_torch(raw, ref, hw, B, Nq, M, L, P):
    """plugin/decoder.py's torch expression of the sampling-point prep (decoder.py:300-330)."""
    n_off = M * L * P * 2
    raw = raw.reshape(B, Nq, -1)
    off = raw[..., :n_off].reshape(B, Nq, M, L, P, 2)
    att = raw[..., n_off:].reshape(B, Nq, M, L * P).softmax(-1).reshape(B, Nq, M, L, P)
    norm = torch.stack([hw[..., 1], hw[..., 0]], -1).to(torch.float32)
    loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    return loc, att


@pytest.mark.parametrize("M,L,P", [(8, 1, 4), (8, 2, 8), (4, 2, 3)])
def test_query_prep_one_frame_against_torch(M, L, P):
    """F = 1 (the decoder): loc / attn within a few fp32 ulp of the torch expression, d_raw against autograd."""
    B, Nq = 2, 37
    raw, ref, hw, gl, ga = _prep_case(B, Nq, M, L, P, 1)
    loc, att = ops.query_prep_forward(raw, ref, hw, B, Nq, M, L, P, 1)
    r = raw.clone().requires_grad_(True)
    wl, wa = _decoder_prep_torch(r, ref, hw, B, Nq, M, L, P)
    assert loc.shape == wl.shape and att.shape == wa.shape
    assert _ulp_err(loc, wl) <= 4 and _ulp_err(att, wa) <= 8
    torch.autograd.backward((wl, wa), (gl, ga))
    for dt in (torch.float32, torch.bfloat16):
        d_raw = ops.query_prep_backward(raw, gl, ga, hw, B, Nq, M, L, P, 1, out_dtype=dt)
        assert d_raw.dtype == dt
        assert rel_err(d_raw.float(), r.grad) < (1e-5 if dt == torch.float32 else 4e-3)


@pytest.mark.parametrize("M,L,P,interleave", [(8, 1, 4, False), (8, 1, 4, True), (8, 4, 8, False), (4, 2, 3, False)])
def test_query_prep_two_frames_is_tsa_prep_bit_for_bit(M, L, P, interleave):
    B, Nq = 2, 45
    raw, ref, hw, gl, ga = _prep_case(B, Nq, M, L, P, 2, seed=3)
    tl, ta = ops.tsa_prep_forward(raw, ref, hw, B, Nq, M, L, P, interleave)
    ql, qa = ops.query_prep_forward(raw, ref, hw, B, Nq, M, L, P, 2, interleave)
    assert torch.equal(tl, ql) and torch.equal(ta, qa)
    if interleave:
        gl, ga = gl.reshape(tl.shape), ga.reshape(ta.shape)
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        a = ops.tsa_prep_backward(raw, gl, ga, hw, B, Nq, M, L, P, interleave, out_dtype=dt)
        b = ops.query_prep_backward(raw, gl, ga, hw, B, Nq, M, L, P, 2, interleave, out_dtype=dt)
        assert torch.equal(a, b), dt


def test_query_prep_refuses_other_frame_counts():
    raw, ref, hw, _, _ = _prep_case(1, 4, 8, 1, 4, 1)
    with pytest.raises(RuntimeError, match="frames"):
        ops.query_prep_forward(raw, ref, hw, 1, 4, 8, 1, 4, 3)


# ---- bevf_refine_points -------------------------------------------------------------------------------------------
def _refine_torch(tmp, ref):
    """plugin/decoder.py's torch expression (decoder.py:106-118)."""
    from bevformer_b200.plugin import inverse_sigmoid
    new = torch.zeros_like(ref)
    new[..., :2] = tmp[..., :2] + inverse_sigmoid(ref[..., :2])
    new[..., 2:3] = tmp[..., 4:5] + inverse_sigmoid(ref[..., 2:3])
    return new.sigmoid()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_refine_points_against_torch(dtype):
    g = torch.Generator().manual_seed(4)
    bs, nq = 2, 900
    ref = torch.rand(bs, nq, 3, generator=g)
    ref[0, :6] = torch.tensor([0.0, 1.0, 1e-7, 1 - 1e-7, -0.5, 1.5])[:, None].expand(6, 3)   # the clamps
    tmp = torch.randn(bs, nq, 10, generator=g) * 2
    ref, tmp = ref.to(DEV, dtype), tmp.to(DEV, dtype)
    before = _lib.launch_count()
    got, ref2d = ops.refine_points(tmp, ref)
    assert _lib.launch_count() == before + 1
    want = _refine_torch(tmp, ref)
    assert got.dtype == dtype and got.shape == want.shape
    assert ref2d.dtype == torch.float32 and ref2d.shape == (bs, nq, 1, 2)
    assert torch.equal(ref2d[:, :, 0], got[..., :2].float())
    if dtype == torch.float32:
        # torch's own log / sigmoid are within an ulp or two each; through exp(s) a last-bit difference of the
        # inverse sigmoid grows by |s| relative to the result
        assert _ulp_err(got, want) <= 8
    else:
        assert max_err(got.float(), want.float()) <= 2.0 ** -8          # one bf16 step of values in [0.5, 1)
    # the regression output read in place through its row stride
    wide = torch.randn(bs, nq, 16, device=DEV).to(dtype)
    got2, _ = ops.refine_points(wide[..., 3:13], ref)
    assert torch.equal(got2, ops.refine_points(wide[..., 3:13].contiguous(), ref)[0])


# ---- MultiheadAttention on the attention kernel --------------------------------------------------------------------
def test_multihead_attention_takes_the_kernel_in_16_bit():
    from bevformer_b200.plugin import MultiheadAttention
    m = MultiheadAttention(256, 8, dropout=0.1)
    m.load_state_dict(syn.make_random_state_dict(m, 2))
    m = m.to(DEV).eval()
    g = torch.Generator().manual_seed(6)
    x, pos = (torch.randn(900, 2, 256, generator=g).to(DEV) for _ in range(2))
    with torch.no_grad():
        want = m(x, query_pos=pos)
        qp = x + pos
        direct = x + m.attn(query=qp, key=qp, value=x, attn_mask=None, key_padding_mask=None)[0]
        assert torch.equal(want, direct)                                # fp32: nn.MultiheadAttention itself
        mb = copy.deepcopy(m).to(torch.bfloat16)
        before = _lib.launch_count()
        got = mb(x.bfloat16(), query_pos=pos.bfloat16())
        assert _lib.launch_count() > before
        mask = torch.zeros(900, 900, dtype=torch.bool, device=DEV)
        before = _lib.launch_count()
        masked = mb(x.bfloat16(), query_pos=pos.bfloat16(), attn_mask=mask)
        assert _lib.launch_count() == before                            # masks keep nn.MultiheadAttention
    assert got.dtype == torch.bfloat16
    assert rel_err(got.float(), want) < 3e-2
    assert rel_err(masked.float(), want) < 3e-2
    # training: the kernel's dropout on the attention probabilities (the module's own output dropout off)
    mb.dropout_layer = torch.nn.Identity()
    mb.train()
    a = mb(x.bfloat16(), query_pos=pos.bfloat16())
    b = mb(x.bfloat16(), query_pos=pos.bfloat16())
    assert not torch.equal(a, b)


# ---- the whole transformer ----------------------------------------------------------------------------------------
W = syn.WORKLOADS["toy"]


def _transformer(dtype=torch.float32):
    m = PerceptionTransformer(num_feature_levels=len(W.levels), num_cams=W.num_cams, encoder=syn.encoder_cfg(W),
                              decoder=copy.deepcopy(syn.DECODER_CFG), embed_dims=W.embed_dims,
                              rotate_center=[W.bev_h // 2, W.bev_w // 2])
    m.load_state_dict(syn.make_random_state_dict(m, 0))
    return m.to(DEV, dtype).eval()


def _inputs(dtype):
    inp, oq, reg = v2_inputs(W)
    return (inp, [f.to(DEV, dtype) for f in inp.mlvl_feats], inp.bev_queries.to(DEV, dtype), oq.to(DEV, dtype),
            reg.to(DEV, dtype), inp.bev_pos.to(DEV, dtype), inp.prev_bev.to(DEV, dtype))


def _names_of_launched_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


def test_forward_fp32_against_reference_golden():
    g = golden("perception_forward_toy")
    m = _transformer()
    inp, feats, q, oq, reg, pos, prev = _inputs(torch.float32)
    q.requires_grad_(True)
    oq.requires_grad_(True)
    count = {"prep": 0, "refine": 0}
    real_prep, real_refine = ops.query_prep_forward, ops.refine_points

    def prep(*a, **k):
        count["prep"] += 1
        return real_prep(*a, **k)

    def refine(*a, **k):
        count["refine"] += 1
        return real_refine(*a, **k)

    ops.query_prep_forward, ops.refine_points = prep, refine
    try:
        before = _lib.launch_count()
        bev, states, ref0, refs = m(feats, q, oq, W.bev_h, W.bev_w, grid_length=list(grid_length_of(W)), bev_pos=pos,
                                    reg_branches=reg, cls_branches=None, prev_bev=prev, img_metas=inp.img_metas)
        launched = _lib.launch_count() - before
    finally:
        ops.query_prep_forward, ops.refine_points = real_prep, real_refine
    layers = syn.DECODER_CFG["num_layers"]
    assert count == {"prep": layers, "refine": layers}
    assert launched >= 2 * layers
    assert bev.shape == g["bev"].shape and states.shape == g["states"].shape and refs.shape == g["refs"].shape
    assert rel_err(bev.detach().cpu(), g["bev"]) < 1e-3
    assert rel_err(states.detach().cpu(), g["states"]) < 1e-3
    assert rel_err(ref0.detach().cpu(), g["ref0"]) < 1e-4 and rel_err(refs.cpu(), g["refs"]) < 1e-4
    (states * fixed_projection(states.shape).to(DEV)).sum().backward()
    assert rel_err(q.grad.cpu()[g["rows_q"]], g["grad_query_rows"]) < 2e-3
    assert rel_err(oq.grad.cpu(), g["grad_oq"]) < 2e-3


def test_forward_kernels_by_name():
    """The decoder's prep and refinement are the library's kernels (one frame: the M = 8 prep kernel)."""
    m = _transformer(torch.bfloat16)
    inp, feats, q, oq, reg, pos, prev = _inputs(torch.bfloat16)
    with torch.no_grad():
        _, names = _names_of_launched_kernels(
            lambda: m(feats, q, oq, W.bev_h, W.bev_w, grid_length=list(grid_length_of(W)), bev_pos=pos,
                      reg_branches=reg, prev_bev=prev, img_metas=inp.img_metas))
    assert any("tsa_prep_m8<2, false, float>" in n for n in names), sorted(names)
    assert any("refine_points_kernel<__nv_bfloat16>" in n for n in names), sorted(names)
    assert any("bevf::" in n and "attn_fwd" in n for n in names), sorted(names)


@pytest.mark.parametrize("mode", ["bf16", "autocast"])
def test_forward_16_bit_against_reference_golden(mode):
    g = golden("perception_forward_toy")
    dtype = torch.bfloat16 if mode == "bf16" else torch.float32
    m = _transformer(dtype)
    inp, feats, q, oq, reg, pos, prev = _inputs(dtype)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
        bev, states, ref0, refs = m(feats, q, oq, W.bev_h, W.bev_w, grid_length=list(grid_length_of(W)), bev_pos=pos,
                                    reg_branches=reg, cls_branches=None, prev_bev=prev, img_metas=inp.img_metas)
    assert states.dtype == torch.bfloat16 and bev.dtype == torch.bfloat16
    assert rel_err(bev.float().cpu(), g["bev"]) < 6e-2
    assert rel_err(states.float().cpu(), g["states"]) < 6e-2
    assert rel_err(refs.float().cpu(), g["refs"]) < 5e-2


# ---- the whole frame on the video path -----------------------------------------------------------------------------
def _sequence(dtype, frames=4):
    feats, q, pos, metas = sequence_inputs(W, frames)
    cb = torch.as_tensor(np.array([m["can_bus"] for m in metas], dtype=np.float64)).to(DEV)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in metas], dtype=np.float32)).to(DEV)
    bare = [{k: v for k, v in m.items() if k not in ("can_bus", "lidar2img")} for m in metas]
    _, oq, reg = v2_inputs(W)
    return ([f.to(DEV, dtype) for f in feats], q.to(DEV, dtype), pos.to(DEV, dtype), cb, l2i, bare,
            oq.to(DEV, dtype), reg.to(DEV, dtype))


def test_device_path_forward_does_not_synchronise():
    feats, q, pos, cb, l2i, bare, oq, reg = _sequence(torch.bfloat16)
    m = _transformer(torch.bfloat16)
    gl = list(grid_length_of(W))
    with torch.no_grad():
        first = m([f[:, 0] for f in feats], q, oq, W.bev_h, W.bev_w, grid_length=gl, bev_pos=pos, reg_branches=reg,
                  prev_bev=None, img_metas=bare[:1], can_bus=cb[0:1], lidar2img=l2i[0:1])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = m([f[:, 1] for f in feats], q, oq, W.bev_h, W.bev_w, grid_length=gl, bev_pos=pos, reg_branches=reg,
                    prev_bev=first[0], img_metas=bare[1:2], can_bus=cb[1:2], lidar2img=l2i[1:2])
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert len(out) == 4 and out[0].shape == (W.num_query, 1, W.embed_dims)
    m.encoder.check_plan()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_captured_whole_frame_stream_equals_eager(dtype):
    feats, q, pos, cb, l2i, bare, oq, reg = _sequence(dtype)
    m = _transformer(dtype)
    gl = grid_length_of(W)
    eager = []
    stream = BEVStream(m)
    for i in range(4):
        res = stream.step([f[:, i] for f in feats], [bare[i]], q, W.bev_h, W.bev_w, pos, gl, can_bus=cb[i:i + 1],
                          lidar2img=l2i[i:i + 1], object_query_embed=oq, reg_branches=reg)
        assert len(res) == 4 and stream.prev_frame_info["prev_bev"] is res[0]
        eager.append(tuple(t.clone() for t in res))
    # the BEV part is what the BEV-only stream computes
    bev_only = BEVStream(m).step([f[:, 0] for f in feats], [bare[0]], q, W.bev_h, W.bev_w, pos, gl, can_bus=cb[0:1],
                                 lidar2img=l2i[0:1])
    assert torch.equal(bev_only.permute(1, 0, 2), eager[0][0])
    stream = BEVStream(m)
    static = stream.capture([f[:, 0] for f in feats], [bare[0]], q, W.bev_h, W.bev_w, pos, gl, can_bus=cb[0:1],
                            lidar2img=l2i[0:1], object_query_embed=oq, reg_branches=reg)
    assert static["can_bus"].shape == (1, 18)
    before = _lib.launch_count()
    got = []
    for i in range(4):                                   # scene-a x 3, then scene-b: both graphs replay
        res = stream.step([f[:, i] for f in feats], [bare[i]], can_bus=cb[i:i + 1], lidar2img=l2i[i:i + 1])
        got.append(tuple(t.clone() for t in res))
    assert _lib.launch_count() == before
    torch.cuda.synchronize()
    for i in range(4):
        for a, b in zip(got[i], eager[i]):
            assert torch.equal(a, b), i
    m.encoder.check_plan()
