"""GPU tests of SpatialCrossAttention's sampler with the sampling-point prep fused in (bevf_sca_rows_forward_fused /
bevf_sca_rows_backward_fused / bevf_sca_prep_backward_multi) against the unfused path on the same inputs: the prep
kernels (bevf_sca_prep_forward / _backward) around the row-list sampler.  The sampler output, the samples the
forward's statistics stand for, and d_raw must be bit-identical (no atomics on their paths); grad_value is summed with
atomics in both and is held to the 1e-2 bar of the mixed accumulation."""
import numpy as np
import pytest
import torch

from bevformer_b200 import ops, synthetic as syn
from bevformer_b200.plugin import ScaPlan
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
M, D = 8, 32


def _case(workload, bs, device_plan, seed=0):
    """Plan of the synthetic rig, raw head output (ring offsets + noise, random logits), value maps and grad_out."""
    w = syn.WORKLOADS[workload]
    metas = syn.make_img_metas(w, bs)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in metas], dtype=np.float32)).to(DEV)
    z = (torch.linspace(0.5, 7.5, w.pillar_points) / 8.0).tolist()
    ref_cam, mask = ops.point_sampling(l2i, syn.PC_RANGE, z, w.img_hw[0], w.img_hw[1], w.bev_h, w.bev_w)
    if device_plan:
        exact = ScaPlan.build(mask, ref_cam, (w.bev_h, w.bev_w))
        qorder = ScaPlan.tile_order(w.bev_h, w.bev_w, DEV)
        plan = ScaPlan.build_device(mask.to(torch.uint8).contiguous(), ref_cam, qorder, exact.num_pairs + 500)
    else:
        plan = ScaPlan.build(mask, ref_cam, (w.bev_h, w.bev_w))
    sd = syn.make_state_dict(w)
    g = torch.Generator().manual_seed(seed)
    nq, l, p = w.num_query, len(w.levels), w.sca_points
    bias = sd["layers.0.attentions.1.deformable_attention.sampling_offsets.bias"].view(1, -1)
    raw = torch.cat([bias + 0.5 * torch.randn(bs * nq, M * l * p * 2, generator=g),
                     torch.randn(bs * nq, M * l * p, generator=g)], 1).to(DEV).contiguous()
    ncam = w.num_cams
    value = torch.randn(bs * ncam, w.num_value, M, D, generator=g).to(DEV, torch.bfloat16)
    rows = plan.row_map.numel()
    gout = (0.1 * torch.randn(rows, M * D, generator=g)).to(DEV, torch.bfloat16)
    ss = torch.tensor(w.levels, dtype=torch.int64, device=DEV)
    lsi = torch.tensor(w.level_start, dtype=torch.int64, device=DEV)
    levels = [tuple(x) for x in w.levels]
    return dict(w=w, plan=plan, raw=raw, value=value, gout=gout, ss=ss, lsi=lsi, levels=levels, bs=bs, nq=nq, l=l, p=p)


def _run(c, fused):
    """(sampler output, grad_value bf16, d_raw bf16 [, stats]) of one forward + backward."""
    plan, raw, v, ss, lsi, levels = c["plan"], c["raw"], c["value"], c["ss"], c["lsi"], c["levels"]
    bs, nq, l, p = c["bs"], c["nq"], c["l"], c["p"]
    _, _, nfine = ops.gv_mode_for(plan.row_map.numel() / max(1, v.shape[0]), p, levels)
    kd = ops.dense_levels_for(plan.row_map.numel() / max(1, v.shape[0]), p, levels)
    dense = dict(map_range=plan.map_range, first_dense_level=max(kd, nfine)) if kd is not None else {}
    if fused:
        out, stats, coarse = ops.sca_rows_forward_fused(v, ss, lsi, raw, plan.ref_cam, plan.pair_q, plan.pair_cam,
                                                        plan.row_map, bs, nq, dense.get("first_dense_level"))
        gv, d_raw = ops.sca_rows_backward_fused(v, ss, lsi, levels, nfine, raw, stats, plan.ref_cam, plan.pair_q,
                                                plan.pair_cam, plan.pair_of, plan.row_map, c["gout"], bs, nq,
                                                coarse=coarse, **dense)
        if coarse is not None:                                # the stored coarse samples are the prep kernel's
            loc, attn = ops.sca_prep_forward(raw, plan.ref_cam, plan.pair_q, plan.pair_cam, ss, bs, nq, M, l, p)
            live = plan.row_map >= 0
            assert torch.equal(coarse[0][live], loc[live][:, :, coarse[2]:])
            assert torch.equal(coarse[1][live], attn[live][:, :, coarse[2]:])
        return out, gv.materialize(), d_raw, stats
    loc, attn = ops.sca_prep_forward(raw, plan.ref_cam, plan.pair_q, plan.pair_cam, ss, bs, nq, M, l, p)
    out = ops.msda_rows_forward(v, ss, lsi, loc, attn, plan.row_map)
    gv, gl, ga = ops.msda_rows_backward_mixed(v, ss, lsi, levels, nfine, loc, attn, plan.row_map, c["gout"], **dense)
    d_raw = ops.sca_prep_backward(raw, gl, ga, plan.pair_of, ss, bs, nq, plan.pair_q.numel(), M, l, p,
                                  out_dtype=torch.bfloat16)
    return out, gv, d_raw, (loc, attn)


CASES = [("base", 1, False), ("small4", 1, False), ("base", 1, True), ("base", 2, False), ("small4", 2, True)]


@pytest.mark.parametrize("workload,bs,device_plan", CASES,
                         ids=[f"{w}-bs{b}-{'device' if d else 'host'}" for w, b, d in CASES])
def test_fused_equals_prep_path(workload, bs, device_plan):
    c = _case(workload, bs, device_plan)
    out_f, gv_f, d_raw_f, stats = _run(c, True)
    out_u, gv_u, d_raw_u, (loc, attn) = _run(c, False)
    torch.cuda.synchronize()
    plan = c["plan"]
    live = plan.row_map >= 0
    if device_plan:
        assert not bool(live.all())                          # the fixed-capacity list has unused rows
    # queries seen by 0, 1 and 2+ cameras all occur (the finish kernel and the sampler epilogue both write d_raw)
    seen = (plan.pair_of >= 0).sum(0)
    assert {0, 1} <= set(seen.unique().tolist()) and int(seen.max()) >= 2
    assert torch.equal(out_f[live], out_u[live])
    assert torch.equal(d_raw_f, d_raw_u)
    # the forward's statistics stand for exactly the prep kernel's loc / attn
    raw, l, p = c["raw"], c["l"], c["p"]
    rows = live.nonzero().flatten()
    r = rows % plan.pair_q.numel()
    b = rows // plan.pair_q.numel()
    q = plan.pair_q[r].long()
    cam = plan.pair_cam[r].long()
    rq = raw[b * c["nq"] + q]                                 # (n, 768)
    lg = rq[:, M * l * p * 2:].view(-1, M, l * p)
    st = stats.view(-1, M, 2)[rows]
    a = torch.exp((lg - st[..., :1]).double()).float() * st[..., 1:]
    assert torch.equal(a.view(-1, M, l, p), attn[rows])
    off = rq[:, :M * l * p * 2].view(-1, M, l, p, 2)
    hw = c["ss"].float()
    zi = torch.arange(p, device=DEV) % plan.ref_cam.shape[3]
    ref = plan.ref_cam[cam, b, q][:, zi]                      # (n, P, 2)
    xy = ref[:, None, None] + off / torch.stack([hw[:, 1], hw[:, 0]], -1)[None, None, :, None]
    assert torch.equal(xy, loc[rows])
    err = rel_err(gv_f.float(), gv_u.float())
    print(workload, bs, device_plan, "grad_value fused vs prep path:", err)
    assert err < 1e-2


def _encoder(workload="base"):
    from bevformer_b200.plugin import build_transformer_layer_sequence
    w = syn.WORKLOADS[workload]
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w))
    enc = enc.to(DEV, torch.bfloat16).eval()                  # no dropout: eager and replayed steps agree
    host = syn.make_encoder_inputs(w, bs=1, seed=0)
    inp = {k: getattr(host, k).to(DEV, torch.bfloat16) for k in ("bev_query", "feat", "bev_pos", "prev_bev")}
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in host.img_metas], dtype=np.float32)).to(DEV)
    proj = torch.randn(1, w.num_query, w.embed_dims, device=DEV, dtype=torch.bfloat16,
                       generator=torch.Generator(DEV).manual_seed(3))
    ss, lsi, shift = host.spatial_shapes.to(DEV), host.level_start_index.to(DEV), host.shift.to(DEV)
    bq = inp["bev_query"].clone().requires_grad_(True)
    ft = inp["feat"].clone().requires_grad_(True)

    def step():
        for t in list(enc.parameters()) + [bq, ft]:
            t.grad = None
        out = enc(bq, ft, ft, bev_h=w.bev_h, bev_w=w.bev_w, bev_pos=inp["bev_pos"],
                  spatial_shapes=ss, level_start_index=lsi, prev_bev=inp["prev_bev"], shift=shift,
                  img_metas=host.img_metas, lidar2img=l2i)
        loss = (out * proj).float().sum()
        loss.backward()
        return out.detach().clone(), bq.grad.clone(), ft.grad.clone()

    return enc, step


def test_encoder_uses_fused_path_and_matches_unfused(monkeypatch):
    from bevformer_b200.plugin.spatial_cross_attention import SpatialCrossAttention
    calls = []
    orig = SpatialCrossAttention._fused_prep

    def spy(self, *a):
        calls.append(orig(self, *a))
        return calls[-1]

    enc, step = _encoder()
    monkeypatch.setattr(SpatialCrossAttention, "_fused_prep", spy)
    out_f, gq_f, gf_f = step()
    assert calls and all(calls)
    monkeypatch.setattr(SpatialCrossAttention, "_fused_prep", lambda self, *a: False)
    out_u, gq_u, gf_u = step()
    torch.cuda.synchronize()
    assert torch.equal(out_f, out_u)                          # forward bit-identical
    assert rel_err(gq_f.float(), gq_u.float()) < 1e-2
    assert rel_err(gf_f.float(), gf_u.float()) < 1e-2


def test_fallbacks_take_the_prep_path(monkeypatch):
    """Deterministic mode and an fp32 encoder never take the fused path."""
    from bevformer_b200.plugin.spatial_cross_attention import SpatialCrossAttention
    calls = []
    orig = SpatialCrossAttention._fused_prep
    monkeypatch.setattr(SpatialCrossAttention, "_fused_prep", lambda self, *a: calls.append(orig(self, *a)) or calls[-1])
    enc, step = _encoder("small4")
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        step()
    finally:
        torch.use_deterministic_algorithms(False)
    assert calls and not any(calls)
    calls.clear()
    enc.float()
    w = syn.WORKLOADS["small4"]
    host = syn.make_encoder_inputs(w, bs=1, seed=0)
    with torch.no_grad():
        enc(host.bev_query.to(DEV), host.feat.to(DEV), host.feat.to(DEV), bev_h=w.bev_h, bev_w=w.bev_w,
            bev_pos=host.bev_pos.to(DEV), spatial_shapes=host.spatial_shapes.to(DEV),
            level_start_index=host.level_start_index.to(DEV), prev_bev=host.prev_bev.to(DEV),
            shift=host.shift.to(DEV), img_metas=host.img_metas)
    assert not any(calls)


def test_cuda_graph_replay_matches_eager():
    """A captured base encoder step (forward + backward, device-built pair list) on the fused path replays to the
    eager step's output; gradients within the atomics' reordering."""
    enc, step = _encoder()
    out_e, gq_e, gf_e = step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    box = {}
    with torch.cuda.graph(g):
        box["r"] = step()
    g.replay()
    torch.cuda.synchronize()
    out_g, gq_g, gf_g = box["r"]
    assert torch.equal(out_g, out_e)
    assert rel_err(gq_g.float(), gq_e.float()) < 1e-2
    assert rel_err(gf_g.float(), gf_e.float()) < 1e-2
