"""fp16 storage in the kernels and the two mixed-precision mechanisms (torch.autocast, fp16 models) on the encoder
path.  Kernel results are compared against fp32 references computed on the SAME fp16-rounded inputs."""
import numpy as np
import pytest
import torch

from bevformer_b200 import ops, synthetic as syn
from oracle import msda_oracle
from tests.util import fixed_projection, golden, rel_err, stats

pytestmark = pytest.mark.gpu
DEV = "cuda"
H = torch.float16
TOL16 = 1e-2                     # the bf16 bar of the sampler tests; fp16 has three more mantissa bits


def _rig(which):
    from tools.bench_msda import rig_sca_inputs, rig_tsa_inputs, rig_tsa_rows_inputs
    if which == "sca":
        v, ss, lsi, loc, attn, row_map = rig_sca_inputs(DEV)
        return v, ss, lsi, loc, attn, row_map
    if which == "tsa_rows":
        v, ss, lsi, loc, attn, row_map, _ = rig_tsa_rows_inputs(DEV)
        return v, ss, lsi, loc, attn, row_map
    v, ss, lsi, loc, attn = rig_tsa_inputs(DEV)
    return v, ss, lsi, loc, attn, None


def _oracle_rows(fn, vr, ss, lsi, loc, attn, row_map, gout=None):
    """Oracle-S over a row list: one call per value map."""
    rm = row_map.cpu().long()
    outs = None
    for b in range(vr.shape[0]):
        idx = (rm == b).nonzero().flatten()
        if not idx.numel():
            continue
        args = [vr[b:b + 1], ss.cpu(), lsi.cpu(), loc[idx][None].contiguous(), attn[idx][None].contiguous()]
        if gout is not None:
            args.append(gout[idx][None].contiguous())
        r = fn(*args)
        r = r if isinstance(r, tuple) else (r,)
        if outs is None:
            outs = [torch.zeros(vr.shape), torch.zeros(loc.shape), torch.zeros(attn.shape)] if gout is not None \
                else [torch.zeros((loc.shape[0],) + r[0].shape[2:])]
        if gout is not None:
            outs[0][b] = r[0][0]; outs[1][idx] = r[1][0]; outs[2][idx] = r[2][0]
        else:
            outs[0][idx] = r[0][0]
    return outs


@pytest.mark.parametrize("which", ["sca", "tsa", "tsa_rows"])
def test_base_rig_fp16_against_oracle(which):
    """The base launches with fp16 value / out / grad_out: forward and all three gradients within the bf16 bars of
    Oracle-S run in fp32 on the fp16-rounded inputs."""
    v, ss, lsi, loc, attn, row_map = _rig(which)
    vh = v.to(H)
    nrows = loc.shape[0] if row_map is not None else loc.shape[0] * loc.shape[1]
    gout = fixed_projection((nrows, 256)).to(DEV, H)
    if row_map is not None:
        out = ops.msda_rows_forward(vh, ss, lsi, loc, attn, row_map)
        assert out.dtype == H
        gv, gl, ga = ops.msda_rows_backward(vh, ss, lsi, loc, attn, row_map, gout)
        (rout,) = _oracle_rows(msda_oracle.msda_forward, vh.float().cpu(), ss, lsi, loc.cpu(), attn.cpu(), row_map)
        rgv, rgl, rga = _oracle_rows(msda_oracle.msda_backward, vh.float().cpu(), ss, lsi, loc.cpu(), attn.cpu(),
                                     row_map, gout.float().cpu())
        used = (row_map >= 0).cpu()
        out, rout = out.float().cpu()[used], rout.reshape(rout.shape[0], -1)[used]
        gl, ga, rgl, rga = gl.cpu()[used], ga.cpu()[used], rgl[used], rga[used]
    else:
        out = ops.msda_forward(vh, ss, lsi, loc, attn)
        assert out.dtype == H
        gv, gl, ga = ops.msda_backward(vh, ss, lsi, loc, attn, gout.view(loc.shape[0], loc.shape[1], -1))
        rout = msda_oracle.msda_forward(vh.float().cpu(), ss.cpu(), lsi.cpu(), loc.cpu(), attn.cpu())
        rgv, rgl, rga = msda_oracle.msda_backward(vh.float().cpu(), ss.cpu(), lsi.cpu(), loc.cpu(), attn.cpu(),
                                                  gout.float().cpu().view(loc.shape[0], loc.shape[1], -1))
        out, gl, ga = out.float().cpu(), gl.cpu(), ga.cpu()
    torch.cuda.synchronize()
    assert gv.dtype == torch.float32
    errs = dict(out=rel_err(out, rout.reshape(out.shape)), gv=rel_err(gv.cpu(), rgv), gl=rel_err(gl, rgl),
                ga=rel_err(ga, rga))
    print(which, "fp16 vs Oracle-S", errs)
    for k, e in errs.items():
        assert e < TOL16, (k, e)


@pytest.mark.parametrize("dim", [4, 32, 64])
def test_head_dims_fp16_against_oracle(dim):
    """Generic head_dims (4, 64) and head_dim 32, fp16 value with fp16 and with fp32 output."""
    v, ss, lsi, loc, attn = syn.make_msda_inputs(2, [(6, 4), (3, 2)], 9, 2, dim, 2, seed=dim, loc_range=(-0.3, 1.3))
    vh = v.to(H)
    gout = fixed_projection((2, 9, 2 * dim)).to(H)
    d = [t.to(DEV) for t in (vh, ss, lsi, loc, attn)]
    out16 = ops.msda_forward(*d)
    gv, gl, ga = ops.msda_backward(*d, gout.to(DEV))
    rout = msda_oracle.msda_forward(vh.float(), ss, lsi, loc, attn)
    rgv, rgl, rga = msda_oracle.msda_backward(vh.float(), ss, lsi, loc, attn, gout.float())
    errs = (rel_err(out16.float().cpu(), rout), rel_err(gv.cpu(), rgv), rel_err(gl.cpu(), rgl), rel_err(ga.cpu(), rga))
    print("head_dim", dim, "fp16 errors", errs)
    assert out16.dtype == H and max(errs) < TOL16
    out32 = ops.msda_forward(*d, out_dtype=torch.float32)
    assert out32.dtype == torch.float32 and rel_err(out32.cpu(), rout) < 1e-5


def test_fixed_point_backward_fp16():
    """Deterministic mode with fp16 value / grad_out: bit-identical twice, within the bar of Oracle-S, and an fp16
    conversion of the fixed-point sums is available."""
    v, ss, lsi, loc, attn, row_map = _rig("sca")
    vh = v.to(H)
    gout = fixed_projection((loc.shape[0], 256)).to(DEV, H)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = ops.msda_backward_fx(vh, ss, lsi, loc, attn, gout, row_map)
        b = ops.msda_backward_fx(vh, ss, lsi, loc, attn, gout, row_map)
        ga, gb = a[0].materialize(), b[0].materialize()
        torch.cuda.synchronize()
        assert ga.dtype == H and torch.equal(ga, gb) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    finally:
        torch.use_deterministic_algorithms(prev)
    rgv, _, _ = _oracle_rows(msda_oracle.msda_backward, vh.float().cpu(), ss, lsi, loc.cpu(), attn.cpu(), row_map,
                             gout.float().cpu())
    e = rel_err(ga.float().cpu(), rgv)
    print("fixed-point fp16 grad_value vs Oracle-S", e)
    assert e < TOL16


GEMM_FWD = [
    # (M, N, K, relu, residual, fp32_out, bias dtype)
    (300, 256, 256, True, True, False, torch.float32),      # BN 256, ragged M tail
    (300, 192, 512, False, True, True, H),                  # BN 128, half-empty last column block, fp16 bias
    (4099, 320, 768, True, False, False, H),                # K = 768
    (77, 16, 2048, False, True, False, torch.float32),      # streamed kernel (reduction too long for the tile)
]


@pytest.mark.parametrize("case", GEMM_FWD)
def test_gemm_forward_fp16(case):
    M, N, K, relu, use_res, f32, bdt = case
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).to(DEV, H)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV, H)
    b = torch.randn(N, generator=g).to(DEV, bdt)
    res = torch.randn(M, N, generator=g).to(DEV, H) if use_res else None
    y = ops.linear_tc(x, w, b, res, relu, torch.float32 if f32 else None)
    ref = x.float() @ w.float().t() + b.float()
    if relu:
        ref = ref.relu()
    if use_res:
        ref = ref + res.float()
    assert y.dtype == (torch.float32 if f32 else H)
    err = (y.float() - ref).abs().max().item()
    print("fwd", case, err)
    assert err < (2e-3 if f32 else 1e-2)


@pytest.mark.parametrize("M,N,K,use_add", [(44511, 768, 256, True), (300, 192, 512, True), (4099, 128, 320, False)])
def test_gemm_dgrad_fp16(M, N, K, use_add):
    g = torch.Generator().manual_seed(M + N + K)
    dy = torch.randn(M, N, generator=g).to(DEV, H)
    w = (torch.randn(N, K, generator=g) / N ** 0.5).to(DEV, H)
    prev = torch.randn(M, K, generator=g).to(DEV, H) if use_add else None
    dx = ops.linear_dgrad_tc(dy, w, addend=prev)
    ref = dy.float() @ w.float()
    if use_add:
        ref = ref + prev.float()
    err = (dx.float() - ref).abs().max().item()
    print("dgrad", M, N, K, err)
    assert dx.dtype == H and err < 1e-2 * max(1.0, ref.abs().max().item() / 8)


@pytest.mark.parametrize("M,N,K", [(30000, 512, 256), (4099, 256, 768)])
def test_gemm_wgrad_fp16(M, N, K):
    """dW + db in the three forms: fp32 reductions, two-pass into the parameter dtype, two-pass accumulate-into."""
    g = torch.Generator().manual_seed(M)
    dy = torch.randn(M, N, generator=g).to(DEV, H)
    x = torch.randn(M, K, generator=g).to(DEV, H)
    rw, rb = dy.double().t() @ x.double(), dy.double().sum(0)
    dw, db = ops.linear_wgrad_tc(dy, x, with_bias=True)
    assert rel_err(dw, rw) < 1e-5 and rel_err(db, rb) < 1e-5
    for gdt in (torch.float32, H):
        dw2, db2 = ops.linear_wgrad_out(dy, x, gdt, True)
        assert dw2.dtype == gdt and rel_err(dw2.float(), rw) < (1e-5 if gdt == torch.float32 else 1e-3)
        assert rel_err(db2.float(), rb) < (1e-5 if gdt == torch.float32 else 1e-3)
    w0, b0 = torch.randn(N, K, generator=g).to(DEV), torch.randn(N, generator=g).to(DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    for det in (False, True):          # atomics form, and the two-pass fixed-order form of deterministic mode
        torch.use_deterministic_algorithms(det)
        try:
            acc_w, acc_b = w0.clone(), b0.clone()
            ops.linear_wgrad_into(dy, x, acc_w, acc_b)
        finally:
            torch.use_deterministic_algorithms(prev)
        assert rel_err(acc_w, w0.double() + rw) < 1e-5 and rel_err(acc_b, b0.double() + rb) < 1e-5, det


def test_elementwise_ops_fp16():
    """LayerNorm (fp32 and fp16 parameters), SCA combine, flatten, dropout, relu-dropout backward, colsum and
    sum_tensors in fp16 against torch fp32 on the rounded inputs."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(3, 700, 256, generator=g).to(DEV, H)
    res = torch.randn(3, 700, 256, generator=g).to(DEV, H)
    dy = torch.randn(3, 700, 256, generator=g).to(DEV, H)
    for pdt in (torch.float32, H):
        gamma = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV, pdt).requires_grad_(True)
        beta = (0.1 * torch.randn(256, generator=g)).to(DEV, pdt).requires_grad_(True)
        xi = x.clone().requires_grad_(True)
        y = ops.LayerNormResidual.apply(xi, res, gamma, beta, 1e-5, 0.0)
        y.backward(dy)
        xr = x.float().requires_grad_(True)
        gr, br = gamma.detach().float().requires_grad_(True), beta.detach().float().requires_grad_(True)
        yr = torch.nn.functional.layer_norm(xr + res.float(), (256,), gr, br, 1e-5)
        yr.backward(dy.float())
        assert y.dtype == H and rel_err(y.float(), yr) < 2e-3
        assert rel_err(xi.grad.float(), xr.grad) < 2e-3
        assert rel_err(gamma.grad.float(), gr.grad) < 2e-3 and rel_err(beta.grad.float(), br.grad) < 2e-3
    c = ops.colsum(x.view(-1, 256))
    assert rel_err(c, x.double().view(-1, 256).sum(0)) < 1e-5
    s = ops.sum_tensors([x, res, dy])
    assert s.dtype == H and rel_err(s.float(), x.float() + res.float() + dy.float()) < 1e-3
    h = torch.relu(x.clone())
    ops.dropout_inplace_(h, 0.25)
    kept = h != 0
    assert abs(kept.float().mean().item() - 0.75 * (x > 0).float().mean().item()) < 0.02
    assert rel_err(h.float()[kept], (torch.relu(x).float() / 0.75).to(H).float()[kept]) < 1e-3
    dz = ops.relu_dropout_backward(dy.view(-1, 256), h.view(-1, 256), 0.25)
    assert torch.equal(dz.view_as(dy), torch.where(kept, (dy.float() / 0.75).to(H), torch.zeros_like(dy)))
    feats = [torch.randn(1, 6, 256, 5, 7, generator=g).to(DEV, H)]
    ce, le = torch.randn(6, 256, generator=g).to(DEV), torch.randn(4, 256, generator=g).to(DEV)
    ff = ops.FlattenFeats.apply(ce, le, *feats)
    ref = (feats[0].flatten(3).permute(1, 3, 0, 2) + ce.to(H)[:, None, None, :]) + le[0].to(H)
    assert ff.dtype == H and torch.equal(ff, ref)
    # SCA combine: slots = mean over the cameras that see a query
    B, Nq, ncam = 1, 50, 3
    pair_of = torch.full((ncam, Nq), -1, dtype=torch.int32)
    pq = []
    for cam in range(ncam):
        for q in range(cam, Nq, 2):
            pair_of[cam, q] = len(pq)
            pq.append(q)
    pair_q = torch.tensor(pq, dtype=torch.int32)
    cnt = (pair_of >= 0).sum(0).clamp(min=1).float()
    inv = (1.0 / cnt)[None].to(DEV)
    out = torch.randn(len(pq), 256, generator=g).to(DEV, H)
    slots = ops.ScaCombine.apply(out, pair_of.to(DEV), pair_q.to(DEV), inv, B, Nq)
    rs = torch.zeros(Nq, 256)
    for cam in range(ncam):
        for q in range(Nq):
            if pair_of[cam, q] >= 0:
                rs[q] += out[pair_of[cam, q]].float().cpu()
    assert slots.dtype == H and rel_err(slots.float().cpu()[0], rs / cnt[:, None]) < 1e-3


def test_fp16_overflow_is_inf():
    """A projection, a LayerNorm output and a grad_value whose true value exceeds 65504 come out as inf."""
    x = torch.full((64, 64), 60.0, device=DEV, dtype=H)
    w = torch.full((16, 64), 30.0, device=DEV, dtype=H)                 # 64 * 60 * 30 = 115200
    y = ops.linear_tc(x, w)
    assert torch.isinf(y).all() and (y > 0).all()
    xl = torch.zeros(8, 256, device=DEV, dtype=H)
    xl[:, 0] = 1.0
    gamma = torch.full((256,), 1e4, device=DEV)                          # |y[:, 0]| = 1e4 * sqrt(255) ~ 1.6e5
    yl = ops.LayerNormResidual.apply(xl, None, gamma, torch.zeros(256, device=DEV), 1e-5, 0.0)
    assert torch.isinf(yl[:, 0]).all() and torch.isfinite(yl[:, 1:]).all()
    ss = torch.tensor([[1, 1]], device=DEV)
    lsi = torch.tensor([0], device=DEV)
    R, P = 64, 4
    value = torch.ones(1, 1, 1, 32, device=DEV, dtype=H)
    loc = torch.full((R, 1, 1, P, 2), 0.5, device=DEV)
    attn = torch.ones(R, 1, 1, P, device=DEV)
    gout = torch.full((R, 32), 60000.0, device=DEV, dtype=H)            # grad_value = 64 * 4 * 6e4 in fp32
    row_map = torch.zeros(R, dtype=torch.int32, device=DEV)
    gv, _, _ = ops.msda_rows_backward(value, ss, lsi, loc, attn, row_map, gout)
    assert gv.dtype == torch.float32 and torch.allclose(gv, torch.full_like(gv, R * P * 60000.0))
    assert torch.isinf(gv.to(H)).all()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        fx = ops.msda_backward_fx(value, ss, lsi, loc, attn, gout, row_map)[0]
        assert torch.isinf(fx.materialize()).all()                      # fp16 conversion in the kernel
    finally:
        torch.use_deterministic_algorithms(prev)


def _encoder(workload, dtype):
    from bevformer_b200.plugin import build_transformer_layer_sequence
    w = syn.WORKLOADS[workload]
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w, seed=0))
    return w, enc.to(DEV, dtype)


def _enc_inputs(w, dtype, with_prev=True):
    inp = syn.make_encoder_inputs(w, bs=1, seed=0, with_prev=with_prev)
    for k in ("bev_query", "feat", "bev_pos", "prev_bev"):
        if getattr(inp, k) is not None:
            setattr(inp, k, getattr(inp, k).to(DEV, dtype))
    inp.shift = inp.shift.to(DEV)
    inp.spatial_shapes, inp.level_start_index = inp.spatial_shapes.to(DEV), inp.level_start_index.to(DEV)
    return inp


@pytest.mark.parametrize("workload", ["toy", "tiny", "small4", "base"])
def test_encoder_half_model(workload):
    """model.half(): eval forward against the fp32 golden rows, backward within the bars of the bf16 test."""
    g = golden("encoder_" + workload)
    w, enc = _encoder(workload, H)
    enc.eval()
    inp = _enc_inputs(w, H)
    for t in (inp.bev_query, inp.feat, inp.bev_pos):
        t.requires_grad_(True)
    out = enc(inp.bev_query, inp.feat, inp.feat, **inp.kwargs())
    assert out.dtype == H
    e = rel_err(out.detach().float().cpu()[:, g["rows_q"]], g["out_rows"])
    print(workload, "fp16 forward vs fp32 golden", e)
    assert e < 6e-2
    (out.float() * fixed_projection(out.shape).to(DEV)).sum().backward()
    torch.cuda.synchronize()
    for got, want in ((inp.bev_query.grad.float().cpu()[g["rows_q"]], g["grad_query_rows"]),
                      (inp.feat.grad.float().cpu()[:, g["rows_s"]], g["grad_feat_rows"]),
                      (inp.bev_pos.grad.float().cpu()[g["rows_q"]], g["grad_pos_rows"])):
        want = torch.from_numpy(want)
        cos = torch.nn.functional.cosine_similarity(got.double().flatten(), want.double().flatten(), dim=0).item()
        assert cos > 0.99 and ((got - want).norm() / want.norm()).item() < 0.12
    for k, p in enc.named_parameters():
        assert p.grad.dtype == H
        got, ref = stats(p.grad.float()), g["gstat:" + k]
        assert abs(got[2] - ref[2]) / max(ref[2], 1e-12) <= 0.10, k


def _step(enc, inp, amp=None, scale=1.0):
    q = inp.bev_query.detach().clone().requires_grad_(True)
    f = inp.feat.detach().clone().requires_grad_(True)
    for p in enc.parameters():
        p.grad = None
    ctx = torch.autocast("cuda", dtype=amp) if amp is not None else torch.autocast("cuda", enabled=False)
    with ctx:
        out = enc(q, f, f, **inp.kwargs())
    (out.float() * fixed_projection(out.shape).to(DEV) * scale).sum().backward()
    torch.cuda.synchronize()
    return out.detach(), q.grad, f.grad, {k: p.grad for k, p in enc.named_parameters()}


@pytest.mark.parametrize("amp", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("arena", [False, True])
def test_autocast_fp32_weights(amp, arena):
    """autocast(bf16 / fp16) over fp32 weights: output in the autocast dtype, outputs and gradients as the all-16-bit
    model built from the same state dict, p.grad fp32."""
    w, enc32 = _encoder("tiny", torch.float32)
    _, enc16 = _encoder("tiny", amp)
    enc32.eval(); enc16.eval()
    if arena:
        enc32.enable_grad_arena()
    inp32, inp16 = _enc_inputs(w, torch.float32), _enc_inputs(w, amp)
    a = _step(enc32, inp32, amp)
    b = _step(enc16, inp16)
    # the bars of the bf16 encoder tests: the two runs differ in how biases and LayerNorm parameters are rounded
    assert a[0].dtype == amp
    e = rel_err(a[0].float(), b[0].float())
    print(amp, "arena" if arena else "", "autocast vs 16-bit model: output", e)
    assert e < 6e-2
    assert a[1].dtype == torch.float32
    for got, want in [(a[1], b[1]), (a[2], b[2])] + [(a[3][k], b[3][k]) for k in a[3]]:
        assert _close(got, want.float())
    for k in a[3]:
        assert a[3][k].dtype == torch.float32, k


def _close(got, want):
    got, want = got.double().flatten(), want.double().flatten()
    if want.norm() == 0:
        return got.norm() == 0
    cos = torch.nn.functional.cosine_similarity(got, want, dim=0).item()
    return cos > 0.99 and ((got - want).norm() / want.norm()).item() < 0.12


def test_kernel_inventory_under_autocast():
    """The autocast step launches the all-16-bit step's kernels plus ATen cast / copy kernels only (no cuBLAS GEMM,
    no ATen LayerNorm or other fallback).  The library's own kernels may appear in a second instantiation: LayerNorm
    reads fp32 parameters here (bevf::layernorm_*<T, float>) where the 16-bit model stores them in T."""
    from torch.profiler import ProfilerActivity, profile

    def names(enc, inp, amp):
        _step(enc, inp, amp)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _step(enc, inp, amp)
        return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}

    for amp in (torch.bfloat16, torch.float16):
        w, enc32 = _encoder("toy", torch.float32)
        _, enc16 = _encoder("toy", amp)
        enc32.train(); enc16.train()
        extra = names(enc32, _enc_inputs(w, torch.float32), amp) - names(enc16, _enc_inputs(w, amp), None)
        bad = [n for n in extra if not (n.startswith("void bevf::") or _is_copy_kernel(n))]
        print(amp, "extra kernels", sorted(extra))
        assert not bad, bad


def _is_copy_kernel(name):
    """ATen's dtype-conversion / copy kernels: ``Tensor.to`` (direct_copy_kernel_cuda), ``torch.cat``
    (CatArrayBatchedCopy)."""
    return "direct_copy_kernel" in name or "CatArrayBatchedCopy" in name or "copy_kernel" in name


def _gemm_names(names):
    """Vendor / ATen GEMM kernels (this library's own are bevf::gemm_*)."""
    return [n for n in names if not n.startswith("void bevf::")
            and any(s in n.lower() for s in ("gemm", "cutlass", "cublas", "xmma", "sm90_"))]


def test_module_entry_points_under_autocast():
    """TemporalSelfAttention, SpatialCrossAttention, MSDeformableAttention3D and FFN of an encoder layer, and
    CustomMSDeformableAttention, each called on its own: under autocast(bf16 / fp16) with fp32 weights each returns
    the autocast dtype, runs its projections on this library's GEMM (no cuBLAS) and agrees with its fp32 result
    within the bf16 bar."""
    from torch.profiler import ProfilerActivity, profile
    from bevformer_b200.plugin import CustomMSDeformableAttention
    from tests.test_decoder_attention import make_case, make_sd

    w, enc = _encoder("toy", torch.float32)
    enc.eval()
    inp = _enc_inputs(w, torch.float32)
    kw = inp.kwargs()
    layer = enc.layers[0]
    tsa, sca, ffn = layer.attentions[0], layer.attentions[1], layer.ffns[0]
    query, pos = inp.bev_query.permute(1, 0, 2).contiguous(), inp.bev_pos.permute(1, 0, 2).contiguous()
    ref_2d = enc._constants(w.bev_h, w.bev_w, 1, query.device)[0]
    ref_2d = torch.stack([ref_2d, ref_2d], 1).reshape(2, w.num_query, 1, 2)     # both queue entries (no prev_bev)
    plan = enc.prepare(kw["img_metas"], w.bev_h, w.bev_w, query.device)
    tsa_ss = torch.tensor([[w.bev_h, w.bev_w]], device=DEV)
    tsa_lsi = torch.zeros(1, dtype=torch.int64, device=DEV)
    ss, lsi = kw["spatial_shapes"], kw["level_start_index"]
    value_dense = inp.feat[0].permute(1, 0, 2).contiguous()                      # camera 0: (bs, S, C)
    dec = CustomMSDeformableAttention(num_levels=1, num_points=4)
    dec.load_state_dict(make_sd([(50, 50)], 4))
    case = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in make_case([(50, 50)], 900, 1, 2).items()}
    calls = {
        "TemporalSelfAttention": (tsa, (query,), dict(query_pos=pos, reference_points=ref_2d, spatial_shapes=tsa_ss,
                                                       level_start_index=tsa_lsi)),
        "SpatialCrossAttention": (sca, (query, inp.feat, inp.feat), dict(query_pos=pos,
                                                                          reference_points_cam=plan.ref_cam,
                                                                          spatial_shapes=ss, level_start_index=lsi,
                                                                          sca_plan=plan)),
        "MSDeformableAttention3D": (sca.deformable_attention, (query,),
                                    dict(value=value_dense, reference_points=plan.ref_cam[0].contiguous(),
                                         spatial_shapes=ss, level_start_index=lsi)),
        "FFN": (ffn, (query,), {}),
        "CustomMSDeformableAttention": (dec.to(DEV).eval(), (), case),
    }
    for name, (mod, args, kwargs) in calls.items():
        with torch.no_grad():
            ref = mod(*args, **kwargs)
            assert ref.dtype == torch.float32
            for amp in (torch.bfloat16, torch.float16):
                with torch.autocast("cuda", dtype=amp):
                    mod(*args, **kwargs)                                  # warm-up
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        out = mod(*args, **kwargs)
                        torch.cuda.synchronize()
                names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
                e = rel_err(out.float(), ref.float())
                print(name, amp, "vs fp32", e)
                assert out.dtype == amp, (name, amp, out.dtype)
                assert not _gemm_names(names), (name, _gemm_names(names))
                assert any(n.startswith("void bevf::gemm") for n in names), name
                assert e < 3e-2, (name, amp, e)


def test_autocast_cuda_graph_replay(monkeypatch):
    """An autocast(bf16) train step captured in a CUDA graph and replayed equals the eager step bit for bit
    (deterministic mode, so that the gradients' sums do not depend on scheduling)."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _graph_replay_case()
    finally:
        torch.use_deterministic_algorithms(prev)


def _graph_replay_case():
    w, enc = _encoder("tiny", torch.float32)
    enc.eval()
    inp = _enc_inputs(w, torch.float32)
    q = inp.bev_query.detach().clone().requires_grad_(True)
    f = inp.feat.detach().clone()
    proj = fixed_projection((1, w.num_query, 256)).to(DEV)
    kw = inp.kwargs()
    # the camera matrices as a resident device tensor: a captured step may not copy them from img_metas
    kw["lidar2img"] = torch.as_tensor(np.asarray([m["lidar2img"] for m in kw["img_metas"]], dtype=np.float32)).to(DEV)

    def step():
        q.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = enc(q, f, f, **kw)
        (out.float() * proj).sum().backward()
        return out

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step().detach().clone()
            eager_g = q.grad.clone()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_g, eager) and torch.equal(q.grad, eager_g)


def test_grad_scaler_fp16():
    """A few autocast(fp16) AdamW steps of the tiny encoder under GradScaler stay finite; with the scale forced to
    2^40 the overflow is found and the step skipped."""
    w, enc = _encoder("tiny", torch.float32)
    enc.train()
    inp = _enc_inputs(w, torch.float32)
    opt = torch.optim.AdamW(enc.parameters(), lr=1e-4)
    scaler = torch.amp.GradScaler("cuda")
    for _ in range(3):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            out = enc(inp.bev_query, inp.feat, inp.feat, **inp.kwargs())
        scaler.scale((out.float() * fixed_projection(out.shape).to(DEV)).sum()).backward()
        scaler.step(opt)
        scaler.update()
    assert all(torch.isfinite(p).all() for p in enc.parameters())
    before = {k: p.detach().clone() for k, p in enc.named_parameters()}
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.float16):
        out = enc(inp.bev_query, inp.feat, inp.feat, **inp.kwargs())
    scaler.scale((out.float() * fixed_projection(out.shape).to(DEV)).sum()).backward()
    scaler.step(opt)
    found = sum(v.item() for v in scaler._found_inf_per_device(opt).values())
    scaler.update()
    assert found > 0 and scaler.get_scale() < 2.0 ** 40
    for k, p in enc.named_parameters():
        assert torch.equal(p, before[k]), k


def test_fp16_enabled_perception_transformer():
    """fp16_enabled = True on PerceptionTransformer with fp16 features (what auto_fp16 hands it): the BEV embedding
    comes back in fp16 and matches the golden fp32 result within the bf16 bars."""
    from tests.test_transformer_gpu import _build, _grid_length
    g = golden("perception_tiny")
    w, pt = _build("tiny", torch.float32)
    pt.fp16_enabled = True
    inp = syn.make_perception_inputs(w, bs=1, with_prev=True, device=DEV)
    with torch.no_grad():
        out = pt.get_bev_features([f.half() for f in inp.mlvl_feats], inp.bev_queries, w.bev_h, w.bev_w,
                                  grid_length=_grid_length(w), bev_pos=inp.bev_pos, prev_bev=inp.prev_bev,
                                  img_metas=inp.img_metas)
    assert out.dtype == H
    e = rel_err(out.float().cpu()[:, g["rows_q"]], g["out_rows"])
    print("fp16_enabled get_bev_features vs golden", e)
    assert e < 6e-2


def test_deterministic_fp16_train_step():
    """Deterministic mode with an fp16 model: two train steps give bit-identical gradients."""
    w, enc = _encoder("tiny", H)
    enc.train()
    inp = _enc_inputs(w, H)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        res = []
        for _ in range(2):
            ops._seed_counter[0] = 0
            ops._seed_state.clear()
            ops._seed_snap.clear()
            res.append(_step(enc, inp))
    finally:
        torch.use_deterministic_algorithms(prev)
    a, b = res
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k
