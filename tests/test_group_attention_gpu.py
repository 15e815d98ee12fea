"""Grouped attention kernel (csrc/attention.cu) and GroupMultiheadAttention on the GPU.

The kernel is checked against an fp64 torch restatement on the same 16-bit-rounded Q, K and V.  Bars follow the
rounding the kernel does (DESIGN.md §3): P is rounded to the storage type before P.V, dS before dS.K and dS^T.Q, Z^T
before Z^T.dO, and D = rowsum(dO * O) reads the rounded O.  Each output element may therefore be off by
4u * (|A| @ |B|) of its own product, with u the unit roundoff (2^-8 bf16, 2^-11 fp16), plus 1e-5 of max |ref| for
the fp32 accumulation and exp2 approximation."""
import warnings

import pytest
import torch

from bevformer_b200 import _lib, ops
from bevformer_b200 import synthetic as syn
from tests.test_group_attention_cpu import (CASES, DECODER_POINTS, case_inputs, decoder_inputs, golden_names, group_decoder_cfg,
                                            run_case, run_decoder, sampled_err)
from tests.util import reference_result

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")     # the key the ops use for the device-side dropout step counter
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}


def _groups(x, G):
    """(N, bs, H*32) -> (bs, G, H, N/G, 32)."""
    N, bs, C = x.shape
    return x.reshape(G, N // G, bs, C // 32, 32).permute(2, 0, 3, 1, 4)


def _ungroup(x):
    bs, G, H, L, D = x.shape
    return x.permute(1, 3, 0, 2, 4).reshape(G * L, bs, H * D)


def restate(q, k, v, do, G, scale, keep=None, drop_p=0.0):
    """fp64 forward, gradients and rounding bars of grouped attention; keep (bs, G, H, Lq, Lk) the dropout mask."""
    q, k, v, do = (t.detach().double().requires_grad_(True) for t in (q, k, v, do))
    qg, kg, vg, dog = _groups(q, G), _groups(k, G), _groups(v, G), _groups(do, G)
    p = torch.softmax(qg @ kg.transpose(-1, -2) * scale, -1)
    z = p if keep is None else p * keep.double() / (1.0 - drop_p)
    o = z @ vg
    dq, dk, dv = torch.autograd.grad(_ungroup(o), (q, k, v), do)
    with torch.no_grad():
        dz = dog @ vg.transpose(-1, -2)
        dp = dz if keep is None else dz * keep.double() / (1.0 - drop_p)
        dmat = (dog * o).sum(-1, keepdim=True)
        ds = p * (dp - dmat)
        ds_abs = ds.abs() + p * (dog.abs() * o.abs()).sum(-1, keepdim=True)
        bars = {"out": _ungroup(z.abs() @ vg.abs()), "dv": _ungroup(z.abs().transpose(-1, -2) @ dog.abs()),
                "dq": _ungroup(ds_abs @ kg.abs()) * scale, "dk": _ungroup(ds_abs.transpose(-1, -2) @ qg.abs()) * scale}
    return {"out": _ungroup(o).detach(), "dq": dq, "dk": dk, "dv": dv}, bars


def operands(nq, nk, bs, heads, dtype, seed, logit_scale=1.0):
    """Q, K, V as column slices of wider buffers (each its own row stride), plus dO."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = heads * 32
    qb = torch.randn(nq, bs, 3 * C, generator=g, device=DEV).to(dtype)
    kb = torch.randn(nk, bs, C + 64, generator=g, device=DEV).to(dtype)
    vb = torch.randn(nk, bs, C, generator=g, device=DEV).to(dtype)
    with torch.no_grad():
        qb[..., C:2 * C] *= logit_scale
    do = torch.randn(nq, bs, C, generator=g, device=DEV).to(dtype)
    return qb, kb, vb, do


def run_kernel(qb, kb, vb, do, heads, G, scale, drop_p=0.0):
    C = heads * 32
    qb, kb, vb = (t.detach().clone().requires_grad_(True) for t in (qb, kb, vb))
    q, k = qb[..., C:2 * C], kb[..., 64:]
    out = ops.GroupAttention.apply(q, k, vb, heads, G, scale, drop_p)
    out.backward(do)
    return {"out": out.detach(), "dq": qb.grad[..., C:2 * C], "dk": kb.grad[..., 64:], "dv": vb.grad}, (q, k, vb)


def check(got, want, bars, dtype):
    u = UNIT[dtype]
    for name in ("out", "dq", "dk", "dv"):
        err = (got[name].double() - want[name]).abs()
        bar = 4 * u * bars[name] + 1e-5 * want[name].abs().max()
        assert torch.isfinite(got[name]).all(), name
        worst = (err - bar).max().item()
        assert worst <= 0, f"{name}: exceeds its bar by {worst:.3g} (max err {err.max().item():.3g})"


# (group length of queries, of keys, groups, batch)
SHAPES = [(1, 1, 4, 2), (7, 7, 11, 1), (64, 64, 4, 2), (65, 65, 11, 2), (900, 900, 1, 1), (900, 900, 11, 1),
          (2048, 2048, 1, 2), (65, 7, 4, 1)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("lq,lk,G,bs", SHAPES)
def test_kernel_against_fp64_restatement(lq, lk, G, bs, dtype):
    heads = 8
    qb, kb, vb, do = operands(lq * G, lk * G, bs, heads, dtype, seed=lq + 7 * G)
    got, (q, k, v) = run_kernel(qb, kb, vb, do, heads, G, 32 ** -0.5)
    want, bars = restate(q, k, v, do, G, 32 ** -0.5)
    check(got, want, bars, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_kernel_large_logits(dtype):
    """Logits scaled by 30: the online softmax's running max must keep exp2 in range."""
    heads, G, L = 8, 4, 130
    qb, kb, vb, do = operands(L * G, L * G, 2, heads, dtype, seed=3, logit_scale=30.0)
    got, (q, k, v) = run_kernel(qb, kb, vb, do, heads, G, 32 ** -0.5)
    want, bars = restate(q, k, v, do, G, 32 ** -0.5)
    check(got, want, bars, dtype)


def test_backward_is_bitwise_reproducible_and_deterministic_mode_is_silent():
    heads, G = 8, 11
    qb, kb, vb, do = operands(9900, 9900, 1, heads, torch.bfloat16, seed=5)
    first, _ = run_kernel(qb, kb, vb, do, heads, G, 32 ** -0.5)
    torch.use_deterministic_algorithms(True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            second, _ = run_kernel(qb, kb, vb, do, heads, G, 32 ** -0.5)
    finally:
        torch.use_deterministic_algorithms(False)
    for name in first:
        assert torch.equal(first[name], second[name]), name


def test_abi_rejects_other_head_dims_and_fp32():
    lib = _lib.load()
    x = torch.zeros(64, 1, 256, device=DEV, dtype=torch.bfloat16)
    lse = torch.zeros(64 * 8, device=DEV)
    args = [x.data_ptr(), 256] * 4 + [lse.data_ptr(), 64, 64, 1, 8]
    assert lib.bevf_attn_forward(*args, 64, 1, 0.125, 0.0, 0, None, ops.BF16, None) != 0
    assert b"head_dim" in lib.bevf_last_error()
    assert lib.bevf_attn_forward(*args, 32, 1, 0.125, 0.0, 0, None, ops.F32, None) != 0
    assert b"bf16 or fp16" in lib.bevf_last_error()
    assert lib.bevf_attn_forward(*args, 32, 3, 0.125, 0.0, 0, None, ops.BF16, None) != 0
    torch.cuda.synchronize()


def _fixed_seed(monkeypatch, seed=0x1234567):
    monkeypatch.setattr(ops, "_next_seed", lambda: seed)
    return seed


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_dropout_against_restatement_with_exported_mask(monkeypatch, dtype):
    heads, G, L, bs, p = 8, 4, 100, 2, 0.1
    seed = _fixed_seed(monkeypatch)
    qb, kb, vb, do = operands(L * G, L * G, bs, heads, dtype, seed=11)
    C = heads * 32
    qb, kb, vb = (t.detach().clone().requires_grad_(True) for t in (qb, kb, vb))
    q, k = qb[..., C:2 * C], kb[..., 64:]
    out = ops.GroupAttention.apply(q, k, vb, heads, G, 32 ** -0.5, p)
    mask = ops.attention_dropout_mask(L * G, L * G, bs, heads, G, p, seed, ops.seed_state(DEV), DEV)
    ops.advance_seed(DEV)               # a later forward's step: the backward keeps its own forward's key
    out.backward(do)
    got = {"out": out.detach(), "dq": qb.grad[..., C:2 * C], "dk": kb.grad[..., 64:], "dv": vb.grad}
    want, bars = restate(q, k, vb, do, G, 32 ** -0.5, keep=mask, drop_p=p)
    check(got, want, bars, dtype)
    n = mask.numel()
    rate = mask.double().mean().item()
    assert abs(rate - (1 - p)) < 5 * (p * (1 - p) / n) ** 0.5, rate


def test_graph_replays_draw_new_masks():
    heads, G, L = 8, 4, 64
    qb, kb, vb, _ = operands(L * G, L * G, 1, heads, torch.bfloat16, seed=13)
    C = heads * 32
    q, k = qb[..., C:2 * C], kb[..., 64:]
    ops.advance_seed(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.advance_seed(DEV)
            ops.GroupAttention.apply(q, k, vb, heads, G, 32 ** -0.5, 0.1)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.advance_seed(DEV)
        out = ops.GroupAttention.apply(q, k, vb, heads, G, 32 ** -0.5, 0.1)
    graph.replay()
    first = out.clone()
    graph.replay()
    assert not torch.equal(first, out)


def _module(case, dtype):
    from bevformer_b200.plugin import GroupMultiheadAttention
    kw, _ = case_inputs(case)
    m = GroupMultiheadAttention(**kw).train(case[1])
    m.load_state_dict(syn.make_random_state_dict(m, 3))
    return m.to(DEV, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_module_against_reference_golden(case, dtype):
    """fp32 takes the torch path, bf16 the GEMM + kernel path except with a mask (torch path in bf16)."""
    want = reference_result(f"group_attn_{case[0]}")
    m = _module(case, dtype)
    _, t = case_inputs(case, dtype, DEV)
    before = _lib.launch_count()
    got = run_case(m, case, t)
    torch.cuda.synchronize()
    launched = _lib.launch_count() - before
    kernel_path = dtype != torch.float32 and not case[5]
    assert (launched > 0) == kernel_path, launched
    assert sorted(got) == golden_names(want)
    bar = 1e-4 if dtype == torch.float32 else 3e-2
    for k, v in got.items():
        assert sampled_err(v, want, k) < bar, k


@pytest.mark.parametrize("name,dtype", [("group_attn_decoder", torch.float32), ("group_attn_decoder_p8", torch.float32)])
def test_group_decoder_against_reference_golden(name, dtype):
    """The toy V2 decoder (3 layers, GroupMultiheadAttention group 4 over 40 queries, training mode, dropout off),
    with the configs' 4 sampling points and with 8 (a 192-wide offsets|weights head that the 16-bit GEMMs take)."""
    from bevformer_b200.plugin import build_transformer_layer_sequence
    want = reference_result(name)
    dec = build_transformer_layer_sequence(group_decoder_cfg(DECODER_POINTS[name])).train()
    dec.load_state_dict(syn.make_random_state_dict(dec, 5))
    dec = dec.to(DEV, dtype)
    t, kw = decoder_inputs(dtype, DEV)
    before = _lib.launch_count()
    got = run_decoder(dec, t, kw)
    torch.cuda.synchronize()
    assert _lib.launch_count() > before
    bar = 1e-4
    for k, v in got.items():
        assert sampled_err(v, want, k) < bar, k


def test_autocast_keeps_the_stacked_qk_projection():
    """Under autocast over fp32 inputs the self-attention's query and key stay one tensor, so Q and K are projected
    by one GEMM over the stacked [W_q; W_k] rows."""
    from bevformer_b200.plugin import GroupMultiheadAttention
    m = GroupMultiheadAttention(256, 8, group=4).to(DEV).train()
    x = torch.randn(40, 2, 256, device=DEV)
    pos = torch.randn_like(x)
    seen = []
    orig = ops.GroupAttention.apply

    def spy(q, k, *a):
        seen.append((tuple(q.shape), k is None))
        return orig(q, k, *a)
    ops.GroupAttention.apply = spy
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = m(x, x, x, query_pos=pos, key_pos=pos)
    finally:
        ops.GroupAttention.apply = orig
    assert y.dtype == torch.bfloat16 and seen == [((40, 2, 512), True)]


def test_cuda_graph_of_module_at_training_shape_matches_eager():
    from bevformer_b200.plugin import GroupMultiheadAttention
    torch.manual_seed(0)
    m = GroupMultiheadAttention(256, 8, dropout=0.0, group=11).to(DEV, torch.bfloat16).train()
    x = torch.randn(9900, 1, 256, device=DEV, dtype=torch.bfloat16)
    pos = torch.randn_like(x)
    gy = torch.randn_like(x)

    def step(xin):
        for p in m.parameters():
            p.grad = None
        y = m(xin, query_pos=pos)
        y.backward(gy)
        return y.detach(), xin.grad, [p.grad for p in m.parameters()]

    xe = x.clone().requires_grad_(True)
    ye, gxe, gpe = step(xe)
    ye, gxe, gpe = ye.clone(), gxe.clone(), [g.clone() for g in gpe]
    xs = x.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xs.grad = None
            step(xs)
    torch.cuda.current_stream().wait_stream(s)
    xs.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for p in m.parameters():
            p.grad = None
        yg = m(xs, query_pos=pos)
        yg.backward(gy)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, ye)
    assert torch.equal(xs.grad, gxe)
    for a, b in zip([p.grad for p in m.parameters()], gpe):
        assert (a.float() - b.float()).abs().max() <= 1e-2 * b.float().abs().max()
