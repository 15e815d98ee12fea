"""Modulated deformable convolution on the H100 against the float64 restatement (tests/dcn_fp64_oracle.py): every
output and gradient per element under its bar, in fp32, bf16 and fp16 storage, at the backbone's shapes; the exact
regime, the deterministic form, checkpointing, mixed precision, CUDA-graph capture and the launch count."""
import pytest
import torch

from tests import dcn_fp64_oracle as O

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}
# (N, C, H, W) of the DCN convs: base layer3 / layer4, small layer3; Cout = C, 3x3, stride 1, padding 1
SHAPES = {"base_l3": (6, 256, 58, 100), "base_l4": (6, 512, 29, 50), "small_l3": (6, 256, 46, 80)}
# the same channel counts at a reduced spatial size, for the full gradients
GRAD_SHAPES = {"base_l3": (2, 256, 12, 15), "base_l4": (2, 512, 9, 8), "small_l3": (2, 256, 10, 11)}
# (N, C, H, W, Cout, k, stride, padding, dilation, dg): the CPU file's geometry at channel counts the kernels take
GEOMETRY = [
    (2, 64, 7, 9, 64, 3, 1, 1, 1, 1),
    (1, 64, 9, 8, 64, 3, 2, 0, 1, 2),
    (2, 64, 8, 8, 64, 3, 1, 2, 2, 4),
    (1, 64, 6, 7, 64, 1, 1, 0, 1, 2),
    (1, 64, 9, 9, 128, 1, 2, 1, 1, 1),
    (1, 128, 10, 6, 64, 3, 2, 1, 2, 4),
]
WORST = {}


def _check(case, name, got, want, bar):
    err = (got.double() - want).abs()
    ratio = (err / bar).max().item() if err.numel() else 0.0
    key = (name, DT.get(got.dtype, str(got.dtype)))
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    bad = ~(err <= bar)
    assert not bad.any(), (f"{case} {name}: {int(bad.sum())} of {err.numel()} elements over the bar, worst err/bar "
                           f"{ratio:.3g}")


def _run(x, off, mask, w, b, dy, stride, padding, dilation, dg):
    from bevformer_b200 import ops
    leaves = [t.detach().clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, w, b)]
    y = ops.modulated_deform_conv2d(leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], stride, padding, dilation,
                                    1, dg)
    y.backward(dy)
    return y.detach(), [t.grad if t is not None else None for t in leaves]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
@pytest.mark.parametrize("shape", list(SHAPES), ids=str)
def test_forward_production_shapes(shape, dtype):
    from bevformer_b200 import ops
    N, C, H, W = SHAPES[shape]
    x, off, mask, w, b, _ = O.normal_inputs(N, C, H, W, C, 3, 3, (1, 1), (1, 1), (1, 1), 1, dtype, seed=1,
                                            device="cuda")
    with torch.no_grad():
        y = ops.modulated_deform_conv2d(x, off, mask, w, b, 1, 1, 1, 1, 1)
    assert y.is_contiguous(memory_format=torch.channels_last)
    geom = O.geometry(x, w, (1, 1), (1, 1), (1, 1), 1)
    g = torch.Generator().manual_seed(3)
    pix = torch.randperm(H * W, generator=g)[:700].cuda()           # 6 x 700 = 4200 output pixels
    want, bar = O.forward(x, off, mask, w, b, geom, pix)
    got = y.permute(0, 2, 3, 1).reshape(N, H * W, C)[:, pix].reshape(-1, C)
    _check(shape, "forward", got, want, bar)


def _grads(case, x, off, mask, w, b, dy, stride, padding, dilation, dg, deterministic=False):
    geom = O.geometry(x, w, stride, padding, dilation, dg)
    y, grads = _run(x, off, mask, w, b, dy, stride, padding, dilation, dg)
    want, bar = O.forward(x, off, mask, w, b, geom)
    N, Cout, Ho, Wo = y.shape
    _check(case, "forward", y.permute(0, 2, 3, 1).reshape(-1, Cout), want, bar)
    ref = O.backward(x, off, mask, w, b, dy, geom, deterministic=deterministic)
    for name, got in zip(("input", "offset", "mask", "weight", "bias"), grads):
        if got is None:
            continue
        assert got.dtype == {"weight": w.dtype, "bias": None if b is None else b.dtype}.get(name, x.dtype)
        _check(case, "grad_" + name + ("_fx" if deterministic and name == "input" else ""), got, *ref[name])
    return grads


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "fixed_point"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
@pytest.mark.parametrize("shape", list(GRAD_SHAPES), ids=str)
def test_gradients_reduced_size(shape, dtype, det):
    N, C, H, W = GRAD_SHAPES[shape]
    inp = O.normal_inputs(N, C, H, W, C, 3, 3, (1, 1), (1, 1), (1, 1), 1, dtype, seed=2, device="cuda")
    with _det(det):
        _grads(shape, *inp, (1, 1), (1, 1), (1, 1), 1, deterministic=det)


class _det:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *a):
        torch.use_deterministic_algorithms(self.prev)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
@pytest.mark.parametrize("case", GEOMETRY, ids=str)
def test_geometry(case, dtype):
    N, C, H, W, Cout, k, s, p, d, dg = case
    inp = O.normal_inputs(N, C, H, W, Cout, k, k, (s, s), (p, p), (d, d), dg, dtype, seed=4, device="cuda",
                          off_scale=3.0)
    _grads(str(case), *inp, (s, s), (p, p), (d, d), dg)


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "fixed_point"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
def test_exact_regime(dtype, det):
    """Integer inputs, quarter-pixel offsets, mask in {0, 1/2, 1}: every output and gradient is the float64 value
    rounded once to its storage type."""
    N, C, H, W, Cout, k, dg = 2, 64, 9, 11, 64, 3, 2
    x, off, mask, w, b, dy = O.exact_inputs(N, C, H, W, Cout, k, k, (1, 1), (1, 1), (1, 1), dg, dtype, seed=5,
                                            device="cuda")
    geom = O.geometry(x, w, (1, 1), (1, 1), (1, 1), dg)
    with _det(det):
        y, grads = _run(x, off, mask, w, b, dy, (1, 1), (1, 1), (1, 1), dg)
    want, _ = O.forward(x, off, mask, w, b, geom)
    assert torch.equal(y.permute(0, 2, 3, 1).reshape(-1, Cout).double(), O.rn(want, dtype))
    ref = O.backward(x, off, mask, w, b, dy, geom)
    for name, got in zip(("input", "offset", "mask", "weight", "bias"), grads):
        assert torch.equal(got.double(), O.rn(ref[name][0], got.dtype)), name
    WORST[("exact", DT[dtype])] = 0.0


def test_deterministic_repeats_bitwise():
    N, C, H, W = GRAD_SHAPES["base_l3"]
    inp = O.normal_inputs(N, C, H, W, C, 3, 3, (1, 1), (1, 1), (1, 1), 1, torch.bfloat16, seed=6, device="cuda",
                          off_scale=0.7)      # small offsets: many samples share pixels, so the scatter collides
    with _det(True):
        a = _run(*inp, (1, 1), (1, 1), (1, 1), 1)[1]
        b = _run(*inp, (1, 1), (1, 1), (1, 1), 1)[1]
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def _bottleneck(dev, dtype):
    """A caffe-style ResNet Bottleneck with DCNv2 on conv2 and frozen BN, as mmdet builds it (stride on the 1x1)."""
    from bevformer_b200.plugin import build_conv_layer
    torch.manual_seed(0)

    class Bottleneck(torch.nn.Module):
        def __init__(self, c=256, mid=64):
            super().__init__()
            self.conv1 = build_conv_layer(None, c, mid, 1, bias=False)
            self.conv2 = build_conv_layer(dict(type="DCNv2", deform_groups=1), mid, mid, kernel_size=3, stride=1,
                                          padding=1, dilation=1, bias=False)
            self.conv3 = build_conv_layer(None, mid, c, 1, bias=False)
            self.bn = torch.nn.ModuleList(torch.nn.BatchNorm2d(n) for n in (mid, mid, c))
            for bn in self.bn:
                bn.eval()
                bn.weight.data.uniform_(0.5, 1.5)
                bn.running_var.uniform_(0.5, 1.5)
                for p in bn.parameters():
                    p.requires_grad_(False)
            with torch.no_grad():
                self.conv2.conv_offset.weight.normal_(0, 0.05)
                self.conv2.conv_offset.bias.normal_(0, 0.5)

        def _inner(self, x):
            h = torch.relu(self.bn[0](self.conv1(x)))
            h = torch.relu(self.bn[1](self.conv2(h)))
            return self.bn[2](self.conv3(h))

        def forward(self, x, with_cp=False):
            h = torch.utils.checkpoint.checkpoint(self._inner, x, use_reentrant=False) if with_cp else self._inner(x)
            return torch.relu(h + x)
    return Bottleneck().to(dev, dtype)


def test_checkpoint_bottleneck_bitwise():
    m = _bottleneck("cuda", torch.float32)
    x = torch.randn(2, 256, 12, 15, device="cuda")
    dy = torch.randn(2, 256, 12, 15, device="cuda")
    out = []
    with _det(True):
        for cp in (False, True):
            m.zero_grad()
            xi = x.clone().requires_grad_(True)
            m(xi, with_cp=cp).backward(dy)
            out.append([xi.grad] + [p.grad.clone() for p in m.parameters() if p.requires_grad])
    assert len(out[0]) == 6                   # x; conv1, conv2, its conv_offset weight and bias, conv3 (BN frozen)
    for u, v in zip(*out):
        assert torch.equal(u, v)


def test_pack_conv_offset_gradients():
    """The Pack module's conv_offset parameters get the gradient of the chain chunk -> cat / sigmoid -> the op: the
    op's grad_offset / grad_mask (checked against the restatement above) through cuDNN's convolution, here against
    the same chain in float64 with the restatement's gradients."""
    from bevformer_b200.plugin import ModulatedDeformConv2dPack
    torch.manual_seed(1)
    m = ModulatedDeformConv2dPack(64, 64, 3, padding=1).cuda()
    with torch.no_grad():
        m.conv_offset.weight.normal_(0, 0.05)
        m.conv_offset.bias.normal_(0, 0.5)
        m.bias.normal_()
    x = torch.randn(2, 64, 9, 10, device="cuda", requires_grad=True)
    dy = torch.randn(2, 64, 9, 10, device="cuda")
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):       # conv_offset in fp32, not TF32
        m(x).backward(dy)
    # float64 chain on the restatement
    w64 = m.conv_offset.weight.detach().double().requires_grad_(True)
    b64 = m.conv_offset.bias.detach().double().requires_grad_(True)
    out = torch.nn.functional.conv2d(x.detach().double(), w64, b64, 1, 1)
    o1, o2, ml = torch.chunk(out, 3, 1)
    off, mk = torch.cat((o1, o2), 1), torch.sigmoid(ml)
    geom = O.geometry(x, m.weight, (1, 1), (1, 1), (1, 1), 1)
    ref = O.backward(x.detach().float(), off.detach().float(), mk.detach().float(), m.weight.detach(),
                     m.bias.detach(), dy, geom)
    torch.autograd.backward([off, mk], [ref["offset"][0], ref["mask"][0]])
    for got, want in ((m.conv_offset.weight.grad, w64.grad), (m.conv_offset.bias.grad, b64.grad)):
        err = (got.double() - want).abs().max().item() / want.abs().max().item()
        WORST[("pack_conv_offset (rel. to max)", "f32")] = max(WORST.get(("pack_conv_offset (rel. to max)", "f32"), 0),
                                                               err)
        assert err < 1e-4, err


@pytest.mark.parametrize("mode", ["autocast_bf16", "fp16_enabled"])
def test_mixed_precision_runs_16bit_kernels(mode, monkeypatch):
    """The sampling kernels receive 16-bit tensors (recorded at the entry of both sampling calls) and the library's
    launch count moves.  (No torch.profiler here: a profiling session in this process changed how a later session
    named the non-template kernel bevf::point_sampling_kernel, and kernel inventories compare names.)"""
    from bevformer_b200 import _lib, ops
    from bevformer_b200.plugin import ModulatedDeformConv2dPack
    m = ModulatedDeformConv2dPack(64, 64, 3, padding=1).cuda()
    x = torch.randn(2, 64, 9, 10, device="cuda", requires_grad=True)
    ref = m(x)
    seen = []
    for fn in ("dcn_sampling_forward", "dcn_sampling_backward"):
        orig = getattr(ops, fn)
        monkeypatch.setattr(ops, fn, lambda xs, *a, _f=orig, _n=fn: (seen.append((_n, xs.dtype)), _f(xs, *a))[1])
    before = _lib.launch_count()
    if mode == "autocast_bf16":
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = m(x)
        want = torch.bfloat16
    else:
        m.fp16_enabled = True
        y = m(x)
        want = torch.float16
    y.float().sum().backward()
    torch.cuda.synchronize()
    assert y.dtype == want and _lib.launch_count() - before >= 4
    assert {n for n, _ in seen} == {"dcn_sampling_forward", "dcn_sampling_backward"}
    assert all(dt == want for _, dt in seen), seen
    err = (y.float() - ref.detach()).abs().max().item() / ref.abs().max().item()
    assert err < 3e-2, err
    assert m.weight.grad.dtype == torch.float32 and torch.isfinite(x.grad).all()


def test_cuda_graph_capture_replays_eager():
    from bevformer_b200 import ops
    N, C, H, W = 2, 256, 12, 15
    x, off, mask, w, b, dy = O.normal_inputs(N, C, H, W, C, 3, 3, (1, 1), (1, 1), (1, 1), 1, torch.bfloat16, seed=8,
                                             device="cuda")
    leaves = [t.clone().requires_grad_(True) for t in (x, off, mask, w, b)]

    def step():
        for t in leaves:
            t.grad = None
        y = ops.modulated_deform_conv2d(*leaves, 1, 1, 1, 1, 1)
        y.backward(dy)
        return y

    with _det(True):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()                                  # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        eager_y = step().detach().clone()
        eager_g = [t.grad.clone() for t in leaves]
        for t in leaves:
            t.grad = None
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            gy = step()
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(gy, eager_y)
    for t, e in zip(leaves, eager_g):
        assert torch.equal(t.grad, e)


def test_launch_count_and_empty_batch():
    from bevformer_b200 import _lib, ops
    x, off, mask, w, b, dy = O.normal_inputs(1, 64, 6, 7, 64, 3, 3, (1, 1), (1, 1), (1, 1), 1, torch.bfloat16,
                                             seed=9, device="cuda")
    before = _lib.launch_count()
    y, _ = _run(x, off, mask, w, b, dy, (1, 1), (1, 1), (1, 1), 1)
    torch.cuda.synchronize()
    assert _lib.launch_count() - before >= 5        # im2col, GEMM, im2col again, dgrad, wgrad, col2im
    before = _lib.launch_count()
    y = ops.modulated_deform_conv2d(x[:0], off[:0], mask[:0], w, b, 1, 1, 1, 1, 1)
    assert y.shape == (0, 64, 6, 7) and _lib.launch_count() == before


def test_summary():
    """The worst err/bar of every (path, storage type), as checked above."""
    assert WORST, "no case ran"
    print("\nDCN worst err/bar")
    for (name, dt), r in sorted(WORST.items()):
        print(f"  {name:34s} {dt:5s} {r:.3g}")
