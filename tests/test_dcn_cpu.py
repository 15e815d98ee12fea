"""Modulated deformable convolution without a GPU: the float64 restatement (tests/dcn_fp64_oracle.py) against
torchvision.ops.deform_conv2d, the modules' parameters and checkpoint migration, the conv registry, and the op's
argument refusals."""
import math

import pytest
import torch

from tests import dcn_fp64_oracle as O

tv_ops = pytest.importorskip("torchvision.ops")

# (N, C, H, W, Cout, k, stride, padding, dilation, dg)
GEOMETRY = [
    (2, 8, 7, 9, 4, 3, 1, 1, 1, 1),
    (1, 8, 9, 8, 5, 3, 2, 0, 1, 2),
    (2, 16, 8, 8, 3, 3, 1, 2, 2, 4),
    (1, 8, 6, 7, 4, 1, 1, 0, 1, 2),
    (1, 4, 9, 9, 2, 1, 2, 1, 1, 1),
    (1, 12, 10, 6, 3, 3, 2, 1, 2, 4),
]


def _offsets(g, shape, scale, kind):
    """Offsets whose fp32 sum with the integer base is exact (multiples of 2^-12 on small maps), so the restatement's
    fp32 position equals torchvision's float64 one; ``kind`` adds integer positions and samples on the map's edges."""
    off = torch.round(torch.randn(shape, generator=g, dtype=torch.float64) * scale * 4096) / 4096
    if kind == "integer":
        off = torch.round(off)
    elif kind == "edges":
        # whole offsets far off the map, and positions landing exactly on -1 and on H / W
        off = off.clone()
        off.view(-1)[::3] = 40.0
        off.view(-1)[1::5] = -40.0
    return off


def _edge_case(N, C, H, W, k, dg, g):
    """Offsets that put sample (ho, wo) = (0, 0) of tap 0 at y = -1, x = W, and sample (0, 1) at y = H, x = -1: the
    boundaries of the sampling box, where nothing contributes."""
    Ho, Wo = H - k + 1, W - k + 1
    off = torch.zeros(N, 2 * dg * k * k, Ho, Wo, dtype=torch.float64)
    off[:, 0, 0, 0], off[:, 1, 0, 0] = -1.0, float(W)
    off[:, 0, 0, 1], off[:, 1, 0, 1] = float(H), -2.0
    off[:, 0, 1, 0], off[:, 1, 1, 0] = -0.5, float(W) - 1.5          # inside the box, corners off the map
    return off


def _tv(x, off, mask, w, b, stride, padding, dilation):
    return tv_ops.deform_conv2d(x, off, w, b, stride=stride, padding=padding, dilation=dilation, mask=mask)


def _compare(N, C, H, W, Cout, k, s, p, d, dg, off):
    g = torch.Generator().manual_seed(N * 1000 + C * 10 + k)
    stride, padding, dilation = (s, s), (p, p), (d, d)
    Ho, Wo = O.out_size(H, W, k, k, stride, padding, dilation)
    x = torch.randn(N, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cout, C, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    mask = torch.rand(N, dg * k * k, Ho, Wo, generator=g, dtype=torch.float64)
    dy = torch.randn(N, Cout, Ho, Wo, generator=g, dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in (x, off, mask, w, b)]
    ref = _tv(leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], stride, padding, dilation)
    ref.backward(dy)
    geom = O.geometry(x, w, stride, padding, dilation, dg)
    y, _ = O.forward(x, off, mask, w, b, geom)
    y = y.reshape(N, Ho, Wo, Cout).permute(0, 3, 1, 2)
    scale = ref.abs().max().item()
    assert (y - ref.detach()).abs().max().item() <= 1e-12 * scale
    grads = O.backward(x, off, mask, w, b, dy, geom)
    # torchvision's coordinate gradient skips mmcv's range test: on y == -1 or x == -1 exactly (the box edge, where
    # the far corner is still on the map) it is not zero.  mmcv's (and the restatement's) is; compare elsewhere.
    py, px = O.positions(off, geom)
    edge = ((py == -1) | (px == -1)).reshape(N, dg * k * k, 1, Ho, Wo).expand(-1, -1, 2, -1, -1)
    edge = edge.reshape(N, 2 * dg * k * k, Ho, Wo)
    assert grads["offset"][0][edge].abs().max().item() == 0 if edge.any() else True
    leaves[1].grad[edge] = 0
    for name, leaf in zip(("input", "offset", "mask", "weight", "bias"), leaves):
        want = leaf.grad
        got = grads[name][0]
        assert got.shape == want.shape, name
        assert (got - want).abs().max().item() <= 1e-12 * max(want.abs().max().item(), 1e-300), name


@pytest.mark.parametrize("case", GEOMETRY)
@pytest.mark.parametrize("kind", ["random", "integer", "edges"])
def test_restatement_matches_torchvision(case, kind):
    N, C, H, W, Cout, k, s, p, d, dg = case
    Ho, Wo = O.out_size(H, W, k, k, (s, s), (p, p), (d, d))
    g = torch.Generator().manual_seed(7)
    off = _offsets(g, (N, 2 * dg * k * k, Ho, Wo), 2.0, kind)
    _compare(N, C, H, W, Cout, k, s, p, d, dg, off)


def test_restatement_on_box_edges():
    N, C, H, W, k, dg = 1, 8, 6, 7, 3, 2
    off = _edge_case(N, C, H, W, k, dg, None)
    _compare(N, C, H, W, 4, k, 1, 0, 1, dg, off)
    # the two boundary samples contribute nothing and have zero offset / mask gradients
    x = torch.randn(N, C, H, W, dtype=torch.float64)
    w = torch.randn(4, C, k, k, dtype=torch.float64)
    mask = torch.ones(N, dg * k * k, H - 2, W - 2, dtype=torch.float64)
    dy = torch.randn(N, 4, H - 2, W - 2, dtype=torch.float64)
    geom = O.geometry(x, w, (1, 1), (0, 0), (1, 1), dg)
    gr = O.backward(x, off, mask, w, None, dy, geom)
    assert gr["mask"][0][0, 0, 0, :2].abs().max() == 0 and gr["offset"][0][0, :2, 0, :2].abs().max() == 0


def test_modules_parameters_and_initialisers():
    from bevformer_b200.plugin import ModulatedDeformConv2d, ModulatedDeformConv2dPack
    torch.manual_seed(0)
    m = ModulatedDeformConv2d(64, 32, 3, stride=2, padding=1, deform_groups=2)
    assert dict((k, tuple(v.shape)) for k, v in m.named_parameters()) == {"weight": (32, 64, 3, 3), "bias": (32,)}
    stdv = 1 / math.sqrt(64 * 9)
    assert m.weight.abs().max().item() <= stdv and m.weight.abs().max().item() > 0.9 * stdv
    assert m.bias.abs().max().item() == 0
    assert (m.stride, m.padding, m.dilation, m.groups, m.deform_groups) == ((2, 2), (1, 1), (1, 1), 1, 2)
    assert ModulatedDeformConv2d(8, 8, 1, bias=False).bias is None
    p = ModulatedDeformConv2dPack(64, 32, 3, padding=1, deform_groups=2, bias=False)
    shapes = dict((k, tuple(v.shape)) for k, v in p.named_parameters())
    assert shapes == {"weight": (32, 64, 3, 3), "conv_offset.weight": (2 * 3 * 9, 64, 3, 3),
                      "conv_offset.bias": (54,)}
    assert p.conv_offset.weight.abs().max() == 0 and p.conv_offset.bias.abs().max() == 0
    assert (p.conv_offset.stride, p.conv_offset.padding, p.conv_offset.dilation) == ((1, 1), (1, 1), (1, 1))
    assert p._version == 2


def test_build_conv_layer():
    from bevformer_b200.plugin import CONV_LAYERS, ModulatedDeformConv2dPack, build_conv_layer
    m = build_conv_layer(dict(type="DCNv2", deform_groups=1), 256, 256, kernel_size=3, stride=1, padding=1,
                         dilation=1, bias=False)
    assert type(m) is ModulatedDeformConv2dPack and m.bias is None and m.kernel_size == (3, 3)
    assert CONV_LAYERS.get("DCNv2") is ModulatedDeformConv2dPack
    assert type(build_conv_layer(None, 3, 8, 3)) is torch.nn.Conv2d
    assert type(build_conv_layer(dict(type="Conv"), 3, 8, 3)) is torch.nn.Conv2d
    with pytest.raises(KeyError):
        build_conv_layer(dict(type="NoSuchConv"), 3, 8, 3)
    with pytest.raises(TypeError):
        build_conv_layer("DCNv2", 3, 8, 3)


def test_version1_checkpoint_migrates_offset_conv():
    from bevformer_b200.plugin import build_conv_layer

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv2 = build_conv_layer(dict(type="DCNv2", deform_groups=1), 16, 16, kernel_size=3, padding=1,
                                          bias=False)
    src = Block()
    sd = {"conv2.weight": torch.randn(16, 16, 3, 3), "conv2_offset.weight": torch.randn(27, 16, 3, 3),
          "conv2_offset.bias": torch.randn(27)}
    dst = Block()
    dst.load_state_dict(sd)            # no version metadata: the original DCNv2 key names
    assert torch.equal(dst.conv2.conv_offset.weight, sd["conv2_offset.weight"])
    assert torch.equal(dst.conv2.conv_offset.bias, sd["conv2_offset.bias"])
    assert torch.equal(dst.conv2.weight, sd["conv2.weight"])
    # a current checkpoint round-trips, and carries version 2
    cur = src.state_dict()
    assert cur._metadata["conv2"]["version"] == 2
    Block().load_state_dict(cur)


def _args(N=1, C=64, H=6, W=6, Cout=64, k=3, dg=1, dtype=torch.bfloat16, off_c=None, mask_c=None, hw=None):
    Ho, Wo = hw or (H - k + 3, W - k + 3)
    x = torch.zeros(N, C, H, W, dtype=dtype)
    off = torch.zeros(N, off_c if off_c is not None else 2 * dg * k * k, Ho, Wo, dtype=dtype)
    mask = torch.zeros(N, mask_c if mask_c is not None else dg * k * k, Ho, Wo, dtype=dtype)
    w = torch.zeros(Cout, C, k, k, dtype=dtype)
    return x, off, mask, w


@pytest.mark.parametrize("bad", ["cpu", "offset_channels", "mask_channels", "offset_size", "mask_size",
                                 "dg_divides", "vector", "k_align", "n_align", "weight_channels"])
def test_refusals(bad):
    from bevformer_b200 import ops
    kw = {}
    if bad == "offset_channels":
        kw = dict(off_c=17)
    elif bad == "mask_channels":
        kw = dict(mask_c=8)
    elif bad == "dg_divides":
        kw = dict(C=64, dg=3)
    elif bad == "vector":
        kw = dict(C=32, dg=8, dtype=torch.float32)            # 4 channels per group < 8? fp32 needs 4: use bf16
        kw["dtype"] = torch.bfloat16
    elif bad == "k_align":
        kw = dict(C=40, k=1)
    elif bad == "n_align":
        kw = dict(Cout=48)
    x, off, mask, w = _args(**kw)
    if bad == "offset_size":
        off = off[..., :-1]
    elif bad == "mask_size":
        mask = mask[:, :, :-1]
    elif bad == "weight_channels":
        w = w[:, :32]
    with pytest.raises(RuntimeError):
        ops.modulated_deform_conv2d(x, off, mask, w, None, 1, 1, 1, 1, kw.get("dg", 1))


def test_groups_not_implemented():
    from bevformer_b200 import ops
    x, off, mask, w = _args()
    with pytest.raises(NotImplementedError):
        ops.modulated_deform_conv2d(x, off, mask, w, None, 1, 1, 1, 2, 1)


def test_cpu_tensors_refused_with_message():
    from bevformer_b200 import ops
    x, off, mask, w = _args()
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.modulated_deform_conv2d(x, off, mask, w, None, 1, 1, 1, 1, 1)


def test_fx_rules_match_the_library():
    from bevformer_b200 import _lib
    lib = _lib.load()
    for rows, kk in ((5800, 9), (1, 1), (34800, 9), (100, 1)):
        assert O.fx_frac_bits(rows, 1, kk) == lib.bevf_msda_fx_frac_bits(rows, 1, kk)
    assert O.fx_exponent(1.0, 1.0) == 2 and O.fx_exponent(0.75, 3.0) == 2
