"""GridMask on the H100 against the reference's masks (tests/golden/ref_grid_mask.npz): for every golden case and
storage type the output and the gradient equal torch's multiply by the golden mask bit for bit, with inf, NaN and -0.0
under both mask values; no host synchronisation at the base size; eval mode, CUDA-graph capture and the reference's
view semantics."""
import numpy as np
import pytest
import torch

from bevformer_b200 import _lib
from bevformer_b200.plugin.grid_mask import GridMask
from tests import grid_mask_oracle as O

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}
BITS = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
GOLD = O.load_golden()
APPLIED = sorted(n for n, c in GOLD.items() if c["applied"])
DEV = torch.device("cuda")


def _module(c, training=None):
    m = GridMask(bool(c["use_h"]), bool(c["use_w"]), rotate=1, offset=False, ratio=float(c["ratio"]),
                 mode=int(c["mode"]), prob=float(c["prob"]))
    return m.train(bool(c["training"]) if training is None else training)


def _specials(shape, dtype, mask, seed):
    """Random normals with inf, -inf, NaN, -0.0, +0.0 planted on pixels under mask 0 and under mask 1 of every plane."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(shape, generator=g, device=DEV).to(dtype)
    h, w = mask.shape
    flat = x.view(-1, h * w)
    for value in (float("inf"), float("-inf"), float("nan"), -0.0, 0.0):
        for keep in (0.0, 1.0):
            idx = np.flatnonzero(mask.reshape(-1) == keep)
            if idx.size:
                pick = torch.from_numpy(np.random.RandomState(seed).choice(idx, min(4, idx.size), replace=False))
                flat[:, pick.to(DEV)] = value
    return x


def _same_bits(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    bits = BITS[a.dtype]
    diff = a.contiguous().view(bits) != b.contiguous().view(bits)
    assert not diff.any(), f"{int(diff.sum())} of {a.numel()} elements differ in their bits"


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
@pytest.mark.parametrize("name", APPLIED)
def test_output_and_gradient_bit_identical(name, dtype):
    c = GOLD[name]
    n, ch, h, w = (int(v) for v in c["shape"])
    mask = torch.from_numpy(c["mask"]).to(DEV, dtype)
    x = _specials((n, ch, h, w), dtype, c["mask"], 1).requires_grad_(True)
    before = _lib.launch_count()
    np.random.seed(int(c["seed"]))
    y = _module(c)(x)
    assert _lib.launch_count() - before == 1
    assert np.random.rand() == float(c["next_rand"])
    want = x.detach().view(-1, h, w) * mask
    _same_bits(y.detach(), want.view(n, ch, h, w))
    gy = _specials((n, ch, h, w), dtype, c["mask"], 2)
    y.backward(gy)
    _same_bits(x.grad, (gy.view(-1, h, w) * mask).view(n, ch, h, w))


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: DT[d])
def test_no_host_synchronisation_at_base_size(dtype):
    """The 6 x 3 x 928 x 1600 call runs under sync debug mode "error"; the reference's `.cuda()` of the mask raises."""
    c = GOLD["base_s0"]
    x = torch.randn(6, 3, 928, 1600, device=DEV).to(dtype)
    m = _module(c)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        np.random.seed(int(c["seed"]))
        y = m(x)
        with pytest.raises(RuntimeError):
            torch.from_numpy(c["mask"]).to(x.dtype).cuda()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    mask = torch.from_numpy(c["mask"]).to(DEV, dtype)
    _same_bits(y, (x.view(-1, 928, 1600) * mask).view(x.shape))


def test_eval_returns_input_after_one_draw():
    c = GOLD["eval"]
    x = torch.randn(*(int(v) for v in c["shape"]), device=DEV)
    m = _module(c)
    before = _lib.launch_count()
    np.random.seed(int(c["seed"]))
    assert m(x) is x
    assert np.random.rand() == float(c["next_rand"]) and _lib.launch_count() == before
    m.train(True)
    m.prob = 0.0                        # training, but the draw always says skip
    np.random.seed(0)
    assert m(x) is x
    after = np.random.rand()
    np.random.seed(0)
    np.random.rand()
    assert after == np.random.rand() and _lib.launch_count() == before


def test_capture_raises_in_train_mode():
    """A training-mode call on a capturing stream raises before it draws; an eval-mode call returns its input.  The
    refusal is caught inside the capture, so the capture itself ends normally and the graph replays."""
    x = torch.randn(2, 3, 32, 48, device=DEV)
    m = GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=1.0)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    raised = []
    with torch.cuda.graph(graph):
        y = x * 2
        state = np.random.get_state()[1].copy()
        try:
            m(y)
        except RuntimeError as e:
            raised.append(str(e))
        untouched = np.array_equal(np.random.get_state()[1], state)
        m.eval()
        z = m(y)
    graph.replay()
    torch.cuda.synchronize()
    assert len(raised) == 1 and "CUDA graph" in raised[0] and untouched
    assert z is y and torch.equal(y, x * 2)


def test_view_semantics():
    """A non-contiguous input that views as (-1, h, w) is masked like the reference's x.view(-1, h, w) * mask; an
    unviewable one raises as the reference's view does."""
    c = GOLD["odd_mode0"]
    n, ch, h, w = (int(v) for v in c["shape"])
    mask = torch.from_numpy(c["mask"]).to(DEV)
    base = torch.randn(n, ch, h, w + 5, device=DEV)
    x = base[..., :w]
    assert not x.is_contiguous()
    np.random.seed(int(c["seed"]))
    y = _module(c)(x)
    assert y.shape == (n, ch, h, w) and y.is_contiguous()
    _same_bits(y, (x.reshape(-1, h, w) * mask).view(n, ch, h, w))
    bad = torch.randn(n, ch, h, w, device=DEV).to(memory_format=torch.channels_last)
    np.random.seed(int(c["seed"]))
    with pytest.raises(RuntimeError, match="view"):
        _module(c)(bad)


def test_fp16_enabled_casts_like_auto_fp16():
    c = GOLD["tiny"]
    x = torch.randn(*(int(v) for v in c["shape"]), device=DEV)
    m = _module(c)
    m.fp16_enabled = True
    np.random.seed(int(c["seed"]))
    y = m(x)
    mask = torch.from_numpy(c["mask"]).to(DEV, torch.float16)
    _same_bits(y, (x.half().view(-1, 480, 800) * mask).view(x.shape))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two devices")
def test_runs_on_the_input_device():
    c = GOLD["odd_mode1"]
    x = torch.randn(*(int(v) for v in c["shape"]), device="cuda:1")
    np.random.seed(int(c["seed"]))
    y = _module(c)(x)
    assert y.device == x.device
    _same_bits(y, x * torch.from_numpy(c["mask"]).to(x.device))
