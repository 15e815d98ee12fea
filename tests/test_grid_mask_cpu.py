"""GridMask on the host: the closed-form mask the kernel evaluates equals the reference's masks (goldens of
tests/golden/make_golden_grid_mask.py), the module makes the reference's np.random calls and hands the kernel the drawn
integers, and the variants no detector builds are refused at construction."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bevformer_b200 import ops
from bevformer_b200.plugin.grid_mask import GridMask
from tests import grid_mask_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = O.load_golden()
CASES = sorted(GOLD)


def test_golden_covers_the_issue_cases():
    sizes = {tuple(int(v) for v in c["shape"][2:]) for c in GOLD.values()}
    assert {(928, 1600), (736, 1280), (480, 800)} <= sizes
    assert any(h % 2 and w % 2 for h, w in sizes)
    modes = {c["mode"] for c in GOLD.values() if c["applied"]}
    assert modes == {0, 1}
    assert any(not c["use_h"] for c in GOLD.values()) and any(not c["use_w"] for c in GOLD.values())
    assert {0.0, 1.0} <= {float(c["ratio"]) for c in GOLD.values()}
    assert {0.0, 1.0} <= {float(c["prob"]) for c in GOLD.values()}
    assert any(not c["training"] for c in GOLD.values())
    near = [O.drawn(c) for c in GOLD.values() if c["applied"] and O.drawn(c)[0] == int(c["shape"][2]) - 1]
    assert any(st_h == d - 1 for d, _, st_h, _ in near) and any(st_w == d - 1 for d, _, _, st_w in near)


@pytest.mark.parametrize("name", CASES)
def test_closed_form_equals_reference_mask(name):
    c = GOLD[name]
    if not c["applied"]:
        assert (c["mask"] == 1).all()
        return
    h, w = c["mask"].shape
    want = O.closed_form_mask(h, w, *O.drawn(c), c["use_h"], c["use_w"], c["mode"])
    np.testing.assert_array_equal(want, c["mask"])


def _module(c):
    m = GridMask(bool(c["use_h"]), bool(c["use_w"]), rotate=1, offset=False, ratio=float(c["ratio"]),
                 mode=int(c["mode"]), prob=float(c["prob"]))
    return m.train(bool(c["training"]))


@pytest.mark.parametrize("name", CASES)
def test_module_draws_like_the_reference(name, monkeypatch):
    """Same np.random calls (kind, arguments, values, order) and end state as the reference; the kernel receives the
    drawn integers, the module's flags and the reference's view of the input."""
    c = GOLD[name]
    launched = []

    def fake(x, *args):
        launched.append((tuple(x.shape), args))
        return x
    monkeypatch.setattr(ops, "grid_mask", fake)
    m = _module(c)
    n, ch, h, w = (int(v) for v in c["shape"])
    x = torch.empty((n, ch, h, w), dtype=torch.uint8)
    np.random.seed(int(c["seed"]))
    with O.Recorder() as rec:
        y = m(x)
    assert np.random.rand() == float(c["next_rand"])
    kind, args, vals = rec.arrays()
    np.testing.assert_array_equal(kind, c["call_kind"])
    np.testing.assert_array_equal(args, c["call_args"])
    np.testing.assert_array_equal(vals, c["call_vals"])
    if not c["applied"]:
        assert y is x and not launched
        return
    d, l, st_h, st_w = O.drawn(c)
    assert m.l == l
    assert launched == [((n * ch, h, w), (d, l, st_h, st_w, bool(c["use_h"]), bool(c["use_w"]), int(c["mode"])))]
    assert y.shape == x.shape


def test_reference_attributes_and_set_prob():
    m = GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=0.7)
    assert (m.use_h, m.use_w, m.rotate, m.offset, m.ratio, m.mode, m.st_prob, m.prob, m.fp16_enable) == \
        (True, True, 1, False, 0.5, 1, 0.7, 0.7, False)
    m.set_prob(3, 24)
    assert m.prob == 0.7 * 3 / 24 and m.st_prob == 0.7


@pytest.mark.parametrize("kw", [dict(rotate=2), dict(rotate=360), dict(offset=True)], ids=str)
def test_variants_no_detector_builds_raise(kw):
    with pytest.raises(NotImplementedError, match="rotate|offset"):
        GridMask(True, True, **kw)


def test_unviewable_input_raises_after_one_draw():
    """The reference draws rand() and then fails in x.view(-1, h, w); so does the module."""
    m = GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=1.0)
    x = torch.empty(2, 3, 8, 10).to(memory_format=torch.channels_last)
    np.random.seed(0)
    with pytest.raises(RuntimeError, match="view"):
        m(x)
    after = np.random.rand()
    np.random.seed(0)
    np.random.rand()
    assert after == np.random.rand()


def test_kernel_entry_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.grid_mask(torch.ones(3, 4, 4), 2, 1, 0, 0)


@pytest.mark.skipif(not os.path.isfile(os.path.join(os.environ.get("BEVF_REFERENCE_ROOT", "/root/reference"),
                                                    "projects", "mmdet3d_plugin", "bevformer", "modules",
                                                    "encoder.py")),
                    reason="needs the reference checkout")
def test_package_path_coexists_with_the_oracle_stub():
    """oracle/mmcv_stub.py swaps projects.mmdet3d_plugin.models[.utils] in sys.modules while it imports the reference;
    the package imported before the stub runs is restored, and one imported after it is this package's."""
    code = (
        "import sys\n"
        "import projects.mmdet3d_plugin.models.utils as u\n"
        "from oracle import mmcv_stub\n"
        "mmcv_stub.load_reference_transformer()\n"
        "assert sys.modules['projects.mmdet3d_plugin.models.utils'] is u\n"
        "from projects.mmdet3d_plugin.models.utils.grid_mask import GridMask\n"
        "from bevformer_b200.plugin import GridMask as G\n"
        "assert GridMask is G and u.GridMask is G\n")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)
    code = (
        "from oracle import mmcv_stub\n"
        "mmcv_stub.load_reference_transformer()\n"
        "from projects.mmdet3d_plugin.models.utils import GridMask\n"
        "from bevformer_b200.plugin import GridMask as G\n"
        "assert GridMask is G\n")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)
