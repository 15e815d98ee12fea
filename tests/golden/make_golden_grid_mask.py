"""Generates the GridMask goldens from the REFERENCE'S OWN GridMask (projects/mmdet3d_plugin/models/utils/grid_mask.py),
loaded by path behind oracle/mmcv_stub.py (mmcv's auto_fp16 is the stub's identity decorator) with ``Tensor.cuda``
as the identity, so it runs on the CPU.  Needs a reference checkout (BEVF_REFERENCE_ROOT) and PIL; the test suite
needs neither:

    python tests/golden/make_golden_grid_mask.py

Writes ref_grid_mask.npz.  ``cases`` lists the case names; for case <c>:
  <c>/shape         (n, c, h, w) of the input
  <c>/config        (use_h, use_w, mode, training) as int64;  <c>/ratio, <c>/prob  float64;  <c>/seed
  <c>/call_kind     the np.random calls of the forward in order: 0 = rand(), 1 = randint(...)
  <c>/call_args     (calls, 2) int64 arguments of each call, -1 where absent
  <c>/call_vals     float64 value each call returned
  <c>/applied       1 if the call masked the input, 0 if it returned it unchanged
  <c>/mask          np.packbits of the (h, w) mask the reference multiplied by (all ones when not applied)
  <c>/next_rand     np.random.rand() right after the forward: a fingerprint of numpy's global state
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mmcv_stub  # noqa: E402
from tests.grid_mask_oracle import Recorder  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
REF_FILE = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "mmdet3d_plugin", "models", "utils", "grid_mask.py")

# name: (n, c, h, w), GridMask kwargs, seed, training.  The detectors build use_h = use_w = True, rotate=1,
# offset=False, ratio=0.5, mode=1, prob=0.7; base / small / tiny are the padded image sizes of those configs.
DETECTOR = dict(use_h=True, use_w=True, ratio=0.5, mode=1, prob=0.7)
CASES = {
    "base_s0": ((6, 3, 928, 1600), dict(DETECTOR, prob=1.0), 0, True),
    "base_s1": ((6, 3, 928, 1600), dict(DETECTOR, prob=1.0), 1, True),
    "small": ((6, 3, 736, 1280), dict(DETECTOR, prob=1.0), 2, True),
    "tiny": ((6, 3, 480, 800), dict(DETECTOR, prob=1.0), 3, True),
    "detector_cfg": ((6, 3, 480, 800), DETECTOR, 11, True),
    "odd_mode0": ((2, 3, 37, 53), dict(DETECTOR, mode=0, prob=1.0), 4, True),
    "odd_mode1": ((1, 3, 15, 9), dict(DETECTOR, prob=1.0), 5, True),
    "odd_tall": ((1, 2, 101, 7), dict(DETECTOR, mode=0, prob=1.0), 6, True),
    "no_h": ((1, 3, 64, 96), dict(DETECTOR, use_h=False, prob=1.0), 7, True),
    "no_w": ((1, 3, 64, 96), dict(DETECTOR, use_w=False, mode=0, prob=1.0), 8, True),
    "no_hw": ((1, 3, 64, 96), dict(DETECTOR, use_h=False, use_w=False, prob=1.0), 9, True),
    "ratio0": ((1, 3, 120, 200), dict(DETECTOR, ratio=0.0, prob=1.0), 10, True),
    "ratio1": ((1, 3, 120, 200), dict(DETECTOR, ratio=1.0, mode=0, prob=1.0), 12, True),
    "ratio099": ((1, 3, 120, 200), dict(DETECTOR, ratio=0.99, prob=1.0), 13, True),
    "prob0": ((1, 3, 48, 64), dict(DETECTOR, prob=0.0), 14, True),
    "eval": ((1, 3, 48, 64), DETECTOR, 15, False),
}
# seeds searched below: d = h - 1 with st_h = d - 1, and d = h - 1 with st_w = d - 1 (first seed >= 100 that draws it)
NEAR_H = {"d_near_h_sth": ((1, 3, 12, 20), "st_h"), "d_near_h_stw": ((1, 3, 9, 31), "st_w")}


def _replay(seed, h):
    """(d, st_h, st_w) the forward draws after seeding with `seed` (prob=1, training)."""
    rs = np.random.RandomState(seed)
    rs.rand()
    d = rs.randint(2, h)
    return d, rs.randint(d), rs.randint(d)


def _near_h_seed(h, which):
    for seed in range(100, 100000):
        d, st_h, st_w = _replay(seed, h)
        if d == h - 1 and (st_h if which == "st_h" else st_w) == d - 1:
            return seed
    raise RuntimeError("no seed found")


def load_reference():
    mmcv_stub.install_stub()
    spec = importlib.util.spec_from_file_location("_bevf_ref_grid_mask", REF_FILE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.GridMask


def run_case(GridMask, shape, kw, seed, training):
    n, c, h, w = shape
    m = GridMask(kw["use_h"], kw["use_w"], rotate=1, offset=False, ratio=kw["ratio"], mode=kw["mode"],
                 prob=kw["prob"])
    m.train(training)
    x = torch.ones((1, 1, h, w), dtype=torch.float32)     # the output is then the mask itself
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    np.random.seed(seed)
    try:
        with Recorder() as rec:
            y = m(x)
    finally:
        torch.Tensor.cuda = cuda
    next_rand = np.random.rand()
    applied = y is not x
    mask = y.reshape(h, w).numpy()
    assert set(np.unique(mask)) <= {0.0, 1.0}
    kind, args, vals = rec.arrays()
    return dict(shape=np.array(shape, np.int64),
                config=np.array([kw["use_h"], kw["use_w"], kw["mode"], training], np.int64),
                ratio=np.float64(kw["ratio"]), prob=np.float64(kw["prob"]), seed=np.int64(seed),
                call_kind=kind, call_args=args, call_vals=vals, applied=np.int64(applied),
                mask=np.packbits(mask.astype(np.uint8).reshape(-1)), next_rand=np.float64(next_rand))


def main():
    GridMask = load_reference()
    cases = dict(CASES)
    for name, (shape, which) in NEAR_H.items():
        cases[name] = (shape, dict(DETECTOR, mode=0, prob=1.0), _near_h_seed(shape[2], which), True)
    out = {"cases": np.array(list(cases))}
    for name, (shape, kw, seed, training) in cases.items():
        for k, v in run_case(GridMask, shape, kw, seed, training).items():
            out[f"{name}/{k}"] = v
        print(name, "applied" if out[f"{name}/applied"] else "skipped", out[f"{name}/call_vals"].tolist())
    path = os.path.join(OUT, "ref_grid_mask.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
