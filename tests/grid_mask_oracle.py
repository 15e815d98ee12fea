"""GridMask restated for the tests: the closed form of the reference's mask (grid_mask.py:90-112), the goldens of
tests/golden/make_golden_grid_mask.py, and a recorder of the np.random calls a forward makes."""
from __future__ import annotations

import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_grid_mask.npz")


def closed_form_mask(h, w, d, l, st_h, st_w, use_h, use_w, mode):
    """(h, w) float32 mask: pixel (y, x) sits at (y + (hh - h) // 2, x + (ww - w) // 2) of the (hh, ww) =
    (int(1.5 h), int(1.5 w)) frame, where the loop zeroes rows y' with (y' - st_h) // d in [0, hh // d) and
    (y' - st_h) % d < l, and the same for columns; mode 1 flips the mask."""
    hh, ww = int(1.5 * h), int(1.5 * w)

    def stripes(n, pad, st):
        c = np.arange(n) + (pad - n) // 2 - st
        k = c // d
        return (k >= 0) & (k < pad // d) & (c % d < l)
    zero = np.zeros((h, w), bool)
    if use_h:
        zero |= stripes(h, hh, st_h)[:, None]
    if use_w:
        zero |= stripes(w, ww, st_w)[None, :]
    mask = (~zero).astype(np.float32)
    return 1 - mask if mode == 1 else mask


def load_golden():
    """case name -> dict of the case's fields, with the mask unpacked to (h, w) float32."""
    z = np.load(GOLDEN)
    out = {}
    for name in z["cases"].tolist():
        c = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
        h, w = (int(v) for v in c["shape"][2:])
        c["mask"] = np.unpackbits(c["mask"])[:h * w].reshape(h, w).astype(np.float32)
        c["use_h"], c["use_w"], c["mode"], c["training"] = (int(v) for v in c["config"])
        out[name] = c
    return out


def drawn(case):
    """(d, l, st_h, st_w) of an applied golden case: the randint results in call order, l from the ratio."""
    vals = case["call_vals"]
    d, st_h, st_w = int(vals[1]), int(vals[2]), int(vals[3])
    return d, min(max(int(d * float(case["ratio"]) + 0.5), 1), d - 1), st_h, st_w


class Recorder:
    """Wraps np.random.rand / randint for the duration of a block and records every call; the wrapped functions are
    the originals, so numpy's state advances exactly as without the recorder."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self.rand, self.randint = np.random.rand, np.random.randint

        def rand(*a):
            v = self.rand(*a)
            self.calls.append((0, a, v))
            return v

        def randint(*a):
            v = self.randint(*a)
            self.calls.append((1, a, v))
            return v
        np.random.rand, np.random.randint = rand, randint
        return self

    def __exit__(self, *exc):
        np.random.rand, np.random.randint = self.rand, self.randint

    def arrays(self):
        """(kind (calls,) 0 = rand / 1 = randint, args (calls, 2) with -1 where absent, values (calls,) float64)"""
        kind = np.array([k for k, _, _ in self.calls], np.int64)
        args = np.full((len(self.calls), 2), -1, np.int64)
        for i, (_, a, _) in enumerate(self.calls):
            args[i, :len(a)] = a
        vals = np.array([float(v) for _, _, v in self.calls], np.float64)
        return kind, args, vals
