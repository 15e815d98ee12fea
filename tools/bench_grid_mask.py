"""GridMask at the detectors' image sizes: the reference's flow against the library's module.

    python tools/bench_grid_mask.py [--iters 20] [--queued-ms 20]

The reference flow is restated here (grid_mask.py:86-122): the numpy stripe loop, the PIL round trip, `.cuda()` of
the mask (a pageable, blocking copy) and the multiply.  Both flows run behind the same queued GPU workload (a chain of
bf16 GEMMs sized to --queued-ms, standing in for the history frames a training step queues before the current
frame), because the blocking copy cannot start before that work drains.  Per image size (6 cameras x 3 channels x H x W, fp32) it prints:
  host_ms     host wall time from the start of the call until it returns (the reference's includes the drain)
  wall_ms     host wall time from queuing the workload to the end of a final synchronise
  queued_dev_ms   the queued workload's device time in the same iterations (CUDA events)
  added_dev_ms    device time from the end of the queued work to the end of the flow's last kernel (CUDA events):
                  what the flow adds to the stream behind that work
  host_idle_ms    host time of the call with nothing queued
  mask_ms     the reference's host mask build alone (numpy + PIL, nothing queued)
  kernel_us   the library kernel alone (CUDA events around replays of a graph of launches), per dtype, with its
              bytes (one read and one write of every element) over that time and the share of the H100 SXM data
              sheet's 3.35 TB/s
The GPU name and power limit are read in the same run.  Medians over --iters.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bevformer_b200 import ops  # noqa: E402
from bevformer_b200.plugin.grid_mask import GridMask  # noqa: E402

SIZES = {"base": (928, 1600), "small": (736, 1280), "tiny": (480, 800)}
HBM = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        out = torch.cuda.get_device_name()
    return out


def reference_mask(h, w, use_h=True, use_w=True, rotate=1, ratio=0.5):
    """grid_mask.py:90-112 restated: the draws, the (1.5 h, 1.5 w) numpy mask, PIL's rotate, the crop."""
    from PIL import Image
    hh, ww = int(1.5 * h), int(1.5 * w)
    d = np.random.randint(2, h)
    l = min(max(int(d * ratio + 0.5), 1), d - 1)
    mask = np.ones((hh, ww), np.float32)
    st_h = np.random.randint(d)
    st_w = np.random.randint(d)
    if use_h:
        for i in range(hh // d):
            s = d * i + st_h
            t = min(s + l, hh)
            mask[s:t, :] *= 0
    if use_w:
        for i in range(ww // d):
            s = d * i + st_w
            t = min(s + l, ww)
            mask[:, s:t] *= 0
    r = np.random.randint(rotate)
    mask = np.asarray(Image.fromarray(np.uint8(mask)).rotate(r))
    return mask[(hh - h) // 2:(hh - h) // 2 + h, (ww - w) // 2:(ww - w) // 2 + w]


def reference_forward(x, mode=1):
    """GridMask.forward of the reference with prob = 1, training."""
    np.random.rand()
    n, c, h, w = x.size()
    x = x.view(-1, h, w)
    mask = torch.from_numpy(reference_mask(h, w).copy()).to(x.dtype).cuda()
    if mode == 1:
        mask = 1 - mask
    return (x * mask.expand_as(x)).view(n, c, h, w)


class Queued:
    """A chain of 4096^3 bf16 GEMMs taking about `ms` on the device: the work a training step has queued when the
    current frame reaches GridMask."""

    def __init__(self, ms):
        self.a = torch.randn(4096, 4096, device="cuda", dtype=torch.bfloat16)
        self.b = torch.randn(4096, 4096, device="cuda", dtype=torch.bfloat16) / 64
        self.n = 1
        one = self.time()
        self.n = max(1, round(ms / one))
        self.ms = self.time()

    def run(self):
        y = self.a
        for _ in range(self.n):
            y = y @ self.b
        return y

    def time(self):
        for _ in range(3):
            self.run()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        self.run()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)


def kernel_us(x, reps=10, replays=20):
    """Time of one bevf_grid_mask launch on x (6, 3, h, w): `reps` launches captured in a CUDA graph, replayed, so
    the host's per-call cost stays out of the number."""
    n, c, h, w = x.shape
    xv = x.view(-1, h, w)
    d = h // 3
    drawn = (d, d // 2, d - 1, d // 3, True, True, 1)
    for _ in range(3):
        ops.grid_mask_apply(xv, *drawn)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            ops.grid_mask_apply(xv, *drawn)
    graph.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(replays):
        graph.replay()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / (reps * replays)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--queued-ms", type=float, default=20.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    gpu = gpu_info()
    queued = Queued(args.queued_ms)
    module = GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=1.0).train()
    rows = []
    for name, (h, w) in SIZES.items():
        x = torch.randn(6, 3, h, w, device="cuda")
        # the two flows compute the same thing for the same draws
        np.random.seed(7)
        want = reference_forward(x)
        np.random.seed(7)
        got = module(x)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), "outputs differ"
        res = {}
        for flow, fn in (("reference", reference_forward), ("library", module)):
            host, wall, qdev, added, idle = [], [], [], [], []
            for it in range(args.iters + 2):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                torch.cuda.synchronize()
                np.random.seed(it)
                t0 = time.perf_counter()
                ev[0].record()
                queued.run()
                ev[1].record()
                t1 = time.perf_counter()
                fn(x)
                t2 = time.perf_counter()
                ev[2].record()
                torch.cuda.synchronize()
                t3 = time.perf_counter()
                np.random.seed(it)
                t4 = time.perf_counter()
                fn(x)
                t5 = time.perf_counter()
                torch.cuda.synchronize()
                if it >= 2:
                    host.append((t2 - t1) * 1e3)
                    wall.append((t3 - t0) * 1e3)
                    qdev.append(ev[0].elapsed_time(ev[1]))
                    added.append(ev[1].elapsed_time(ev[2]))
                    idle.append((t5 - t4) * 1e3)
            res[flow] = dict(host_ms=float(np.median(host)), wall_ms=float(np.median(wall)),
                             queued_dev_ms=float(np.median(qdev)), added_dev_ms=float(np.median(added)),
                             host_idle_ms=float(np.median(idle)))
        build = []
        for it in range(args.iters):
            np.random.seed(it)
            t0 = time.perf_counter()
            reference_mask(h, w)
            build.append((time.perf_counter() - t0) * 1e3)
        res["reference"]["mask_ms"] = float(np.median(build))
        kern = {}
        for dt in (torch.float32, torch.bfloat16, torch.float16):
            xd = x.to(dt)
            us = kernel_us(xd)
            nbytes = 2 * xd.numel() * xd.element_size()
            kern[str(dt).replace("torch.", "")] = dict(us=us, gbps=nbytes / us / 1e3,
                                                       hbm_share=nbytes / (us * 1e-6) / HBM)
        rows.append(dict(size=name, h=h, w=w, queued_ms=queued.ms, **{f: res[f] for f in res}, kernel=kern))
        r, lb = res["reference"], res["library"]
        print(f"{name:5s} {h}x{w}: " + " | ".join(
            f"{f} host {v['host_ms']:.3f} ms (idle {v['host_idle_ms']:.3f}), wall {v['wall_ms']:.2f} ms, queued "
            f"{v['queued_dev_ms']:.2f} ms, added {v['added_dev_ms']:.3f} ms" for f, v in (("reference", r),
                                                                                      ("library", lb)))
              + f" | mask build {r['mask_ms']:.2f} ms | kernel " + ", ".join(f"{k} {v['us']:.1f} us ({v['gbps']:.0f} GB/s, "
                                                             f"{100 * v['hbm_share']:.0f} %)" for k, v in kern.items()))
    print(json.dumps({"gpu": gpu, "results": rows}))


if __name__ == "__main__":
    main()
