"""Modulated deformable convolution (DCNv2) at the backbone's shapes: the library op against torchvision's
deform_conv2d and cuDNN's dense 3x3 convolution of the same shape.

    python tools/bench_dcn.py [--iters 50] [--warmup 10] [--profile out_dir]

Prints one table row per (shape, pass): CUDA-event medians after warm-up, achieved TFLOP/s over the 2 M Cout 9 Cin
FLOP of one conv (forward; forward + backward counts 3x) and its share of the H100 SXM data sheet's dense
989 TFLOP/s (BF16), with the GPU name and power limit read in the same run.  Output parity against torchvision is
checked at the timed size.  ``--profile`` adds a separate torch.profiler run that splits the library's time between
the sampling kernels (dcn_im2col / dcn_col2im) and the GEMMs.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bevformer_b200 import ops  # noqa: E402

SHAPES = {"base layer3": (6, 256, 58, 100), "base layer4": (6, 512, 29, 50), "small layer3": (6, 256, 46, 80)}
PEAK = 989e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        out = torch.cuda.get_device_name()
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def inputs(N, C, H, W, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, C, H, W, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    off = (torch.randn(N, 18, H, W, device="cuda", generator=g) * 2).to(dtype)
    mask = torch.rand(N, 9, H, W, device="cuda", generator=g).to(dtype)
    w = (torch.randn(C, C, 3, 3, device="cuda", generator=g) / (3 * C ** 0.5)).to(dtype)
    b = torch.zeros(C, device="cuda", dtype=dtype)
    dy = torch.randn(N, C, H, W, device="cuda", generator=g).to(dtype)
    return x, off, mask, w, b, dy


def runners(x, off, mask, w, b, dy):
    leaves = [t.detach().clone().requires_grad_(True) for t in (x, off, mask, w, b)]

    def lib_fwd():
        with torch.no_grad():
            return ops.modulated_deform_conv2d(x, off, mask, w, b, 1, 1, 1, 1, 1)

    def lib_fb():
        y = ops.modulated_deform_conv2d(*leaves, 1, 1, 1, 1, 1)
        y.backward(dy)

    out = {"library": (lib_fwd, lib_fb)}
    try:
        import torchvision.ops as tv
        # torchvision has no bf16 kernels: it runs on the same values in fp16 (exact for these bf16 values)
        xt, ot, mt, wt, bt, dyt = (t.to(torch.float16) for t in (x.contiguous(), off, mask, w, b, dy))
        tv.deform_conv2d(xt[:1, :, :4, :4], ot[:1, :, :4, :4], wt, None, padding=1, mask=mt[:1, :, :4, :4])

        def tv_fwd():
            with torch.no_grad():
                return tv.deform_conv2d(xt, ot, wt, bt, padding=1, mask=mt)

        tl = [t.detach().clone().requires_grad_(True) for t in (xt, ot, mt, wt, bt)]

        def tv_fb():
            y = tv.deform_conv2d(tl[0], tl[1], tl[3], tl[4], padding=1, mask=tl[2])
            y.backward(dyt)
        out["torchvision fp16"] = (tv_fwd, tv_fb)
    except Exception as e:  # noqa: BLE001
        out["torchvision fp16"] = f"not available ({type(e).__name__}: {str(e)[:80]})"
    xd = x.detach().clone().requires_grad_(True)
    wd = w.detach().clone().requires_grad_(True)

    def cudnn_fwd():
        with torch.no_grad():
            return F.conv2d(x, w, b, padding=1)

    def cudnn_fb():
        F.conv2d(xd, wd, None, padding=1).backward(dy)
    out["cuDNN dense 3x3"] = (cudnn_fwd, cudnn_fb)
    return out


def profile_split(x, off, mask, w, b, dy, out_dir):
    leaves = [t.detach().clone().requires_grad_(True) for t in (x, off, mask, w, b)]
    for _ in range(3):
        ops.modulated_deform_conv2d(*leaves, 1, 1, 1, 1, 1).backward(dy)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            ops.modulated_deform_conv2d(*leaves, 1, 1, 1, 1, 1).backward(dy)
        torch.cuda.synchronize()
    split = {"sampling (dcn_im2col)": 0.0, "sampling backward (dcn_col2im)": 0.0, "GEMMs (gemm.cu)": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 10 / 1000.0
        if t <= 0:
            continue
        n = ev.key
        if "dcn_im2col" in n:
            split["sampling (dcn_im2col)"] += t
        elif "dcn_col2im" in n:
            split["sampling backward (dcn_col2im)"] += t
        elif "gemm" in n or "wgrad" in n or "ws_kernel" in n:
            split["GEMMs (gemm.cu)"] += t
        else:
            split["other"] += t
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "dcn_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile", default=None, help="directory for the profiler's table (split run)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn.py needs a GPU")
    print(f"GPU: {gpu_info()}; bf16 storage; median of {a.iters} after {a.warmup} warm-up calls")
    print(f"{'shape':14s} {'pass':9s} {'implementation':16s} {'ms':>8s} {'TFLOP/s':>8s} {'% of 989':>8s}")
    results = []
    for name, (N, C, H, W) in SHAPES.items():
        tensors = inputs(N, C, H, W)
        flop = 2.0 * N * H * W * C * 9 * C
        run = runners(*tensors)
        ref = run["library"][0]().float()
        tv = run["torchvision fp16"]
        if not isinstance(tv, str):
            d = (tv[0]().float() - ref).abs().max().item() / ref.abs().max().item()
            print(f"{name:14s} parity: max |library - torchvision| / max|out| = {d:.2e}")
        for impl, fns in run.items():
            if isinstance(fns, str):
                print(f"{name:14s} {'':9s} {impl:16s} {fns}")
                continue
            for pas, fn, mult in (("fwd", fns[0], 1), ("fwd+bwd", fns[1], 3)):
                ms = timed(fn, a.iters, a.warmup)
                tf = mult * flop / (ms * 1e-3) / 1e12
                print(f"{name:14s} {pas:9s} {impl:16s} {ms:8.3f} {tf:8.1f} {100 * tf * 1e12 / PEAK:7.1f}%")
                results.append(dict(shape=name, passes=pas, impl=impl, ms=ms, tflops=tf))
        if a.profile is not None:
            split = profile_split(*tensors, a.profile if a.profile else None)
            tot = sum(split.values())
            print(f"{name:14s} library fwd+bwd split (torch.profiler, ms per call): " +
                  ", ".join(f"{k} {v:.3f} ({100 * v / tot:.0f}%)" for k, v in split.items()))
        del tensors, run
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": gpu_info(), "results": results}))


if __name__ == "__main__":
    main()
