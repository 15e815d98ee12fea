"""Microbenchmark of the wgmma projections at the encoder's shapes (development tool, GPU only):
CUDA-event timing with an L2 flush before every iteration, achieved HBM GB/s on the compulsory bytes
rows*(K+N)*size, and the same shapes through cuBLAS for comparison."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200 import ops  # noqa: E402

SHAPES = [  # (name, M, N, K, relu, fp32_out)
    ("tsa_value_proj", 80000, 256, 256, False, False),
    ("tsa_heads", 40000, 192, 512, False, True),
    ("out_proj", 40000, 256, 256, False, False),
    ("sca_heads", 40000, 768, 256, False, True),
    ("sca_value_proj", 184950, 256, 256, False, False),
    ("ffn_up", 40000, 512, 256, True, False),
    ("ffn_down", 40000, 256, 512, False, False),
]


def timed(fn, iters, flush):
    ev = [(torch.cuda.Event(True), torch.cuda.Event(True)) for _ in range(iters)]
    for _ in range(3):
        fn()
    for s, e in ev:
        flush.zero_()
        s.record(); fn(); e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in ev)
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    dev = "cuda"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    hbm = 3350.0  # H100 SXM data sheet, GB/s
    try:
        hbm = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    for name, M, N, K, relu, f32 in SHAPES:
        x = torch.randn(M, K, device=dev).bfloat16()
        w = (torch.randn(N, K, device=dev) / K ** 0.5).bfloat16()
        b = torch.randn(N, device=dev).bfloat16()
        dy = torch.randn(M, N, device=dev).bfloat16()
        od = torch.float32 if f32 else torch.bfloat16
        if args.profile:
            ops.linear_tc(x, w, b, None, relu, od); ops.linear_wgrad_tc(dy, x); torch.cuda.synchronize()
            continue
        t = timed(lambda: ops.linear_tc(x, w, b, None, relu, od), args.iters, flush)
        tw = timed(lambda: ops.linear_wgrad_tc(dy, x), args.iters, flush)
        tw2 = timed(lambda: ops.linear_wgrad_out(dy, x, torch.bfloat16, True), args.iters, flush)
        tl = timed(lambda: torch.nn.functional.linear(x, w, b), args.iters, flush)
        td = td_acc = None
        if N % 64 == 0 and K % 64 == 0:
            prev = torch.randn(M, K, device=dev).bfloat16()
            td = timed(lambda: ops.linear_dgrad_tc(dy, w), args.iters, flush)
            td_acc = timed(lambda: ops.linear_dgrad_tc(dy, w, addend=prev), args.iters, flush)
        byts = M * K * 2 + M * N * (4 if f32 else 2) + N * K * 2
        bw = M * (K + N) * 2 + N * K * 4
        print(json.dumps(dict(shape=name, M=M, N=N, K=K, tc_us=round(t * 1e3, 1), cublas_us=round(tl * 1e3, 1),
                              dgrad_us=None if td is None else round(td * 1e3, 1),
                              dgrad_acc_us=None if td_acc is None else round(td_acc * 1e3, 1),
                              wgrad_us=round(tw * 1e3, 1), wgrad_2pass_us=round(tw2 * 1e3, 1), tc_GBs=round(byts / t / 1e6, 1),
                              tc_frac=round(byts / t / 1e6 / hbm, 3), wgrad_frac=round(bw / tw / 1e6 / hbm, 3),
                              tflops=round(2 * M * N * K / t / 1e9, 1))), flush=True)


if __name__ == "__main__":
    main()
