"""SpatialCrossAttention sampler backward at base, one timing per grad_value strategy (development tool, GPU only).

The SCA launch of the headline benchmark (the base rig's in-view pairs, 4 levels, 8 points, bf16) through:
  mixed             bevf_msda_rows_backward_mixed: levels 0-1 scaled fp16, levels 2-3 fp32 L2 reductions
  dense_same        bevf_msda_rows_backward_dense, same stream: levels 1-3 on the tensor cores, level 0 fp32 reductions
  dense_second      the same with the dense kernel on the library's second stream
  mixed_dense_k{1,2}_{same,second}
                    bevf_msda_rows_backward_mixed_dense: levels [0, k) scaled fp16, levels [k, 4) on the tensor cores
  mixed_dense_k2_d3_{same,second}
                    levels 0-1 scaled fp16, level 2 fp32 reductions, level 3 on the tensor cores
  replicated_d3_{same,second}
                    bevf_msda_rows_backward_replicated: levels 0-1 scaled fp16, level 2 in the scaled-fp16 copies of
                    ops.gv_replicas_for (3 at base), level 3 on the tensor cores
Each timing is one op as the encoder issues it (scale source, zero-fill of the accumulators, the kernels), bracketed
by CUDA events on the caller's stream (the second stream is joined into it); the bf16 conversion / merge pass is not
included (it is the same pass for every mixed form).  The modes alternate in one process, ROUNDS x ITERS launches
each; the median per mode is printed with the card, its power limit and clocks, and the error of each mode's
grad_value against the mixed path's (max|diff| / max|ref|).
Usage: python tools/bench_sca_backward.py [--iters 30] [--rounds 3] [--out results/sca_backward.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200 import _lib, ops, synthetic as syn  # noqa: E402
from tools.bench_msda import rig_sca_inputs  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--modes", default=None, help="comma-separated subset of the modes (the first one is the error reference)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sca_backward.py needs a GPU")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    v, ss, lsi, loc, attn, row_map = rig_sca_inputs(dev)
    w = syn.WORKLOADS["base"]
    levels = [tuple(x) for x in w.levels]
    per_cam = torch.bincount(row_map[row_map >= 0].long(), minlength=v.shape[0])
    ends = per_cam.cumsum(0)
    rng = torch.stack([ends - per_cam, ends], 1).to(torch.int32).contiguous()
    vd = v.to(torch.bfloat16)
    g = torch.Generator().manual_seed(1)
    gout = (torch.randn(loc.shape[0], 256, generator=g) * 0.1).to(dev, torch.bfloat16)

    def mixed(k, dense, kd=None, replicas=None):
        def run():
            return ops.msda_rows_backward_mixed(vd, ss, lsi, levels, k, loc, attn, row_map, gout, lazy=True,
                                                map_range=rng if dense else None, first_dense_level=kd,
                                                replicas=replicas)[0]
        return run

    def dense_fp32():
        return ops.msda_rows_backward(vd, ss, lsi, loc, attn, row_map, gout, dense=(levels, rng))[0]

    modes = {"mixed": (0, mixed(2, False)), "dense_same": (1, dense_fp32), "dense_second": (2, dense_fp32)}
    for k in (1, 2):
        modes[f"mixed_dense_k{k}_same"] = (1, mixed(k, True))
        modes[f"mixed_dense_k{k}_second"] = (2, mixed(k, True))
    modes["mixed_dense_k2_d3_same"] = (1, mixed(2, True, 3))
    modes["mixed_dense_k2_d3_second"] = (2, mixed(2, True, 3))
    reps = ops.gv_replicas_for(row_map.numel() / v.shape[0], loc.shape[3], levels)
    modes["replicated_d3_same"] = (1, mixed(2, True, 3, reps))
    modes["replicated_d3_second"] = (2, mixed(2, True, 3, reps))
    if args.modes:
        modes = {n: modes[n] for n in args.modes.split(",")}

    def materialize(x):
        return x.materialize().float() if isinstance(x, ops.LazyGradValue) else x.float()

    ref = None
    errs = {}
    for name, (dm, fn) in modes.items():
        _lib.check(lib.bevf_msda_set_dense_backward(dm), lib)
        out = materialize(fn())
        torch.cuda.synchronize()
        if ref is None:
            ref = out
        errs[name] = ((out - ref).abs().max() / ref.abs().max()).item()
    times = {n: [] for n in modes}
    for _ in range(args.rounds):
        for name, (dm, fn) in modes.items():
            _lib.check(lib.bevf_msda_set_dense_backward(dm), lib)
            for _ in range(3):
                fn()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for s, e in ev:
                s.record()
                fn()
                e.record()
            torch.cuda.synchronize()
            times[name] += [s.elapsed_time(e) for s, e in ev]
    lib.bevf_msda_set_dense_backward(-1)
    res = {"card": card(), "pairs": int((row_map >= 0).sum().item()), "launches_per_mode": args.rounds * args.iters,
           "median_ms": {n: float(torch.tensor(t).median()) for n, t in times.items()},
           "min_ms": {n: float(min(t)) for n, t in times.items()},
           "max_ms": {n: float(max(t)) for n, t in times.items()},
           "grad_value_err_vs_mixed": errs}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
