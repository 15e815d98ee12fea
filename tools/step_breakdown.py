"""Per-kernel GPU time of one training step of the base encoder (development tool).

Runs the same step as bench.py eagerly under torch.profiler (CUPTI activity records: real kernel
durations, warm caches, no replay) and prints the kernels grouped by name with their time per step.
Usage: python tools/step_breakdown.py [--steps 2] [--deterministic] [--out results/step_breakdown.txt]
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import sys

import torch
import torch.utils.deterministic

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200 import synthetic as syn  # noqa: E402
from bevformer_b200.plugin import build_transformer_layer_sequence  # noqa: E402


def short(name: str) -> str:
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"at::native::", "", name)
    name = re.sub(r"\(anonymous namespace\)::", "", name)
    return name[:110]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--workload", default="base")
    ap.add_argument("--out", default=None)
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True) (uninitialised-memory fill off)")
    args = ap.parse_args()
    if args.deterministic:
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True)
        torch.utils.deterministic.fill_uninitialized_memory = False
    dev = torch.device("cuda", 0)
    w = syn.WORKLOADS[args.workload]
    dtype = torch.bfloat16
    enc = build_transformer_layer_sequence(syn.encoder_cfg(w))
    enc.load_state_dict(syn.make_state_dict(w))
    enc = enc.to(dev, dtype).train()
    host = syn.make_encoder_inputs(w, bs=1, seed=0)
    inp = {k: getattr(host, k).to(dev, dtype) for k in ("bev_query", "feat", "bev_pos", "prev_bev")}
    shift = host.shift.to(dev)
    ss, lsi = host.spatial_shapes.to(dev), host.level_start_index.to(dev)
    proj = torch.randn(1, w.num_query, w.embed_dims, device=dev, dtype=dtype)
    plan = enc.prepare(host.img_metas, w.bev_h, w.bev_w, dev)
    bq = inp["bev_query"].requires_grad_(True)
    ft = inp["feat"].requires_grad_(True)

    def step():
        for t in list(enc.parameters()) + [bq, ft]:
            t.grad = None
        out = enc(bq, ft, ft, bev_h=w.bev_h, bev_w=w.bev_w, bev_pos=inp["bev_pos"], spatial_shapes=ss,
                  level_start_index=lsi, prev_bev=inp["prev_bev"], shift=shift,
                  img_metas=host.img_metas, sca_plan=plan)
        (out * proj).sum().backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    agg = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            a = agg[short(ev.name)]
            a[0] += ev.device_time          # us
            a[1] += 1
    rows = sorted(agg.items(), key=lambda kv: -kv[1][0])
    total = sum(v[0] for _, v in rows) / args.steps
    lines = [f"kernel time per step: {total / 1e3:.3f} ms over {sum(v[1] for _, v in rows) // args.steps} launches"]
    for name, (us, n) in rows:
        lines.append(f"{us / args.steps / 1e3:8.3f} ms {n // args.steps:5d}x {us / n:8.1f} us  {name}")
    text = "\n".join(lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
