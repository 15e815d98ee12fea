"""ms/step of the base training step in the four precision modes a user switches on, alternated in one process.

    bf16           bf16 weights and inputs (the bench.py headline configuration)
    autocast-bf16  fp32 weights and inputs under torch.autocast(dtype=torch.bfloat16)
    fp16           fp16 weights and inputs (model.half())
    autocast-fp16  fp32 weights and inputs under torch.autocast(dtype=torch.float16), loss scaled by a GradScaler

Every mode is built the way bench.py builds its step: train mode (dropout), the flat gradient arena with the
side-stream overlap, point sampling + pair list + forward + backward captured in one CUDA graph and replayed.  The
modes are timed in rounds (mode order rotated every round) so that clock and neighbour drift hit them alike.
Prints one line per mode and round, then the median per mode, with the GPU name and power limit.

    python tools/bench_precision.py [--config base] [--steps 20] [--warmup 5] [--rounds 3]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bevformer_b200 import synthetic as syn  # noqa: E402
from bevformer_b200.plugin import build_transformer_layer_sequence  # noqa: E402

MODES = {  # name: (parameter / input dtype, autocast dtype or None, GradScaler)
    "bf16": (torch.bfloat16, None, False),
    "autocast-bf16": (torch.float32, torch.bfloat16, False),
    "fp16": (torch.float16, None, False),
    "autocast-fp16": (torch.float32, torch.float16, True),
}


def gpu_description() -> str:
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return f"{name}, power limit / max SM clock: {q.stdout.strip() or 'unknown'}"
    except (OSError, subprocess.SubprocessError):
        return f"{name}, power limit unknown"


def build_step(workload, mode, dev):
    """(CUDA graph of one training step in ``mode``, the objects its replays read).  The graph holds raw pointers
    to the parameters, inputs and scaler state allocated outside it: the caller keeps the second element alive
    for as long as it replays the graph."""
    pdt, amp, use_scaler = MODES[mode]
    enc = build_transformer_layer_sequence(syn.encoder_cfg(workload))
    enc.load_state_dict(syn.make_state_dict(workload))
    enc = enc.to(dev, pdt).train()
    enc.enable_grad_arena(overlap=True)
    host = syn.make_encoder_inputs(workload, bs=1, seed=0)
    inp = {k: getattr(host, k).to(dev, pdt) for k in ("bev_query", "feat", "bev_pos", "prev_bev")}
    inp["bev_query"].requires_grad_(True)
    inp["feat"].requires_grad_(True)
    l2i = torch.as_tensor(np.asarray([m["lidar2img"] for m in host.img_metas], dtype=np.float32)).to(dev)
    shift, ss, lsi = host.shift.to(dev), host.spatial_shapes.to(dev), host.level_start_index.to(dev)
    proj = torch.randn(1, workload.num_query, workload.embed_dims, device=dev)
    scaler = torch.amp.GradScaler("cuda") if use_scaler else None
    leaves = list(enc.parameters()) + [inp["bev_query"], inp["feat"]]

    def body():
        with torch.autocast("cuda", dtype=amp, enabled=amp is not None):
            out = enc(inp["bev_query"], inp["feat"], inp["feat"], bev_h=workload.bev_h, bev_w=workload.bev_w,
                      bev_pos=inp["bev_pos"], spatial_shapes=ss, level_start_index=lsi, prev_bev=inp["prev_bev"],
                      shift=shift, img_metas=host.img_metas, lidar2img=l2i)
        loss = (out.float() * proj).sum()
        (scaler.scale(loss) if scaler is not None else loss).backward()

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(3):
            for t in leaves:
                t.grad = None
            body()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize()
    for t in leaves:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    return graph, (enc, inp, l2i, shift, ss, lsi, proj, scaler, host)


def time_graph(graph, steps, warmup) -> float:
    for _ in range(warmup):
        graph.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        graph.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="base", choices=sorted(syn.WORKLOADS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision.py: no CUDA device (this library has no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(1234)
    w = syn.WORKLOADS[args.config]
    print(f"GPU: {gpu_description()}")
    print(f"workload: {args.config} encoder training step (CUDA graph, gradient arena), "
          f"{args.steps} steps after {args.warmup} warm-up per measurement")
    built = {m: build_step(w, m, dev) for m in MODES}
    graphs = {m: g for m, (g, _keep) in built.items()}
    times = {m: [] for m in MODES}
    order = list(MODES)
    for r in range(args.rounds):
        for m in order[r % len(order):] + order[:r % len(order)]:
            ms = time_graph(graphs[m], args.steps, args.warmup)
            times[m].append(ms)
            print(f"round {r}  {m:14s} {ms:8.3f} ms/step", flush=True)
    for m in MODES:
        print(f"{m:14s} median {statistics.median(times[m]):8.3f} ms/step  "
              f"({' / '.join(f'{t:.3f}' for t in times[m])})")


if __name__ == "__main__":
    main()
