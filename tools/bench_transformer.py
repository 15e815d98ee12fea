"""What the object-query decoder costs a video frame: BEVStream frames/s at tiny, small and base (bf16, eval, device
path, 900 object queries through the configs' 6-layer decoder with box refinement) for a BEV-only frame
(``get_bev_features``) against a whole-transformer frame (``PerceptionTransformer.forward``), each eager and
captured (one CUDA-graph replay per frame), alternating the four in one process.  Also the host enqueue time of a
frame against its GPU span (queue empty beforehand), the decoder's share of a captured frame's GPU span, and the
kernels per frame counted by torch.profiler in a separate untimed frame.  Needs a GPU; prints the card's name and
power limit next to the numbers.

    python tools/bench_transformer.py [--workloads tiny,small,base] [--frames 50] [--warmup 5] [--rounds 3] [--json PATH]
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200 import synthetic as syn                                      # noqa: E402
from bevformer_b200.plugin import BEVStream, PerceptionTransformer              # noqa: E402
from tools.bench_stream import card                                              # noqa: E402

MODES = ("bev_eager", "bev_captured", "full_eager", "full_captured")
NUM_QUERY = 900
DECODER_LAYERS = 6


def reg_branches(c, n, g):
    """The head's regression branches with box refinement (bevformer_head.py: Linear-ReLU x 2, Linear(C, 10))."""
    branches = torch.nn.ModuleList(torch.nn.Sequential(torch.nn.Linear(c, c), torch.nn.ReLU(), torch.nn.Linear(c, c),
                                                       torch.nn.ReLU(), torch.nn.Linear(c, 10)) for _ in range(n))
    with torch.no_grad():
        for p in branches.parameters():
            p.copy_(0.05 * torch.randn(p.shape, generator=g))
    return branches


class Scene:
    """One workload's whole transformer, a fixed pyramid, `n` frames of ego motion as device tensors, and one
    BEVStream per mode (the captured ones recorded up front)."""

    def __init__(self, workload, n, dev):
        w = self.w = syn.WORKLOADS[workload]
        dec = copy.deepcopy(syn.DECODER_CFG)
        dec["num_layers"] = DECODER_LAYERS
        m = PerceptionTransformer(num_feature_levels=len(w.levels), num_cams=w.num_cams, encoder=syn.encoder_cfg(w),
                                  decoder=dec, embed_dims=w.embed_dims)
        sd = syn.make_random_state_dict(m, 0)
        sd.update(syn.make_perception_state_dict(w))
        m.load_state_dict(sd)
        self.m = m.to(dev, torch.bfloat16).eval()
        inp = syn.make_perception_inputs(w, bs=1, with_prev=False, device=dev, dtype=torch.bfloat16)
        self.feats, self.q, self.pos = inp.mlvl_feats, inp.bev_queries, inp.bev_pos
        self.gl = (0.512 * 200 / w.bev_h, 0.512 * 200 / w.bev_w)
        g = torch.Generator().manual_seed(5)
        self.oq = torch.randn(NUM_QUERY, 2 * w.embed_dims, generator=g).to(dev, torch.bfloat16)
        self.reg = reg_branches(w.embed_dims, DECODER_LAYERS, g).to(dev, torch.bfloat16)
        base = inp.img_metas[0]
        pos, ang, cbs = np.array([10.0, -4.0, 0.0]), 30.0, []
        for i in range(n):
            cb = np.array(syn.make_can_bus(0), dtype=np.float64)
            pos = pos + np.array([0.9, -0.3 + 0.01 * (i % 7), 0.0])
            ang = ang + 1.5 - 0.5 * (i % 5)
            cb[:3], cb[-1] = pos, ang
            cbs.append(cb)
        self.bare = [{k: v for k, v in base.items() if k not in ("can_bus", "lidar2img")} | {"scene_token": "bench"}]
        self.cb = torch.as_tensor(np.array(cbs)).to(dev)
        self.l2i = torch.as_tensor(np.asarray([base["lidar2img"]], dtype=np.float32)).to(dev)
        self.streams = {mode: BEVStream(self.m) for mode in MODES}
        for mode in ("bev_captured", "full_captured"):
            self.streams[mode].capture(self.feats, self.bare, self.q, w.bev_h, w.bev_w, self.pos, self.gl,
                                       can_bus=self.cb[0:1], lidar2img=self.l2i, **self.head(mode))

    def head(self, mode):
        return dict(object_query_embed=self.oq, reg_branches=self.reg) if mode.startswith("full") else {}

    def frame(self, mode, i):
        w, s = self.w, self.streams[mode]
        if mode.endswith("captured"):
            return s.step(None, self.bare, can_bus=self.cb[i:i + 1])          # pyramid and matrices already in place
        return s.step(self.feats, self.bare, self.q, w.bev_h, w.bev_w, self.pos, self.gl, can_bus=self.cb[i:i + 1],
                      lidar2img=self.l2i, **self.head(mode))

    def run(self, mode, first, count):
        for i in range(first, first + count):
            self.frame(mode, i)


def kernels_per_frame(scene, mode, i):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        scene.frame(mode, i)
        torch.cuda.synchronize()
    kernels = copies = 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            if e.name.startswith(("Memcpy", "Memset")):
                copies += 1
            else:
                kernels += 1
    return kernels, copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="tiny,small,base")
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_transformer.py measures on a GPU; none is available")
    dev = torch.device("cuda")
    name, limit = card()
    result = dict(gpu=name, power_limit=limit, dtype="bf16", num_query=NUM_QUERY, decoder_layers=DECODER_LAYERS,
                  frames=args.frames, warmup=args.warmup, rounds=args.rounds, workloads={})
    print(f"# {name}, power limit {limit}; bf16 eval, device path, {NUM_QUERY} object queries, {DECODER_LAYERS} decoder "
          f"layers; {args.frames} frames after {args.warmup} warm-ups, median of {args.rounds} alternating rounds")
    n = args.warmup + args.frames + 8
    for workload in args.workloads.split(","):
        scene = Scene(workload, n, dev)
        fps = {mode: [] for mode in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                scene.streams[mode].reset()
                scene.run(mode, 0, args.warmup)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                scene.run(mode, args.warmup, args.frames)
                torch.cuda.synchronize()
                fps[mode].append(args.frames / (time.perf_counter() - t0))
        row = {}
        for mode in MODES:
            enq, span = [], []
            for k in range(6):                              # queue empty before each frame
                i = args.warmup + args.frames + k
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                s.record()
                scene.frame(mode, i)
                e.record()
                t1 = time.perf_counter()
                torch.cuda.synchronize()
                enq.append((t1 - t0) * 1e3)
                span.append(s.elapsed_time(e))
            kernels, copies = kernels_per_frame(scene, mode, args.warmup + args.frames + 6)
            row[mode] = dict(fps=round(statistics.median(fps[mode]), 1), fps_rounds=[round(x, 1) for x in fps[mode]],
                             enqueue_ms=round(statistics.median(enq), 3), gpu_span_ms=round(statistics.median(span), 3),
                             kernels_per_frame=kernels, copies_per_frame=copies)
            print(f"{workload:6s} {mode:13s} {row[mode]['fps']:8.1f} frames/s   enqueue {row[mode]['enqueue_ms']:7.3f} ms"
                  f"   gpu span {row[mode]['gpu_span_ms']:7.3f} ms   kernels/frame {kernels:4d}   copies/frame {copies:3d}")
        full, bev = row["full_captured"]["gpu_span_ms"], row["bev_captured"]["gpu_span_ms"]
        row["decoder_share_captured"] = round((full - bev) / full, 3) if full > 0 else None
        print(f"{workload:6s} decoder share of a captured frame's GPU span: {row['decoder_share_captured']}")
        scene.m.encoder.check_plan()
        result["workloads"][workload] = row
        del scene
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
