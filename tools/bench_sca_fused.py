"""SpatialCrossAttention's sampler with and without the fused sampling-point prep, at base (development tool, GPU only).

  prep   bevf_sca_prep_forward + bevf_msda_rows_forward;  bevf_msda_rows_backward_mixed_dense + bevf_sca_prep_backward
  fused  bevf_sca_rows_forward_fused;  bevf_sca_rows_backward_fused + bevf_sca_prep_backward_multi
Both run on the base rig's in-view pairs with the encoder's grad_value accumulation (levels 0-1 scaled fp16, level 2
fp32, level 3 on the dense kernel).  Each timing is one forward or one backward as the encoder issues it, bracketed by
CUDA events; the bf16 merge of grad_value is left out (the same pass for both).  The two paths alternate in one
process, ROUNDS x ITERS launches each; the median per path is printed with the card, its power limit and clocks.
Usage: python tools/bench_sca_fused.py [--iters 30] [--rounds 3] [--out results/sca_fused.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200 import ops  # noqa: E402
from tests.test_sca_fused_prep_gpu import _case  # noqa: E402
from tools.bench_sca_backward import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sca_fused.py needs a GPU")
    c = _case("base", 1, True)
    plan, raw, v, ss, lsi, levels, gout = c["plan"], c["raw"], c["value"], c["ss"], c["lsi"], c["levels"], c["gout"]
    bs, nq, l, p = c["bs"], c["nq"], c["l"], c["p"]
    rows_per_map = plan.row_map.numel() / v.shape[0]
    _, _, nfine = ops.gv_mode_for(rows_per_map, p, levels)
    kd = ops.dense_levels_for(rows_per_map, p, levels)
    dense = dict(map_range=plan.map_range, first_dense_level=max(kd, nfine)) if kd is not None else {}
    saved = {}

    def prep_fwd():
        loc, attn = ops.sca_prep_forward(raw, plan.ref_cam, plan.pair_q, plan.pair_cam, ss, bs, nq, 8, l, p)
        saved["la"] = (loc, attn)
        return ops.msda_rows_forward(v, ss, lsi, loc, attn, plan.row_map)

    def prep_bwd():
        loc, attn = saved["la"]
        _, gl, ga = ops.msda_rows_backward_mixed(v, ss, lsi, levels, nfine, loc, attn, plan.row_map, gout, lazy=True,
                                                 **dense)
        return ops.sca_prep_backward(raw, gl, ga, plan.pair_of, ss, bs, nq, plan.pair_q.numel(), 8, l, p,
                                     out_dtype=torch.bfloat16)

    def fused_fwd():
        out, saved["stats"], saved["coarse"] = ops.sca_rows_forward_fused(
            v, ss, lsi, raw, plan.ref_cam, plan.pair_q, plan.pair_cam, plan.row_map, bs, nq,
            dense.get("first_dense_level"))
        return out

    def fused_bwd():
        return ops.sca_rows_backward_fused(v, ss, lsi, levels, nfine, raw, saved["stats"], plan.ref_cam, plan.pair_q,
                                           plan.pair_cam, plan.pair_of, plan.row_map, gout, bs, nq, coarse=saved["coarse"],
                                           **dense)[1]

    fns = {"prep_forward": prep_fwd, "prep_backward": prep_bwd, "fused_forward": fused_fwd,
           "fused_backward": fused_bwd}
    times = {n: [] for n in fns}
    for _ in range(args.rounds):
        for name, fn in fns.items():
            for _ in range(3):
                fn()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for s, e in ev:
                s.record()
                fn()
                e.record()
            torch.cuda.synchronize()
            times[name] += [s.elapsed_time(e) for s, e in ev]
    res = {"card": card(), "pairs": int((plan.row_map >= 0).sum().item()), "launches_per_path": args.rounds * args.iters,
           "median_ms": {n: float(torch.tensor(t).median()) for n, t in times.items()},
           "min_ms": {n: float(min(t)) for n, t in times.items()},
           "max_ms": {n: float(max(t)) for n, t in times.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
