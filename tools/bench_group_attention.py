"""GroupMultiheadAttention timings: the module (wgmma projections + grouped attention kernel) against the reference
path (groups moved to the batch axis around nn.MultiheadAttention, as group_attention.py:147-157 does) and against
F.scaled_dot_product_attention on the same grouped problem, alternating in one process with CUDA events.

Shapes: the BEVFormerV2 training shape (bs 1, 9900 queries, group 11, 8 heads x 32) and the eval shape (900 queries,
one group).  Two sections:
  kernel      attn_fwd / attn_bwd_dq / attn_bwd_dkv alone (torch.profiler device times), with and without dropout,
              against their exp floor (one exp per score per kernel at 16 per SM per clock, max SM clock) and the
              tensor-core FLOPs of each kernel over the dense bf16 data-sheet rate;
  module_e2e  the whole module (GEMMs, adds, dropout, autograd and Python included) against the other two paths;
              at the eval shape also the forward captured in a CUDA graph, which takes the host out.

    python tools/bench_group_attention.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bevformer_b200.plugin import GroupMultiheadAttention  # noqa: E402

TC_PEAK = 989e12               # dense bf16, H100 SXM data sheet (700 W)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def reference_forward(m, x, pos, group):
    """group_attention.py:136-160 on nn.MultiheadAttention (the module's own parameters)."""
    q = x + pos
    nq, bs = x.shape[0], x.shape[1]
    if m.training:
        q_, k_, v_ = (torch.cat(t.split(nq // group, 0), 1) for t in (q, q, x))
    else:
        q_, k_, v_ = q, q, x
    out = m.attn(q_, k_, v_)[0]
    if m.training:
        out = torch.cat(out.split(bs, 1), 0)
    return x + out


def sdpa_forward(m, x, pos, group):
    """The same grouped problem on F.scaled_dot_product_attention (projections on torch)."""
    a = m.attn
    nq, bs, C = x.shape
    G = group if m.training else 1
    q = x + pos
    w, b = a.in_proj_weight, a.in_proj_bias
    qk = F.linear(q, w[:2 * C], b[:2 * C])
    v = F.linear(x, w[2 * C:], b[2 * C:])

    def heads(t):
        return t.reshape(G, nq // G, bs, 8, 32).permute(2, 0, 3, 1, 4).reshape(bs * G, 8, nq // G, 32)

    o = F.scaled_dot_product_attention(heads(qk[..., :C]), heads(qk[..., C:]), heads(v),
                                       dropout_p=a.dropout if m.training else 0.0)
    o = o.reshape(bs, G, 8, nq // G, 32).permute(1, 3, 0, 2, 4).reshape(nq, bs, C)
    return x + F.linear(o, a.out_proj.weight, a.out_proj.bias)


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def graph_fwd_ms(fn, iters):
    """Forward time with the host taken out: the call captured once in a CUDA graph and replayed."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        fn()
    g.replay()
    return timed(g.replay, iters)


def kernel_times(nq, G, drop_p, iters):
    """Per-kernel device time (us) of attn_fwd / attn_bwd_dq / attn_bwd_dkv alone, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    from bevformer_b200 import _lib, ops
    dev = torch.device("cuda:0")
    lib = _lib.load()
    C, bs = 256, 1
    qk = torch.randn(nq, bs, 2 * C, device=dev, dtype=torch.bfloat16)
    v, do = (torch.randn(nq, bs, C, device=dev, dtype=torch.bfloat16) for _ in range(2))
    out, dv = torch.empty_like(v), torch.empty_like(v)
    dqk = torch.empty_like(qk)
    lse, delta = (torch.empty(bs * nq * 8, device=dev) for _ in range(2))
    sb = ops.seed_state(dev)
    st = torch.cuda.current_stream().cuda_stream
    esz = 2

    def step():
        _lib.check(lib.bevf_attn_forward(qk.data_ptr(), 2 * C, qk.data_ptr() + C * esz, 2 * C, v.data_ptr(), C,
                                         out.data_ptr(), C, lse.data_ptr(), nq, nq, bs, 8, 32, G, 32 ** -0.5,
                                         drop_p, 7, sb.data_ptr(), ops.BF16, st), lib)
        _lib.check(lib.bevf_attn_backward(qk.data_ptr(), 2 * C, qk.data_ptr() + C * esz, 2 * C, v.data_ptr(), C,
                                          out.data_ptr(), C, do.data_ptr(), C, lse.data_ptr(), delta.data_ptr(),
                                          dqk.data_ptr(), 2 * C, dqk.data_ptr() + C * esz, 2 * C, dv.data_ptr(), C,
                                          nq, nq, bs, 8, 32, G, 32 ** -0.5, drop_p, 7, sb.data_ptr(), ops.BF16, st),
                   lib)
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
    res = {}
    for ev in prof.key_averages():
        for k in ("attn_fwd", "attn_bwd_dq", "attn_bwd_dkv"):
            if k + "<" in ev.key or ev.key.endswith(k):
                res[k] = ev.device_time_total / ev.count
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda")
    props = torch.cuda.get_device_properties(dev)
    clock_hz = float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                                    capture_output=True, text=True).stdout.split()[0]) * 1e6
    exp_rate = props.multi_processor_count * 16 * clock_hz
    print("gpu:", gpu_info())
    results = []
    # kernels alone: floors per kernel.  exp: one per score per pass.  Tensor-core FLOPs per score:
    # fwd QK^T + PV = 4 * 32, dQ pass QK^T + dO V^T + dS K = 6 * 32, dK/dV pass K Q^T + V dO^T + Z^T dO + dS^T Q = 8 * 32
    flops_per_score = {"attn_fwd": 4 * 32, "attn_bwd_dq": 6 * 32, "attn_bwd_dkv": 8 * 32}
    for name, nq, G in (("train", 9900, 11), ("eval", 900, 1)):
        scores = G * 8 * (nq // G) ** 2
        for drop in (0.0, 0.1):
            kt = kernel_times(nq, G, drop, args.iters)
            for k, us in kt.items():
                row = dict(section="kernel", shape=name, dropout=drop, kernel=k, us=round(us, 2),
                           exp_floor_us=round(scores / exp_rate * 1e6, 2),
                           exp_floor_share=round(scores / exp_rate * 1e6 / us, 3),
                           tc_tflops=round(flops_per_score[k] * scores / us / 1e6, 1),
                           tc_floor_share_989=round(flops_per_score[k] * scores / TC_PEAK * 1e6 / us, 3))
                results.append(row)
                print(json.dumps(row))
    # whole module (three GEMMs, adds, dropout, autograd and Python included): end-to-end times, not kernel shares
    for name, nq, group, train in (("train", 9900, 11, True), ("eval", 900, 11, False)):
        torch.manual_seed(0)
        m = GroupMultiheadAttention(256, 8, dropout=0.1, group=group).to(dev, torch.bfloat16).train(train)
        x = torch.randn(nq, 1, 256, device=dev, dtype=torch.bfloat16, requires_grad=True)
        pos = torch.randn_like(x)
        gy = torch.randn_like(x)
        paths = {"module": lambda: m(x, query_pos=pos), "reference": lambda: reference_forward(m, x, pos, group),
                 "sdpa": lambda: sdpa_forward(m, x, pos, group)}
        times = {k: {"fwd": [], "fwd_bwd": [], "fwd_graph": []} for k in paths}
        for fn in paths.values():                      # warm-up of every path
            for _ in range(3):
                fn().backward(gy)
        for _ in range(args.rounds):
            for k, fn in paths.items():
                with torch.no_grad():
                    times[k]["fwd"].append(timed(fn, args.iters))
                times[k]["fwd_bwd"].append(timed(lambda: fn().backward(gy), args.iters))
                if not train:
                    times[k]["fwd_graph"].append(graph_fwd_ms(fn, args.iters))
        for k, t in times.items():
            row = dict(section="module_e2e", shape=name, path=k, fwd_ms=round(min(t["fwd"]), 4),
                       fwd_bwd_ms=round(min(t["fwd_bwd"]), 4))
            if t["fwd_graph"]:
                row["fwd_graph_replay_ms"] = round(min(t["fwd_graph"]), 4)
            results.append(row)
            print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
