"""Shapes of the weight-stationary GEMM tile plan that test_gemm_gpu.py does not reach: 256-wide column
blocks with a ragged row tail, fp32 output with a residual over three column blocks, a half-empty last column
block, and 64-wide blocks over a long reduction.  Each case runs in a subprocess with a hard timeout."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FWD_CASES = [
    # (M, N, K, relu, residual, fp32_out, bf16_bias)
    (300, 256, 256, True, True, False, False),       # BN 256, ragged M tail, residual
    (44511, 768, 256, False, True, True, False),     # three 256 blocks, fp32 out (two staging fills), residual
    (300, 192, 512, False, True, True, True),        # BN 128, second block half empty, bf16 bias
    (4099, 320, 128, True, False, False, False),     # BN 256 over N = 320: last block 64 wide
    (77, 16, 1024, False, True, False, False),       # BN 64 over a 1024-long reduction, one partial tile
]

FWD_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, {root!r})
    from bevformer_b200 import ops
    M, N, K, relu, use_res, f32, bbf16 = {case!r}
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    b = torch.randn(N, generator=g).cuda()
    if bbf16: b = b.bfloat16()
    res = torch.randn(M, N, generator=g).bfloat16().cuda() if use_res else None
    y = ops.linear_tc(x, w, b, res, relu, torch.float32 if f32 else torch.bfloat16)
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t() + b.float()
    if relu: ref = ref.relu()
    if use_res: ref = ref + res.float()
    err = (y.float() - ref).abs().max().item()
    print("ERR", err, flush=True)
    assert err < (2e-3 if f32 else 4e-2), err
    assert torch.equal(y, ops.linear_tc(x, w, b, res, relu, torch.float32 if f32 else torch.bfloat16))
""")


@pytest.mark.parametrize("case", FWD_CASES)
def test_linear_ws_forward(case):
    r = subprocess.run([sys.executable, "-c", FWD_SCRIPT.format(root=ROOT, case=case)], capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]


DGRAD_CASES = [
    # (M, N, K, addend): dX (M, K) = dY (M, N) . W (N, K)
    (44511, 768, 256, True),      # BN 64 over a 768-long reduction, four column blocks, ragged M
    (300, 192, 512, True),        # BN 256, R = 192, ragged M
    (4099, 128, 320, False),      # BN 256 over K = 320: last block 64 wide
]

DGRAD_SCRIPT = textwrap.dedent("""
    import sys, torch
    sys.path.insert(0, {root!r})
    from bevformer_b200 import ops
    M, N, K, use_add = {case!r}
    g = torch.Generator().manual_seed(M + N + K)
    dy = torch.randn(M, N, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / N ** 0.5).bfloat16().cuda()
    prev = torch.randn(M, K, generator=g).bfloat16().cuda() if use_add else None
    dx = ops.linear_dgrad_tc(dy, w, addend=prev)
    torch.cuda.synchronize()
    ref = dy.float() @ w.float()
    if use_add: ref = ref + prev.float()
    err = (dx.float() - ref).abs().max().item()
    print("ERR", err, flush=True)
    assert dx.shape == (M, K) and err < 4e-2 * max(1.0, ref.abs().max().item() / 8), err
    # same products in the same order as the forward kernel on W^T
    assert torch.equal(dx, ops.linear_tc(dy, w.t().contiguous(), None, prev))
""")


@pytest.mark.parametrize("case", DGRAD_CASES)
def test_linear_ws_dgrad(case):
    r = subprocess.run([sys.executable, "-c", DGRAD_SCRIPT.format(root=ROOT, case=case)], capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
