"""Mixed precision without a GPU: how the compute dtype is resolved, the fp16 entry points of the library, and the
reference's fp16 config building unchanged."""
import os
import re
import subprocess

import pytest
import torch

from bevformer_b200 import precision
from oracle import mmcv_stub

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CFG = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs") + os.sep


class _M(torch.nn.Module):
    pass


def test_compute_dtype_resolution():
    m = _M()
    x16, x32 = torch.zeros(2, dtype=torch.bfloat16), torch.zeros(2)
    assert precision.compute_dtype(m, x32) == torch.float32
    assert precision.compute_dtype(m, None, x16) == torch.bfloat16
    assert precision.compute_dtype(m) == torch.float32
    m.fp16_enabled = True                                  # mmcv's wrap_fp16_model
    assert precision.compute_dtype(m, x32) == torch.float16
    m.fp16_enabled = False
    assert precision.compute_dtype(m, x32) == torch.float32


def test_autocast_wins(monkeypatch):
    """Under CUDA autocast its dtype wins over fp16_enabled and the inputs (autocast state faked: no GPU here)."""
    m = _M()
    m.fp16_enabled = True
    for dt in (torch.bfloat16, torch.float16):
        monkeypatch.setattr(torch, "is_autocast_enabled", lambda device_type=None: True)
        monkeypatch.setattr(torch, "get_autocast_dtype", lambda device_type, dt=dt: dt)
        got, ctx = precision.entered(m, torch.zeros(2))
        assert got == dt and isinstance(ctx, torch.autocast)
    monkeypatch.undo()
    got, _ = precision.entered(m, torch.zeros(2))
    assert got == torch.float16


def test_cast_leaves_non_floating_inputs():
    i = torch.arange(4)
    f = torch.zeros(3)
    assert precision.cast(i, torch.float16) is i and precision.cast(None, torch.float16) is None
    assert precision.cast(f, torch.float16).dtype == torch.float16
    out = precision.cast([f, i], torch.bfloat16)
    assert out[0].dtype == torch.bfloat16 and out[1] is i


def test_header_and_library_export_fp16():
    hdr = open(os.path.join(ROOT, "include", "bevformer_b200.h")).read()
    assert re.search(r"BEVF_DTYPE_F16\s*=\s*2", hdr)
    names = ["bevf_linear_forward_dt", "bevf_linear_dgrad_dt", "bevf_linear_dgrad_acc_dt", "bevf_linear_wgrad_dt",
             "bevf_linear_wgrad_out_dt", "bevf_linear_wgrad_into_dt"]
    for n in names:
        assert n + "(" in hdr, n
    from bevformer_b200 import _lib, build
    lib = build.build()
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for n in names:
        assert re.search(r"\b" + n + r"\b", syms), n
        assert n in _lib.SIGNATURES
    from bevformer_b200 import ops
    assert ops._DT[torch.float16] == 2


@pytest.mark.skipif(not os.path.isdir(REF_CFG), reason="needs the reference tree (BEVF_REFERENCE_ROOT)")
def test_reference_fp16_config_builds():
    """The reference's fp16 config (bevformer_fp16/bevformer_tiny_fp16.py) builds unchanged: same encoder as tiny."""
    from bevformer_b200.plugin import config
    enc = config.build_encoder(REF_CFG + "bevformer_fp16/bevformer_tiny_fp16.py")
    assert type(enc).__name__ == "BEVFormerEncoder"
    assert sum(p.numel() for p in enc.parameters()) == 2026368
