"""Host-side pieces of deterministic mode (no GPU): the fixed-point fraction-bit choice of the sampler backward and
the PyTorch-style alert of ops without a deterministic implementation."""
import math
import warnings

import pytest
import torch

from bevformer_b200 import _lib, ops


@pytest.fixture
def restore_flag():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.mark.parametrize("rows,L,P", [(1, 1, 1), (40000, 1, 4), (44511, 4, 8), (2 ** 20, 4, 8), (2 ** 31 - 1, 16, 16)])
def test_frac_bits_leave_no_room_for_overflow(rows, L, P):
    k = _lib.load().bevf_msda_fx_frac_bits(rows, L, P)
    count = rows * L * P * 4
    assert k == min(40, 62 - math.ceil(math.log2(count)))
    assert count * 2 ** k <= 2 ** 62           # every contribution is below 2^k after scaling: the sum fits int64


def test_frac_bits_rejects_bad_sizes():
    lib = _lib.load()
    assert lib.bevf_msda_fx_frac_bits(-1, 1, 1) == -1 and lib.bevf_msda_fx_frac_bits(10, 0, 4) == -1


def test_alert_follows_pytorch_contract(restore_flag):
    torch.use_deterministic_algorithms(False)
    ops.alert_not_deterministic("x")                         # off: silent
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
        ops.alert_not_deterministic("x")
    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        ops.alert_not_deterministic("x")
    assert any("deterministic" in str(w.message) for w in rec)
