"""ops.gv_replicas_for / ops.replica_plan: which pyramid levels the mixed sampler backward accumulates in replicated
scaled-fp16 copies, and how many (host logic, no GPU)."""
import pytest

from bevformer_b200 import ops

BASE = [(116, 200), (58, 100), (29, 50), (15, 25)]
SMALL4 = [(92, 160), (46, 80), (23, 40), (12, 20)]


@pytest.fixture(autouse=True)
def policy_env(monkeypatch):
    monkeypatch.delenv("BEVF_GV_ACC", raising=False)
    monkeypatch.delenv("BEVF_GV_MAXCONTRIB", raising=False)


def test_base():
    # SCA at base: 10 / 41 / 164 / 630 contributions per pixel; levels 0-1 fp16, level 3 dense, level 2 in 3 copies
    assert ops.gv_replicas_for(44511 / 6, 8, BASE) == {2: 3}
    assert ops.replica_plan({2: 3}, 2) == (1, 3)


def test_small4():
    rows = 22500 * 1.9 / 6                       # about 1.9 in-view cameras per BEV query of the 150 x 150 grid
    mode = ops.gv_mode_for(rows, 8, SMALL4)
    kd = ops.dense_levels_for(rows, 8, SMALL4)
    reps = ops.gv_replicas_for(rows, 8, SMALL4)
    assert sorted(reps) == list(range(mode[2], len(SMALL4) if kd is None else kd))
    for l, k in reps.items():
        h, w = SMALL4[l]
        assert (k - 1) * 64 < rows * 8 * 4 / (h * w) <= k * 64


def test_tiny_and_tsa_have_none():
    assert ops.gv_replicas_for(2500.0, 8, [(15, 25)]) == {}             # bevformer_tiny: no mixed mode
    assert ops.gv_replicas_for(40000.0, 4, [(1, 40000)]) == {}         # TSA: every level fp16 already


def test_fp32_accumulation_has_none(monkeypatch):
    monkeypatch.setenv("BEVF_GV_ACC", "fp32")
    assert ops.gv_replicas_for(44511 / 6, 8, BASE) == {}


def test_cap_follows_maxcontrib(monkeypatch):
    monkeypatch.setenv("BEVF_GV_MAXCONTRIB", "32")
    # cut at 32: level 0 (10) fp16, levels 1 (41) and 2 (164) replicated in 2 and 6 copies, level 3 dense
    assert ops.gv_replicas_for(44511 / 6, 8, BASE) == {1: 2, 2: 6}
    assert ops.replica_plan({1: 2, 2: 6}, 1) == (2, 6)


def test_plan_needs_levels_right_after_the_fine_ones():
    assert ops.replica_plan({}, 2) == (0, 1)
    assert ops.replica_plan(None, 2) == (0, 1)
    with pytest.raises(RuntimeError):
        ops.replica_plan({3: 2}, 1)
