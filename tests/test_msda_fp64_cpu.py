"""tests/msda_fp64_oracle.py pinned against Oracle-S, and its bars shown to reject plausible kernel bugs.

The restatement rounds the sample coordinate as the kernels do (two float32 operations) and computes the rest in
float64.  Where float32 and float64 coordinates pick the same cell (locations that are multiples of 2^-12 on small
maps: loc * W - 0.5 is exact in both), it must equal Oracle-S in float64 to 1e-12.  Exactly on cell borders its cell
choice must be Oracle-S float32's (same rounding sequence), which shows in grad_loc's slope.  The mutation checks
apply each bug to the restatement and require the bars of the GPU file to reject the result."""
import pytest
import torch

from oracle import msda_oracle
from tests import msda_fp64_oracle as mo

F64 = torch.float64


def _grid_inputs(levels, M, P, D, NB, Q, seed, extremes=True):
    d = mo.make_inputs(levels, M, P, D=D, NB=NB, Q=Q, seed=seed, border_frac=0.0)
    loc = torch.round(d["loc"] * 4096) / 4096                                  # exact in fp32 and fp64
    if extremes:
        flat = loc.view(-1, 2)
        special = torch.tensor([[float("nan"), 0.5], [0.5, float("inf")], [-float("inf"), 0.5], [1e9, 0.5],
                                [0.5, -1e9], [-0.5, 0.5], [1.5, 0.5], [0.5, -0.25]])
        for i in range(special.shape[0]):
            flat[(7 * i + 3) % flat.shape[0]] = special[i]
    d["loc"] = loc.contiguous()
    return d


def _oracle64(d, row_sel=None):
    v, hw, st = d["value"].double(), d["level_hw"], d["level_start"]
    out = msda_oracle.msda_forward(v, hw, st, d["loc"].double(), d["attn"].double())
    gv, gl, ga = msda_oracle.msda_backward(v, hw, st, d["loc"].double(), d["attn"].double(), d["grad_out"].double())
    return out, gv, gl, ga


@pytest.mark.parametrize("shape", [
    dict(levels=[(6, 5), (3, 2), (1, 1)], M=3, P=3, D=32, NB=2, Q=7),
    dict(levels=[(1, 9), (8, 1)], M=2, P=5, D=30, NB=1, Q=5),
    dict(levels=[(4, 4)], M=1, P=2, D=4, NB=3, Q=4),
])
def test_dense_layout_matches_oracle_s_f64(shape):
    d = _grid_inputs(seed=1, **shape)
    out, gv, gl, ga = _oracle64(d)
    r_out, _ = mo.forward(d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"])
    r = mo.backward(d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"], d["grad_out"])
    for name, got, want in (("out", r_out, out), ("grad_value", r["grad_value"], gv),
                            ("grad_loc", r["grad_loc"], gl), ("grad_attn", r["grad_attn"], ga)):
        assert got.shape == want.shape, name
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12), (name, (got - want).abs().max().item())
    assert torch.isfinite(r["grad_loc"]).all() and torch.isfinite(r_out).all()


def test_row_list_layout_matches_oracle_s_f64():
    """Row list with unused rows (-1): every used row equals Oracle-S on its own map; unused rows add nothing."""
    levels, M, P, D, NB, R = [(5, 7), (2, 3)], 5, 3, 32, 3, 23
    d = mo.make_inputs(levels, M, P, D=D, NB=NB, R=R, unused=(4, 5, 17), seed=2, border_frac=0.0)
    d["loc"] = (torch.round(d["loc"] * 4096) / 4096).contiguous()
    rm = d["row_map"].long()
    out, _ = mo.forward(d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"], d["row_map"])
    r = mo.backward(d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"], d["grad_out"], d["row_map"])
    gv_ref = torch.zeros(d["value"].shape, dtype=F64)
    for b in range(NB):
        idx = (rm == b).nonzero().flatten()
        lc, ac = d["loc"][idx][None].double(), d["attn"][idx][None].double()
        o = msda_oracle.msda_forward(d["value"][b:b + 1].double(), d["level_hw"], d["level_start"], lc, ac)[0]
        gv, gl, ga = msda_oracle.msda_backward(d["value"][b:b + 1].double(), d["level_hw"], d["level_start"], lc, ac,
                                               d["grad_out"][idx][None].double())
        assert torch.allclose(out[idx], o, rtol=1e-12, atol=1e-12)
        assert torch.allclose(r["grad_loc"][idx], gl[0], rtol=1e-12, atol=1e-12)
        assert torch.allclose(r["grad_attn"][idx], ga[0], rtol=1e-12, atol=1e-12)
        gv_ref[b] = gv[0]
    assert torch.allclose(r["grad_value"], gv_ref, rtol=1e-12, atol=1e-12)
    dead = (rm < 0).nonzero().flatten()
    assert out[dead].abs().max() == 0 and r["grad_loc"][dead].abs().max() == 0
    # counts: every non-zero-weight corner of a used row is one contribution
    assert r["gv_count"][..., 0].sum() > 0


def test_cell_choice_on_borders_matches_oracle_s_f32():
    """On cell borders (x, y exactly integers after the float32 rounding) and at -1 + ulp / W - ulp the
    restatement's cell is Oracle-S float32's: same sample validity, and grad_loc with the same slope (the float32
    oracle's own rounding stays far below the slope changes a cell flip would cause)."""
    levels, M, P, D = [(7, 11), (3, 5), (1, 3)], 2, 4, 8
    gen = torch.Generator().manual_seed(5)
    hw, starts, S = mo.pyramid(levels)
    n = 64
    loc = mo.border_locs(hw, n * M * P, gen, kinds=("integer", "inside_edge", "outside_edge"))
    loc = loc.view(1, n, M, P, len(levels), 2).permute(0, 1, 2, 4, 3, 5).contiguous()
    value = torch.randn(1, S, M, D, generator=gen)
    attn = torch.rand(1, n, M, len(levels), P, generator=gen)
    gout = torch.randn(1, n, M * D, generator=gen)
    ogv, ogl, oga = msda_oracle.msda_backward(value, hw, starts, loc, attn, gout)
    r = mo.backward(value, hw, starts, loc, attn, gout)
    bar = 1e-5 * (1 + r["gl_mag"])
    assert ((ogl.double() - r["grad_loc"]).abs() <= bar).all()
    assert ((oga.double() - r["grad_attn"]).abs() <= 1e-5 * (1 + r["ga_mag"])).all()
    # every kind of border position is present: valid and invalid samples, x exactly on an integer
    x, _, valid = mo._coords(loc, hw)
    assert valid.any() and (~valid).any() and ((x == torch.floor(x)) & valid).any()


# ------------------------------------------------------------------------------------------------
# mutation checks: each bug must break the bar of the loosest GPU path that the output goes through
# ------------------------------------------------------------------------------------------------
MUT_CASE = mo.SHAPES["rows_m5"]          # see its comment in SHAPES
MUT_SEED = 4                             # with D = 32: the inputs of the GPU file's rows_m5 backward cases


def _bars(d, fwd_mag, fwd_ref, r):
    """The loosest bars of the GPU file for each output (bf16 value, bf16 output, scaled fp16 / dense grad_value)."""
    L, P = d["attn"].shape[-2:]
    D = d["value"].shape[-1]
    scale = 2.0 ** (3 - __import__("math").floor(__import__("math").log2(d["grad_out"].abs().max().item())))
    gvb = torch.maximum(mo.bar_gv_f16(r["gv_mag"], r["gv_count"], r["grad_value"], scale),
                        mo.bar_gv_dense(r["gv_mag"], r["gv_dense_mag"], r["gv_count"]))
    return dict(out=mo.bar_forward(fwd_mag, fwd_ref, L * P, torch.bfloat16, True), grad_value=gvb,
                grad_loc=mo.bar_grad_loc(r["gl_mag"], D), grad_attn=mo.bar_grad_attn(r["ga_mag"], D))


@pytest.mark.parametrize("mutation", mo.MUTATIONS)
def test_bars_reject_mutation(mutation):
    d = mo.make_inputs(seed=MUT_SEED, **MUT_CASE)
    args = (d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"])
    ref_out, fwd_mag = mo.forward(*args, d["row_map"])
    r = mo.backward(*args, d["grad_out"], d["row_map"], dense_mult=True)
    bars = _bars(d, fwd_mag, ref_out, r)
    # the unmutated restatement holds its own bars trivially; the mutated one must not
    mut_out, _ = mo.forward(*args, d["row_map"], mutate=mutation)
    m = mo.backward(*args, d["grad_out"], d["row_map"], mutate=mutation)
    got = dict(out=mut_out, grad_value=m["grad_value"], grad_loc=m["grad_loc"], grad_attn=m["grad_attn"])
    ref = dict(out=ref_out, grad_value=r["grad_value"], grad_loc=r["grad_loc"], grad_attn=r["grad_attn"])
    rejected = {k: bool(((got[k] - ref[k]).abs() > bars[k]).any()) for k in got}
    assert any(rejected.values()), (mutation, rejected)
    # the outputs each bug must show in
    must = {"swap_01_10": ("out", "grad_value", "grad_loc", "grad_attn"),
            "drop_last_sample": ("out", "grad_value"),
            "neighbour_level_offset": ("out", "grad_value", "grad_attn"),
            "grad_loc_without_wh": ("grad_loc",),
            "scatter_to_partner_map": ("grad_value",),
            "fma_coordinates": ("grad_loc",)}[mutation]
    assert all(rejected[k] for k in must), (mutation, rejected)


def test_bars_reject_mutation_dense_layout():
    """The same bugs on a dense (B, Q, ...) launch with fp32 storage bars."""
    d = mo.make_inputs([(6, 10), (3, 5)], 8, 3, D=32, NB=2, Q=9, seed=3, border_frac=0.3)
    args = (d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"])
    ref_out, mag = mo.forward(*args)
    r = mo.backward(*args, d["grad_out"])
    for mutation in ("swap_01_10", "drop_last_sample", "neighbour_level_offset", "grad_loc_without_wh",
                     "fma_coordinates"):
        o, _ = mo.forward(*args, mutate=mutation)
        m = mo.backward(*args, d["grad_out"], mutate=mutation)
        bad = ((o - ref_out).abs() > mo.bar_forward(mag, ref_out, 6)).any() or \
            ((m["grad_value"] - r["grad_value"]).abs() > mo.bar_grad_value_f32(r["gv_mag"], r["gv_count"])).any() or \
            ((m["grad_loc"] - r["grad_loc"]).abs() > mo.bar_grad_loc(r["gl_mag"], 32)).any()
        assert bad, mutation


def test_grad_value_rows_subset_matches_full():
    """backward(gv_rows=...) returns exactly the full grad_value's rows (what the large-offset GPU case uses)."""
    d = mo.make_inputs([(5, 6), (2, 2)], 3, 2, D=8, NB=2, R=20, unused=(3,), seed=4)
    args = (d["value"], d["level_hw"], d["level_start"], d["loc"], d["attn"], d["grad_out"], d["row_map"])
    full = mo.backward(*args)
    NB, S, M, D = d["value"].shape
    rows = torch.tensor([0, 5, S + 3, 2 * S - 1])
    sub = mo.backward(*args, gv_rows=rows)
    flat = full["grad_value"].reshape(NB * S, M, D)
    assert torch.equal(sub["grad_value"], flat[rows])
    assert torch.equal(sub["gv_count"], full["gv_count"].reshape(NB * S, M, D)[rows])
