"""GroupMultiheadAttention (group_attention.py:18-162), the decoder self-attention of the Group DETR BEVFormerV2
configs: registry coverage of all seven V2 configs, parameter layout and the torch path against the reference's own
class (its results stored under tests/golden/ref_group_attn_*.npz; ``python -m tests.test_group_attention_cpu``
regenerates them from an unmodified reference tree through ``reference_results()``)."""
import copy
import glob
import importlib
import os
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

from bevformer_b200 import synthetic as syn
from oracle import mmcv_stub
from tests.util import GOLDEN, fixed_projection, reference_result, reference_sample

V2_CFGS = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs", "bevformerv2")
C, HEADS, BS, NQ, GROUP = 256, 8, 2, 40, 4

# constructor spellings: the V2 configs' (deprecated `dropout`), the explicit one, batch-first without biases
SPELLINGS = (dict(embed_dims=C, num_heads=HEADS, dropout=0.1, group=11),
             dict(embed_dims=C, num_heads=HEADS, attn_drop=0.1, proj_drop=0.2, dropout_layer=None, group=2),
             dict(embed_dims=C, num_heads=HEADS, batch_first=True, bias=False))

# module cases: (name, training, batch_first, positional encodings, separate key tensor, attn_mask)
CASES = (("eval_seq", False, False, "query_pos", False, False),
         ("train_seq", True, False, "query_pos", False, False),
         ("train_bf_key", True, True, "both", True, False),
         ("eval_bf_nopos", False, True, None, False, False),
         ("eval_mask", False, False, "query_pos", False, True))

_REF_GROUP = None


def load_reference_group_attention():
    """The reference's own GroupMultiheadAttention, imported unmodified behind the oracle's mmcv stub plus the three
    symbols this file needs besides: mmcv.cnn.build_conv_layer, mmcv.cnn.bricks.drop.build_dropout (mmcv's Dropout
    is nn.Dropout(drop_prob)) and mmcv.utils.to_2tuple."""
    global _REF_GROUP
    if _REF_GROUP is not None:
        return _REF_GROUP
    mmcv_stub.load_reference_modules()
    cnn = sys.modules["mmcv.cnn"]
    if not hasattr(cnn, "build_conv_layer"):
        cnn.build_conv_layer = lambda cfg, *a, **k: nn.Conv2d(*a, **k)

    def build_dropout(cfg, default_args=None):
        cfg = dict(cfg)
        assert cfg.pop("type", "Dropout") == "Dropout"
        return nn.Dropout(cfg.get("drop_prob", 0.5))

    extra = {"mmcv.cnn.bricks.drop": mmcv_stub._mod("mmcv.cnn.bricks.drop", build_dropout=build_dropout)}
    saved = mmcv_stub._with_bricks_stub()
    saved_extra = {k: sys.modules.get(k) for k in extra}
    sys.modules.update(extra)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = importlib.import_module(mmcv_stub._PKG + ".group_attention")
    finally:
        mmcv_stub._restore(saved)
        mmcv_stub._restore(saved_extra)
    _REF_GROUP = mod.GroupMultiheadAttention
    return _REF_GROUP


def load_reference_group_decoder():
    """The reference's DetectionTransformerDecoder (decoder.py:52-129) with its GroupMultiheadAttention registered."""
    dec = mmcv_stub.load_reference_decoder()
    mmcv_stub.ATTENTION.register_module(name="GroupMultiheadAttention", module=load_reference_group_attention(),
                                        force=True)
    return dec


# toy group decoders: the configs' 4 sampling points, and 8 (a 192-wide offsets|weights head, which the 16-bit GEMMs
# take, so the decoder also runs in bf16)
DECODER_POINTS = {"group_attn_decoder": 4, "group_attn_decoder_p8": 8}


def group_decoder_cfg(num_points=4):
    """The V2 decoder (3 layers here) with Group DETR's self-attention, group 4 over 40 queries, dropout off."""
    cfg = copy.deepcopy(syn.DECODER_CFG)
    layer = cfg["transformerlayers"]
    layer["attn_cfgs"][0] = dict(type="GroupMultiheadAttention", group=GROUP, embed_dims=C, num_heads=HEADS,
                                 dropout=0.0)
    layer["attn_cfgs"][1]["dropout"] = 0.0
    layer["attn_cfgs"][1]["num_points"] = num_points
    layer["ffn_dropout"] = 0.0
    return cfg


def case_inputs(case, dtype=torch.float64, device="cpu"):
    """(module kwargs, forward tensors) of a module case: seeded, sequence-first or batch-first."""
    name, training, batch_first, pos, sep_key, mask = case
    g = torch.Generator().manual_seed(17 + [c[0] for c in CASES].index(name))
    shape = (BS, NQ, C) if batch_first else (NQ, BS, C)
    t = {"query": torch.randn(shape, generator=g)}
    if pos in ("query_pos", "both"):
        t["query_pos"] = torch.randn(shape, generator=g)
    if sep_key:
        t["key"] = torch.randn(shape, generator=g)
    if pos == "both":
        t["key_pos"] = torch.randn(shape, generator=g)
    t = {k: v.to(device, dtype).requires_grad_(True) for k, v in t.items()}
    if mask:
        t["attn_mask"] = (torch.rand(NQ, NQ, generator=g) < 0.3).fill_diagonal_(False).to(device)
    return dict(embed_dims=C, num_heads=HEADS, group=GROUP, batch_first=batch_first), t


def run_case(module, case, tensors):
    """Forward + backward of (out * fixed projection).sum(); returns {name: tensor} of out and every gradient."""
    out = module(**tensors)
    (out * fixed_projection(out.shape).to(out)).sum().backward()
    res = {"out": out.detach()}
    for k, v in tensors.items():
        if v.is_floating_point():
            res["grad_" + k] = v.grad
    for k, p in module.named_parameters():
        res["grad_" + k] = p.grad
    return res


def decoder_inputs(dtype=torch.float64, device="cpu"):
    w = syn.WORKLOADS["toy"]
    query, query_pos, bev, ref, reg = syn.make_decoder_inputs(w, bs=BS, num_query=NQ)
    kw = dict(key=None, reference_points=ref.to(device, dtype), reg_branches=reg.to(device, dtype),
              cls_branches=None, spatial_shapes=torch.tensor([[w.bev_h, w.bev_w]], device=device),
              level_start_index=torch.tensor([0], device=device))
    t = {k: v.to(device, dtype).requires_grad_(True) for k, v in (("query", query), ("query_pos", query_pos),
                                                                  ("value", bev))}
    return t, kw


def run_decoder(dec, t, kw):
    states, refs = dec(**t, **kw)
    (states * fixed_projection(states.shape).to(states)).sum().backward()
    return {"states": states.detach(), "refs": refs.detach(), "grad_query": t["query"].grad,
            "grad_query_pos": t["query_pos"].grad, "grad_value": t["value"].grad}


def reference_results():
    """{golden name: arrays} from the reference's own GroupMultiheadAttention / decoder (needs the reference tree)."""
    ref = load_reference_group_attention()
    default_dl = next(d for d in ref.__init__.__defaults__ if isinstance(d, dict))
    res = {}
    for i, kw in enumerate(SPELLINGS):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = ref(**copy.deepcopy(kw))
        # the deprecated `dropout` kwarg writes into the shared default dict: every construction here is made as in
        # a fresh process
        default_dl["drop_prob"] = 0.0
        sd = m.state_dict()
        res[f"group_attn_params{i}"] = {
            "keys": np.array(list(sd)), "shapes": np.array([str(tuple(v.shape)) for v in sd.values()]),
            "drop": np.array([m.attn.dropout, m.proj_drop.p,
                              m.dropout_layer.p if isinstance(m.dropout_layer, nn.Dropout) else -1.0])}
    for case in CASES:
        kw, t = case_inputs(case)
        m = ref(**kw).double().train(case[1])
        m.load_state_dict(syn.make_random_state_dict(m, 3))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            got = run_case(m, case, t)
        res[f"group_attn_{case[0]}"] = {f"{k}__{f}": v for k, r in got.items() for f, v in reference_sample(r).items()}
    D = load_reference_group_decoder()
    for name, points in DECODER_POINTS.items():
        cfg = group_decoder_cfg(points)
        cfg.pop("type")
        dec = D(**cfg).double().train()
        dec.load_state_dict(syn.make_random_state_dict(dec, 5))
        t, kw = decoder_inputs()
        got = run_decoder(dec, t, kw)
        out = {f"{k}__{f}": v for k, r in got.items() for f, v in reference_sample(r).items()}
        out["keys"] = np.array(sorted(dec.state_dict()))
        res[name] = out
    return res


def write_golden():
    for name, arrays in reference_results().items():
        path = os.path.join(GOLDEN, f"ref_{name}.npz")
        np.savez_compressed(path, **arrays)
        print(f"ref_{name}: {os.path.getsize(path)} bytes")


def sampled_err(got: torch.Tensor, ref, name: str) -> float:
    """max |got - ref| over the stored sample positions, relative to max |ref| of the whole tensor."""
    assert tuple(got.shape) == tuple(int(x) for x in ref[name + "__shape"]), name
    flat = got.detach().reshape(-1).double().cpu()
    idx = torch.from_numpy(ref[name + "__idx"])
    want = torch.from_numpy(ref[name + "__sample"]).double()
    return ((flat[idx] - want).abs().max() / max(float(ref[name + "__stats"][3]), 1e-30)).item()


def golden_names(ref):
    return sorted({k.split("__")[0] for k in ref.files if "__" in k})


@pytest.mark.skipif(not os.path.isdir(V2_CFGS), reason="needs the reference tree (BEVF_REFERENCE_ROOT)")
def test_all_seven_v2_configs_build():
    from bevformer_b200.plugin import GroupMultiheadAttention, registry
    paths = sorted(glob.glob(os.path.join(V2_CFGS, "*.py")))
    assert len(paths) == 7
    grouped = 0
    for path in paths:
        ns = {}
        with open(path) as f:
            exec(compile(f.read(), path, "exec"), ns)  # noqa: S102 - reference config, read-only
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m = registry.build_from_cfg(copy.deepcopy(ns["model"]["pts_bbox_head"]["transformer"]), registry.TRANSFORMER)
        ga = [x for x in m.modules() if isinstance(x, GroupMultiheadAttention)]
        if ga:
            grouped += 1
            assert all(x.group == ns["group_detr"] and x.attn.dropout == 0.1 for x in ga)
    assert grouped == 5


@pytest.mark.parametrize("i", range(len(SPELLINGS)))
def test_parameters_match_reference_class(i):
    from bevformer_b200.plugin import GroupMultiheadAttention
    want = reference_result(f"group_attn_params{i}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = GroupMultiheadAttention(**copy.deepcopy(SPELLINGS[i]))
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in want["keys"]]
    assert [str(tuple(v.shape)) for v in sd.values()] == [str(s) for s in want["shapes"]]
    got_drop = [m.attn.dropout, m.proj_drop.p, m.dropout_layer.p if isinstance(m.dropout_layer, nn.Dropout) else -1.0]
    assert np.allclose(got_drop, want["drop"])


def test_deprecated_dropout_updates_the_given_dict_only():
    from bevformer_b200.plugin import GroupMultiheadAttention
    dl = dict(type="Dropout", drop_prob=0.0)
    with pytest.warns(DeprecationWarning):
        GroupMultiheadAttention(C, HEADS, dropout=0.3, dropout_layer=dl)
    assert dl["drop_prob"] == 0.3
    with pytest.warns(DeprecationWarning):
        GroupMultiheadAttention(C, HEADS, dropout=0.3)
    assert GroupMultiheadAttention(C, HEADS).dropout_layer.p == 0.0


def test_queries_must_split_into_groups():
    from bevformer_b200.plugin import GroupMultiheadAttention
    m = GroupMultiheadAttention(C, HEADS, group=3).train()
    with pytest.raises(RuntimeError):
        m(torch.randn(NQ, BS, C))
    m.eval()(torch.randn(NQ, BS, C))          # eval ignores the grouping


@pytest.mark.parametrize("name", sorted(DECODER_POINTS))
def test_group_decoder_parameters_match_reference(name):
    from bevformer_b200.plugin import build_transformer_layer_sequence
    dec = build_transformer_layer_sequence(group_decoder_cfg(DECODER_POINTS[name]))
    assert sorted(dec.state_dict()) == [str(k) for k in reference_result(name)["keys"]]


def test_unsupported_dropout_layer_type_raises():
    from bevformer_b200.plugin import GroupMultiheadAttention
    with pytest.raises(NotImplementedError):
        GroupMultiheadAttention(C, HEADS, dropout_layer=dict(type="DropPath", drop_prob=0.1))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_torch_path_matches_reference_fp64(case):
    from bevformer_b200.plugin import GroupMultiheadAttention
    want = reference_result(f"group_attn_{case[0]}")
    kw, t = case_inputs(case)
    m = GroupMultiheadAttention(**kw).double().train(case[1])
    m.load_state_dict(syn.make_random_state_dict(m, 3))
    got = run_case(m, case, t)
    assert sorted(got) == golden_names(want)
    for k, v in got.items():
        assert sampled_err(v, want, k) < 1e-12, k


if __name__ == "__main__":
    write_golden()
