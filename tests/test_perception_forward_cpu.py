"""PerceptionTransformer with its decoder, on CPU: parameter names against the reference class built from the same
dicts (golden ``perception_forward_toy``, made by the reference's own class), and the decoder-less instance."""
import copy
import os

import pytest

from bevformer_b200 import synthetic as syn
from oracle import mmcv_stub
from tests.util import golden

W = syn.WORKLOADS["toy"]
REF_CFG = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs") + os.sep


def _toy(decoder=True):
    from bevformer_b200.plugin import PerceptionTransformer
    return PerceptionTransformer(num_feature_levels=len(W.levels), num_cams=W.num_cams, encoder=syn.encoder_cfg(W),
                                 decoder=copy.deepcopy(syn.DECODER_CFG) if decoder else None,
                                 embed_dims=W.embed_dims, rotate_center=[W.bev_h // 2, W.bev_w // 2])


def test_keys_match_reference_class_with_decoder():
    m = _toy()
    assert sorted(m.state_dict()) == [str(k) for k in golden("perception_forward_toy")["keys"]]
    assert len(m.decoder.layers) == syn.DECODER_CFG["num_layers"]


@pytest.mark.skipif(not os.path.isdir(REF_CFG), reason="needs the reference tree (BEVF_REFERENCE_ROOT)")
@pytest.mark.parametrize("size", ["tiny", "base"])
def test_flagship_config_transformer_keys_match_reference(size):
    """The unchanged transformer dict of bevformer_{tiny,base}.py builds through this package's registry with exactly
    the keys of the reference class built from it, decoder included."""
    from bevformer_b200.plugin.config import load_config
    from bevformer_b200.plugin.registry import TRANSFORMER, build_from_cfg
    cfg = load_config(REF_CFG + f"bevformer/bevformer_{size}.py")["model"]["pts_bbox_head"]["transformer"]
    m = build_from_cfg(copy.deepcopy(cfg), TRANSFORMER)
    assert type(m).__name__ == "PerceptionTransformer" and m.decoder is not None
    assert sorted(m.state_dict()) == [str(k) for k in golden("perception_forward_toy")[f"keys_{size}"]]


def test_decoderless_forward_raises():
    m = _toy(decoder=False)
    assert m.decoder is None
    with pytest.raises(NotImplementedError):
        m(None, None)
    inp = syn.make_perception_inputs(W, bs=1)
    with pytest.raises(NotImplementedError):
        m(inp.mlvl_feats, inp.bev_queries, None, W.bev_h, W.bev_w, bev_pos=inp.bev_pos, img_metas=inp.img_metas)


def test_forward_has_no_cpu_path():
    m = _toy()
    inp = syn.make_perception_inputs(W, bs=1)
    from tests.golden.make_golden import v2_inputs
    _, oq, reg = v2_inputs(W)
    with pytest.raises(RuntimeError):
        m(inp.mlvl_feats, inp.bev_queries, oq, W.bev_h, W.bev_w, bev_pos=inp.bev_pos, reg_branches=reg,
          img_metas=inp.img_metas)
