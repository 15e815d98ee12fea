"""Generates tests/golden/perception_forward_toy.npz from the REFERENCE'S OWN PerceptionTransformer.forward
(Oracle-R, oracle/mmcv_stub.py), with the helpers and conventions of make_golden.py.  Needs a reference checkout
(BEVF_REFERENCE_ROOT); the test suite does not:

    python tests/golden/make_golden_perception.py
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from bevformer_b200 import synthetic as syn  # noqa: E402
from bevformer_b200.plugin import config  # noqa: E402
from oracle import mmcv_stub  # noqa: E402
from tests.golden.make_golden import (OUT, fixed_projection, grid_length_of, row_subset, save_capped,  # noqa: E402
                                      stats, v2_inputs)


def perception_forward_case(name, workload, seed=0, keep_rows=256):
    """The reference's own PerceptionTransformer.forward (transformer.py:202-289): get_bev_features with a
    rotated prev_bev, then the object-query decoder with box refinement; eval mode.  Gradients of bev_queries
    and object_query_embed under a fixed projection of the decoder states.  Also the sorted parameter names of the
    reference class built from the flagship configs' own transformer dicts (keys_tiny, keys_base)."""
    w = syn.WORKLOADS[workload]
    mmcv_stub.load_reference_decoder()
    PT = mmcv_stub.load_reference_transformer()
    m = PT(num_feature_levels=len(w.levels), num_cams=w.num_cams, encoder=syn.encoder_cfg(w),
           decoder=copy.deepcopy(syn.DECODER_CFG), embed_dims=w.embed_dims,
           rotate_center=[w.bev_h // 2, w.bev_w // 2]).eval()
    m.load_state_dict(syn.make_random_state_dict(m, seed))
    inp, oq, reg = v2_inputs(w, seed)
    inp.bev_queries.requires_grad_(True)
    oq.requires_grad_(True)
    bev, states, ref0, refs = m(inp.mlvl_feats, inp.bev_queries, oq, w.bev_h, w.bev_w,
                                grid_length=list(grid_length_of(w)), bev_pos=inp.bev_pos, reg_branches=reg,
                                cls_branches=None, prev_bev=inp.prev_bev.clone(), img_metas=inp.img_metas)
    (states * fixed_projection(states.shape)).sum().backward()
    rq = row_subset(w.num_query, keep_rows)
    cfg_keys = {}
    for size in ("tiny", "base"):             # the flagship configs' own transformer dicts, unchanged
        path = os.path.join(mmcv_stub.REFERENCE_ROOT, "projects", "configs", "bevformer", f"bevformer_{size}.py")
        tcfg = config.load_config(path)["model"]["pts_bbox_head"]["transformer"]
        tcfg = {k: v for k, v in copy.deepcopy(tcfg).items() if k != "type"}
        cfg_keys[f"keys_{size}"] = np.array(sorted(PT(**tcfg).state_dict()))
    save_capped(os.path.join(OUT, f"perception_forward_{name}.npz"), bev=bev.detach().numpy(),
                states=states.detach().numpy(), ref0=ref0.detach().numpy(), refs=refs.detach().numpy(),
                keys=np.array(sorted(m.state_dict())), rows_q=rq, **cfg_keys,
                grad_query_rows=inp.bev_queries.grad[rq].numpy(), grad_query_stats=stats(inp.bev_queries.grad),
                grad_oq=oq.grad.numpy(), grad_oq_stats=stats(oq.grad))
    print(f"perception_forward_{name}: bev {tuple(bev.shape)} states {tuple(states.shape)}")


if __name__ == "__main__":
    if not mmcv_stub.reference_available():
        raise SystemExit("needs a reference checkout (set BEVF_REFERENCE_ROOT)")
    perception_forward_case("toy", "toy")
