"""bevf_nms_free_decode against torch.sigmoid on the device and the float64 restatement of NMSFreeCoder.decode
(tests/head_oracle.py): selection, order and tie rule, labels, boxes, score-threshold branches, centre filter,
compaction and zero-fill."""
import numpy as np
import pytest
import torch

from bevformer_b200 import ops
from bevformer_b200.plugin import NMSFreeCoder
from tests import head_oracle as ho

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PCR = [-61.2, -61.2, -10.0, 61.2, 61.2, 10.0]


def _inputs(bs, nq, ncls, seed, logit_scale=3.0, box_scale=40.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    cls = (logit_scale * torch.randn(bs, nq, ncls, generator=g) - 2.0).to(DEV, dtype)
    box = torch.randn(bs, nq, 10, generator=g)
    box[..., (0, 1)] *= box_scale                       # some centres fall outside post_center_range
    box[..., 4] *= 6.0
    return cls, box.to(DEV, dtype)


def _ulps(a, b):
    a = a.float().contiguous().view(torch.int32).long()
    b = b.float().contiguous().view(torch.int32).long()
    return (a - b).abs()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("bs,nq,ncls,k", [(1, 900, 10, 300), (2, 77, 10, 100), (2, 30, 10, 300), (1, 50, 7, 1)])
def test_topk_scores_labels_and_boxes(dtype, bs, nq, ncls, k):
    cls, box = _inputs(bs, nq, ncls, seed=nq + k)
    cls = cls.to(dtype)
    big = [-1e4] * 3 + [1e4] * 3                           # no centre filter: every candidate is kept
    bboxes, scores, labels, num = ops.nms_free_decode(cls, box, k, big)
    torch.cuda.synchronize()
    dev_scores = torch.sigmoid(cls.float()).reshape(bs, -1)   # torch.sigmoid of the same logits on the device
    want = ho.decode_fp64(cls.float(), box.float(), k, big)
    for i in range(bs):
        assert num[i].item() == k
        w = want[i]
        # the scores are non-increasing; order and labels are those of the device's own scores under the rule
        # (score descending, flat index ascending)
        s = scores[i]
        assert (s[1:] <= s[:-1]).all()
        kth = w["scores"][-1].item()
        ref_dev = ho.decode_fp64(cls.float(), box.float(), k, big, scores=dev_scores)[i]
        assert torch.equal(labels[i].cpu(), ref_dev["labels"]), "order / labels differ from the device scores' top-k"
        assert _ulps(s.cpu(), ref_dev["scores"].float()).max().item() <= 1
        assert torch.allclose(bboxes[i].double().cpu(), ref_dev["bboxes"], rtol=1e-6, atol=1e-6)
        # against the float64 top-k: the same set except elements within 1 ulp of the k-th score
        near = 2 * np.spacing(np.float32(kth))
        a = set(ref_dev["index"].tolist())
        b = set(w["index"].tolist())
        sd = torch.sigmoid(cls[i].double().cpu().reshape(-1))
        for j in a ^ b:
            assert abs(sd[j].item() - kth) <= near, j


def test_exact_ties_come_in_ascending_index_order():
    nq, ncls, k = 200, 10, 300
    cls = torch.full((1, nq, ncls), -1.0)
    cls[0, ::3, ::2] = 0.5                              # hundreds of exactly equal scores
    cls[0, 7, 3] = 2.0
    cls = cls.to(DEV)
    box = torch.zeros(1, nq, 10, device=DEV)
    box[..., 7] = 1.0
    box[0, :, 8] = torch.arange(nq, device=DEV, dtype=torch.float32)     # vx = query index: the flat index is recoverable
    bboxes, scores, labels, num = ops.nms_free_decode(cls, box, k, PCR)
    torch.cuda.synchronize()
    flat = torch.arange(nq * ncls).reshape(nq, ncls)
    tied = flat[::3, ::2].reshape(-1).sort().values
    want = torch.cat([flat[7, 3:4], tied, flat.reshape(-1)[~torch.isin(flat.reshape(-1), tied) &
                                                             (flat.reshape(-1) != 73)]])[:k]
    assert num.item() == k
    got = bboxes[0, :, 7].cpu().long() * ncls + labels[0].cpu()
    assert torch.equal(got, want)
    s = scores[0].cpu()
    assert (s[1:] <= s[:-1]).all()


def test_max_num_at_the_edge_sorts_everything():
    cls, box = _inputs(2, 12, 10, seed=11)
    k = 120
    bboxes, scores, labels, num = ops.nms_free_decode(cls, box, k, [-1e4] * 3 + [1e4] * 3)
    torch.cuda.synchronize()
    ref = ho.decode_fp64(cls, box, k, [-1e4] * 3 + [1e4] * 3, scores=torch.sigmoid(cls).reshape(2, -1))
    for i in range(2):
        assert num[i].item() == k and torch.equal(labels[i].cpu(), ref[i]["labels"])
    with pytest.raises(RuntimeError, match="max_num"):
        ops.nms_free_decode(cls, box, k + 1, PCR)


@pytest.mark.parametrize("thr", [None, 0.0, 0.3, 0.97, 0.999, -0.5])
@pytest.mark.parametrize("z_shift", [False, True])
def test_threshold_branches_and_centre_filter(thr, z_shift):
    """Sample 0: 0.3 passes at once, 0.97 and 0.999 need the decay loop (top score ~0.85), 0.0 runs the loop but
    applies no mask, -0.5 passes everything.  Sample 1: every score is below 0.01, so any positive threshold falls
    through to "> -1" and the kept set is every candidate with its centre in range."""
    cls, box = _inputs(2, 400, 10, seed=5, logit_scale=1.0)
    cls[1] -= 10.0
    assert torch.sigmoid(cls[1]).max().item() < 0.01
    bboxes, scores, labels, num = ops.nms_free_decode(cls, box, 100, PCR, thr, z_shift)
    torch.cuda.synchronize()
    dev_scores = torch.sigmoid(cls).reshape(2, -1)
    want = ho.decode_fp64(cls, box, 100, PCR, thr, z_shift, scores=dev_scores)
    in_range = ho.decode_fp64(cls, box, 100, PCR, None, z_shift, scores=dev_scores)
    for i in range(2):
        n = num[i].item()
        assert n == len(want[i]["scores"])
        assert torch.equal(labels[i, :n].cpu(), want[i]["labels"])
        assert torch.allclose(bboxes[i, :n].double().cpu(), want[i]["bboxes"], rtol=1e-6, atol=1e-6)
        assert (bboxes[i, n:] == 0).all() and (scores[i, n:] == 0).all() and (labels[i, n:] == 0).all()
        if not z_shift:                                # the filter reads the centre before get_bboxes' shift
            c = bboxes[i, :n, :3].cpu()
            assert (c >= torch.tensor(PCR[:3])).all() and (c <= torch.tensor(PCR[3:])).all()
    if thr not in (None, 0.0):
        assert num[1].item() == len(in_range[1]["scores"]) < 100        # the fall-through branch on sample 1


@pytest.mark.parametrize("case", sorted(ho.NMS_CASES))
def test_against_the_reference_coder_golden(case):
    """The reference NMSFreeCoder's own fp32 decode of the same inputs (tests/golden/ref_nms_decode_<case>.npz)."""
    from tests.util import golden
    g = golden(f"ref_nms_decode_{case}")
    cls, box = ho.nms_case_inputs(case)
    bboxes, scores, labels, num = ops.nms_free_decode(cls.float().to(DEV), box.float().to(DEV), 100, PCR,
                                                      ho.NMS_CASES[case][0])
    torch.cuda.synchronize()
    assert num.cpu().tolist() == g["fp32_num"].tolist()
    cut = np.cumsum(g["fp32_num"])[:-1]
    for i, (wb, ws, wl) in enumerate(zip(np.split(g["fp32_bboxes"], cut), np.split(g["fp32_scores"], cut),
                                         np.split(g["fp32_labels"], cut))):
        n = num[i].item()
        np.testing.assert_array_equal(labels[i, :n].cpu().numpy(), wl)
        np.testing.assert_allclose(scores[i, :n].cpu().numpy(), ws, rtol=3e-7, atol=0)
        np.testing.assert_allclose(bboxes[i, :n].cpu().numpy(), wb, rtol=1e-6, atol=1e-6)


def test_subnormal_scores_rank_as_torch_sigmoid():
    """Logits below about -87.3 give subnormal sigmoids; they keep their order (not flushed to zero ties)."""
    cls = torch.linspace(-88.5, -87.4, 20, device=DEV).flip(0).reshape(1, 2, 10).contiguous()
    box = torch.zeros(1, 2, 10, device=DEV)
    box[..., 7] = 1.0
    bboxes, scores, labels, num = ops.nms_free_decode(cls, box, 20, PCR)
    torch.cuda.synchronize()
    want = torch.sigmoid(cls).reshape(-1)
    assert (want > 0).all() and (want < 1.2e-38).all()
    assert torch.equal(scores[0].view(torch.int32), want.view(torch.int32))
    assert torch.equal(labels[0].cpu(), torch.arange(20) % 10)


def test_coder_decode_returns_the_reference_list():
    cls, box = _inputs(2, 900, 10, seed=1)
    coder = NMSFreeCoder(pc_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], post_center_range=PCR, max_num=300,
                         num_classes=10)
    preds = dict(all_cls_scores=cls[None], all_bbox_preds=box[None])
    out = coder.decode(preds)
    want = ho.decode_fp64(cls, box, 300, PCR, scores=torch.sigmoid(cls).reshape(2, -1))
    assert len(out) == 2
    for o, w in zip(out, want):
        assert set(o) == {"bboxes", "scores", "labels"}
        assert torch.equal(o["labels"].cpu(), w["labels"]) and o["bboxes"].shape == (len(w["labels"]), 9)
    with pytest.raises(NotImplementedError):
        NMSFreeCoder(pc_range=[0] * 6, post_center_range=None).decode(preds)
