"""decode + threshold + batched NMS kernels vs reference fixtures and the C/numpy oracle (H100)."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200 import _C
from yolort_b200.models.box_head import PostProcess

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ANCH = R.DEFAULT_ANCHORS


@pytest.mark.parametrize("case", ["few", "trick", "vanilla", "empty"])
def test_postprocess_vs_reference_fixture(case):
    z = util.load_npz(f"postprocess_{case}.npz")
    heads = [torch.from_numpy(z[f"h{i}"]).to(DEV) for i in range(3)]
    pp = PostProcess([8, 16, 32], float(z["thr"]), 0.45, 300, anchors_px=[[float(v) for v in a] for a in ANCH])
    out = pp(heads)
    assert list(out[0].keys()) == ["scores", "labels", "boxes"]   # box_head.py:427 insertion order
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        got = util.to_np(got)
        assert got["labels"].dtype == np.int64 and got["boxes"].dtype == np.float32
        # expf on the GPU differs from the CPU's vectorised exp by <= 2 ulp: scores/boxes to 1e-6 relative,
        # labels and order exact except between candidates whose scores tie to that precision
        util.assert_dets_close(got, ref, box_atol=2e-4, score_atol=2e-6, allow_tie_swaps=True)
        exact = np.array_equal(got["labels"], ref["labels"])
        print(case, "n =", len(ref["scores"]), "order identical:", exact)


def _random_boxes(n, seed, ncls=5, tie=False):
    g = torch.Generator().manual_seed(seed)
    b = torch.rand(n, 4, generator=g) * 100
    b[:, 2:] += b[:, :2]
    s = torch.rand(n, generator=g)
    if tie:
        s[::7] = 0.5
    l = torch.randint(0, ncls, (n,), generator=g)
    return b, s, l


@pytest.mark.parametrize("n", [0, 1, 31, 300, 1000, 1001, 4096, 4097, 20000])
@pytest.mark.parametrize("sem", [R.TV_AUTO, R.EXACT_PER_CLASS, R.OFFSET_TRICK])
def test_batched_nms_bit_exact_vs_oracle(n, sem):
    b, s, l = _random_boxes(n, seed=n + 17)
    ref = R.batched_nms(b.numpy(), s.numpy(), l.numpy(), 0.45, sem)[:4096]
    got = _C.batched_nms(b.to(DEV), s.to(DEV), l.to(DEV), 0.45, sem, max_keep=4096).cpu().numpy()
    assert got.dtype == np.int64
    assert np.array_equal(got, ref), (len(got), len(ref), np.nonzero(got[:min(len(got), len(ref))] != ref[:min(len(got), len(ref))])[0][:5])


def test_batched_nms_ties_keep_index_order_and_topk_stop():
    b, s, l = _random_boxes(3000, seed=3, tie=True)
    ref = R.batched_nms(b.numpy(), s.numpy(), l.numpy(), 0.45, R.EXACT_PER_CLASS)
    got = _C.batched_nms(b.to(DEV), s.to(DEV), l.to(DEV), 0.45, R.EXACT_PER_CLASS, max_keep=300).cpu().numpy()
    assert np.array_equal(got, ref[:300])      # stable order: equal scores come back in index order


def test_nms_semantic_corner_cases():
    b = torch.tensor([[0, 0, 2, 1], [1, 0, 3, 1], [10, 10, 9, 9]], dtype=torch.float32)
    s = torch.tensor([0.9, 0.9, 0.1])
    l = torch.zeros(3, dtype=torch.int64)
    # IoU exactly 1/3: strict '>' keeps it; inverted box has positive area and no overlap -> kept
    assert _C.batched_nms(b.to(DEV), s.to(DEV), l.to(DEV), 1.0 / 3.0, R.EXACT_PER_CLASS).tolist() == [0, 1, 2]
    assert _C.batched_nms(b.to(DEV), s.to(DEV), l.to(DEV), 0.33, R.EXACT_PER_CLASS).tolist() == [0, 2]
    # different labels never suppress each other in either semantics
    l2 = torch.tensor([0, 1, 2])
    for sem in (R.EXACT_PER_CLASS, R.OFFSET_TRICK):
        assert _C.batched_nms(b.to(DEV), s.to(DEV), l2.to(DEV), 0.1, sem).tolist() == [0, 1, 2]


def test_candidate_arena_grows_instead_of_truncating():
    # ~86k candidates in one image (> the default 16 384 per-image share of the arena): must re-run, not truncate
    # (the oracle's per-class NMS is quadratic: a 16x larger version of this test took 50 s of CPU)
    g = torch.Generator().manual_seed(8)
    heads = [torch.randn(1, 3, 160 // s, 160 // s, 85, generator=g) * 1.5 + 1.0 for s in (8, 16, 32)]
    ref = R.postprocess(heads, 0.3, 0.45, 300)[0]
    assert ref["n_candidates"] > 30000
    out = PostProcess([8, 16, 32], 0.3, 0.45, 300, anchors_px=[[float(v) for v in a] for a in ANCH])(
        [h.to(DEV) for h in heads])[0]
    util.assert_dets_close(util.to_np(out), ref, box_atol=5e-4, score_atol=2e-6, allow_tie_swaps=True)


_ANCH4 = [[float(v) for v in a] for a in ANCH] + [[436.0, 615.0, 739.0, 380.0, 925.0, 792.0]]


@pytest.mark.parametrize("levels", [
    [(16, 24), (8, 12), (4, 6)],
    [(16, 24), (8, 12), (4, 6), (2, 3)],          # the P6 fixture's extents: 510 pixels, warps straddle level borders
    [(20, 20), (10, 10), (5, 5), (3, 3)],
])
@pytest.mark.parametrize("obj_shift", [-4.0, -1.0])   # ~2 % / ~25 % of the anchors pass objectness
def test_nhwc_row_decode_multi_level_vs_oracle(levels, obj_shift):
    """The plan's NHWC-256 head layout through the coalesced row kernel (lane-owns-pixel load, compacted class scan)
    + NMS against the oracle's decode + batched_nms on the same fp16 logits, for 3 and 4 detection levels."""
    g = torch.Generator().manual_seed(31 * len(levels) + levels[0][0] + int(obj_shift))
    n, a, nc = 2, 3, 80
    k = nc + 5
    strides = [8, 16, 32, 64][: len(levels)]
    anchors = _ANCH4[: len(levels)]
    nhwc, ref_heads = [], []
    for (h, w) in levels:
        t = torch.randn(n, h, w, a, k, generator=g) * 1.5
        t[..., 4] += obj_shift
        t[..., 5:] -= 1.0
        th = t.half()
        buf = torch.zeros(n, h, w, 256, dtype=torch.float16)
        buf[..., : a * k] = th.view(n, h, w, a * k)
        nhwc.append(buf.to(DEV))
        ref_heads.append(th.float().permute(0, 3, 1, 2, 4).contiguous())
    ref = R.postprocess(ref_heads, 0.25, 0.45, 300, R.TV_AUTO, strides, anchors)
    got = _C.decode_nms(nhwc, "nhwc", strides, anchors, 0.25, 0.45, 300, num_classes=nc)
    for gd, rd in zip(got, ref):
        print(levels, obj_shift, "candidates", rd["n_candidates"], "dets", len(rd["scores"]))
        util.assert_dets_close(util.to_np(gd), rd, box_atol=2e-4, score_atol=2e-6, allow_tie_swaps=True)
