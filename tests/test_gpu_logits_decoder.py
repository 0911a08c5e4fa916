"""LogitsDecoder / dense decode (SURVEY.md section 8f row 3) vs the oracle's restatement of
box_head.py:328-360 (H100)."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200.models import yolov5n
from yolort_b200.models.anchor_utils import AnchorGenerator
from yolort_b200.relay import LogitsDecoder

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("levels,nc,dtype", [(3, 80, torch.float32), (4, 80, torch.float16), (3, 3, torch.float32),
                                             (3, 91, torch.bfloat16)])
def test_dense_decode_vs_oracle(levels, nc, dtype):
    strides = util.P6_STRIDES[:levels] if levels == 4 else [8, 16, 32]
    anchors = util.P6_ANCHORS if levels == 4 else R.DEFAULT_ANCHORS
    g = torch.Generator().manual_seed(levels * 100 + nc)
    H, W = 128, 192
    heads = [(torch.randn(2, 3, H // s, W // s, nc + 5, generator=g) * 2.0).to(dtype) for s in strides]
    want_b, want_s = R.decode([h.float() for h in heads], strides, anchors)
    ag = AnchorGenerator(strides, anchors)
    grids, shifts = ag([torch.zeros(1, 1, H // s, W // s) for s in strides])
    dec = LogitsDecoder(strides)          # anchors from reference-style shifts (logits_decoder.py:26-31 signature)
    boxes, scores = dec([h.to(DEV) for h in heads], grids, shifts)
    assert tuple(boxes.shape) == tuple(want_b.shape) and tuple(scores.shape) == tuple(want_s.shape)
    assert boxes.dtype == torch.float32 and scores.dtype == torch.float32
    np.testing.assert_allclose(scores.cpu().numpy(), want_s.numpy(), rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(boxes.cpu().numpy(), want_b.numpy(), rtol=2e-6, atol=2e-4)


def test_model_with_logits_decoder_post_process():
    """relay/trt_inference.py:43: YOLO(..., post_process=LogitsDecoder(strides)) returns dense (boxes, scores);
    thresholding + NMS of those on the CPU reproduces the model's own detections."""
    sd = util.synth_state_dict(util.layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0)
    m = yolov5n(size=(128, 128), score_thresh=0.15).eval()
    m.load_state_dict(sd)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, 96, 128, generator=g).to(DEV)
    dets = m.model(x)
    m.model.post_process = LogitsDecoder([8, 16, 32])
    boxes, scores = m.model(x)
    n_anchors = 3 * (12 * 16 + 6 * 8 + 3 * 4)
    assert tuple(boxes.shape) == (2, n_anchors, 4) and tuple(scores.shape) == (2, n_anchors, 80)
    b, s = boxes.cpu().numpy(), scores.cpu().numpy()
    for i in range(2):
        inds, labels = np.nonzero(s[i] > np.float32(0.15))
        cb, cs = b[i][inds], s[i][inds, labels]
        keep = R.batched_nms(cb, cs, labels, 0.45)[:300]
        got = util.to_np(dets[i])
        util.assert_dets_close(got, {"scores": cs[keep], "labels": labels[keep].astype(np.int64), "boxes": cb[keep]},
                               box_atol=1e-4, score_atol=1e-6, allow_tie_swaps=True)
