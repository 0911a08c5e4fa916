"""Parity at the REAL shapes of BASELINE.json's configs (H100), at north_star's tolerance.

* stage-wise: every launch of the plan at the benchmark's own shape against a plain fp32 PyTorch op on the launch's
  own fp16/bf16 input (tests/stagewise.py): |err| <= 2^-9 (fp16) / 2^-6 (bf16) x (1 + |ref|), zero violations;
* end to end against the CPU oracle (oracle/restate.py, pinned to the reference by tests/golden): class indices exact
  and boxes within 1e-3 x canvas side on the matched detections (parity_util.assert_e2e_parity).

configs[1] yolov5s batch 32 640x640 fp16 (the bench's weights), configs[2] yolov5m 640x640 bf16, configs[3] yolov5l
mixed 416-1280 sizes incl. the 639-trap sizes 800 / 950 / 523, configs[4] yolov5x 1280x1280 fp16.
"""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from stagewise import check_plan_stagewise
from yolort_b200.models import yolov5l, yolov5m, yolov5s, yolov5x

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bench_model():
    import bench

    m = yolov5s(score_thresh=bench.SCORE_THRESH).eval()
    sd = bench.make_state_dict(m)
    m.load_state_dict(sd)
    return m.to(DEV), sd, bench


def _zoo(ctor, name, gain, dtype=None, **kw):
    """Model + weights of bench.py's configs c3-c5 (He gain < 2, the bench's head load knob)."""
    import bench

    m = ctor(**kw).eval()
    sd = bench.zoo_state_dict(m, gain)
    m.load_state_dict(sd)
    m = m.to(DEV)
    return (m.to(dtype) if dtype is not None else m), sd


def _calibrated_thresh(sd, im, size, target=1200):
    """Score threshold that lets ~`target` candidates of image `im` through (midway between two neighbouring oracle
    scores, so that the threshold itself sits in a gap): a realistic NMS load -- detections below the 300 cap, no
    top-k lottery among near-tied scores -- whatever the logit spread of the random weights is."""
    batch, _, _ = R.letterbox([im], float(size[0]), float(size[1]))
    net = R.Net(sd)
    with torch.no_grad():
        heads = net.head(net.backbone(batch))
    _, scores = R.decode(heads)
    s = np.sort(scores[0].numpy().ravel())[::-1]
    return float((s[target - 1] + s[target]) / 2)


def _stagewise(m, x_u8_list, n, h, w):
    """Run the plan at (n, h, w) with every activation kept and check each launch on its own input."""
    plan = m.model.get_plan(n, h, w, keep_intermediates=True)
    geoms, (Hb, Wb) = m.transform.geometry(x_u8_list)
    assert (Hb, Wb) == (h, w)
    m.transform.letterbox_into(x_u8_list, geoms, Hb, Wb, plan.input, 1)
    torch.cuda.synchronize()
    res = check_plan_stagewise(plan, m.model.backbone.body["0"])
    assert len(res) == len(plan._low.L.ops)
    bad = [r for r in res if r.violations]
    assert not bad, bad[:5]
    m.model.engine()._plans.clear()      # free the un-shared arena


def test_c2_yolov5s_bs32_640_fp16_every_launch_at_bench_shape():
    m, sd, bench = _bench_model()
    ims = [im.to(DEV) for im in bench.make_images(32, 1234)]
    _stagewise(m, ims, 32, 640, 640)


def test_c2_yolov5s_bs32_640_fp16_detections_vs_oracle():
    """The bench's model, weights and images: all 32 images on the GPU in one batch, the first 8 through the CPU oracle
    (every image has the 640x640 canvas, so the oracle's batch composition does not matter)."""
    m, sd, bench = _bench_model()
    ims = bench.make_images(32, 1234)
    out = m([im.to(DEV) for im in ims])
    ref = R.detect(sd, ims[:8], score_thresh=bench.SCORE_THRESH)
    util.assert_e2e_parity("c2 yolov5s bs32 640 fp16", out[:8], ref, 640.0, min_matched=0.99, min_within=0.999,
                           max_box_rel=1e-3, max_score_err=5e-3)


def test_c3_yolov5m_bs16_640_bf16_every_launch():
    m, sd = _zoo(yolov5m, "m", 1.4, dtype=torch.bfloat16)
    ims = [util.synth_image_u8(640, 640, 300 + i).to(DEV) for i in range(16)]
    _stagewise(m, ims, 16, 640, 640)


def test_c3_yolov5m_640_bf16_detections_vs_oracle():
    m, sd = _zoo(yolov5m, "m", 1.4, dtype=torch.bfloat16)
    ims = [util.synth_image_u8(640, 640, 300 + i) for i in range(4)]
    thr = _calibrated_thresh(sd, ims[0], (640, 640))
    m.model.post_process.score_thresh = thr
    out = m([im.to(DEV) for im in ims])
    ref = R.detect(sd, ims, score_thresh=thr)
    # bf16 activations (8-bit mantissa) through ~80 layers against an fp32 reference: the stated tolerance is looser
    # (logit errors of ~1e-2 move scores across the threshold and boxes by up to a few pixels)
    util.assert_e2e_parity("c3 yolov5m 640 bf16", out, ref, 640.0, min_matched=0.50, min_within=0.50,
                           max_box_rel=2e-2, max_score_err=5e-2, iou_thr=0.8)


def test_c3_yolov5m_640_fp16_detections_vs_oracle():
    m, sd = _zoo(yolov5m, "m", 1.4)
    ims = [util.synth_image_u8(640, 640, 300 + i) for i in range(4)]
    thr = _calibrated_thresh(sd, ims[0], (640, 640))
    m.model.post_process.score_thresh = thr
    out = m([im.to(DEV) for im in ims])
    ref = R.detect(sd, ims, score_thresh=thr)
    util.assert_e2e_parity("c3 yolov5m 640 fp16", out, ref, 640.0, min_matched=0.97, min_within=0.99,
                           max_box_rel=1e-3, max_score_err=5e-3)


_C4_SIZES = [(800, 600), (950, 523), (523, 950), (416, 416), (1280, 720), (720, 1280), (1000, 1000), (639, 481)]


def test_c4_yolov5l_mixed_416_1280_detections_vs_oracle():
    """Dynamic-shape batch: sizes drawn from 416..1280 including 800 / 950 / 523 (long side letterboxes to 639, not 640:
    SURVEY.md 0.7); canvas = batch maximum rounded up to 32; boxes come back in each image's own pixel frame."""
    m, sd = _zoo(yolov5l, "l", 1.4)
    ims = [util.synth_image_u8(h, w, 700 + i) for i, (h, w) in enumerate(_C4_SIZES)]
    thr = _calibrated_thresh(sd, ims[3], (640, 640))
    m.model.post_process.score_thresh = thr
    out = m([im.to(DEV) for im in ims])
    ref = R.detect(sd, ims, score_thresh=thr)
    side = float(max(max(s) for s in _C4_SIZES))      # boxes are in original-image pixels
    util.assert_e2e_parity("c4 yolov5l mixed 416-1280 fp16", out, ref, side, min_matched=0.97, min_within=0.99,
                           max_box_rel=1e-3, max_score_err=5e-3)


def test_c4_yolov5l_mixed_batch_every_launch():
    m, sd = _zoo(yolov5l, "l", 1.4)
    ims = [util.synth_image_u8(h, w, 700 + i).to(DEV) for i, (h, w) in enumerate(_C4_SIZES)]
    geoms, (Hb, Wb) = m.transform.geometry(ims)
    _stagewise(m, ims, len(ims), Hb, Wb)


def test_c5_yolov5x_1280_fp16_every_launch():
    m, sd = _zoo(yolov5x, "x", 1.3, size=(1280, 1280))
    ims = [util.synth_image_u8(1280, 1280, 900 + i).to(DEV) for i in range(2)]
    _stagewise(m, ims, 2, 1280, 1280)


def test_c5_yolov5x_1280_fp16_detections_vs_oracle():
    """One 1280x1280 image through the fp32 CPU oracle (0.82 TFLOP) and the GPU path."""
    m, sd = _zoo(yolov5x, "x", 1.3, size=(1280, 1280))
    ims = [util.synth_image_u8(1280, 1280, 900)]
    thr = _calibrated_thresh(sd, ims[0], (1280, 1280))
    m.model.post_process.score_thresh = thr
    out = m([im.to(DEV) for im in ims])
    ref = R.detect(sd, ims, score_thresh=thr, size=(1280, 1280))
    util.assert_e2e_parity("c5 yolov5x 1280 fp16", out, ref, 1280.0, min_matched=0.97, min_within=0.99,
                           max_box_rel=1e-3, max_score_err=5e-3)
