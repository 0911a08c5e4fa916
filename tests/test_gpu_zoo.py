"""The other model sizes of BASELINE.json's configs (m / l / x: channel widths 48..1280, deeper C3 stacks, bf16,
mixed input sizes, 1280-pixel canvas) against the CPU oracle (H100)."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200.models import yolov5l, yolov5m, yolov5x

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# He gain 2.0 (the n/s fixtures) makes the deeper residual chains of m/l/x blow up with random weights (oracle
# activations reach 1e5..1e7, past fp16 range). Two regimes instead:
#   "lively": activations grow to O(50) like the yolov5s fixtures -> raw head logits compared numerically
#             (detections are chaotic there: rounding the WEIGHTS to fp16 inside the fp32 oracle already moves them);
#   "stable": detections of the oracle survive fp16 weight rounding (match >= 0.99) -> detection parity.
_LIVELY = {"m": 1.7, "l": 1.7, "x": 1.5}
_STABLE = {"m": 1.4, "l": 1.4, "x": 1.3}


def _build(ctor, name, gain, dtype=None, **kw):
    sd = util.synth_state_dict(util.layouts()[name], knob_obj=7.0, knob_cls=4.5, seed=1, gain=gain)
    m = ctor(**kw).eval()
    m.load_state_dict(sd)
    m = m.to(DEV)
    return (m.to(dtype) if dtype is not None else m), sd


def _check_dets(m, sd, ims, min_frac, iou=0.9, **kw):
    ref = R.detect(sd, ims, **kw)
    out = m([im.to(DEV) for im in ims])
    for got, want, im in zip(out, ref, ims):
        frac = util.match_fraction(util.to_np(got), want, iou_thr=iou, side=max(im.shape[1:]))
        print(tuple(im.shape[1:]), "matched", round(frac, 3), len(got["scores"]), len(want["scores"]))
        assert len(want["scores"]) > 0
        assert frac >= min_frac


def _check_heads(m, sd, n, h, w, tol):
    """Raw head logits of one pre-letterboxed batch vs the fp32 oracle network."""
    g = torch.Generator().manual_seed(n * 1000 + h + w)
    x = torch.rand(n, 3, h, w, generator=g)
    m.model(x.to(DEV))
    plan = m.model.get_plan(n, h, w)
    m.model.run_plan(plan)
    torch.cuda.synchronize()
    net = R.Net(sd)
    with torch.no_grad():
        want = net.head(net.backbone(x.half().float()))
    for i, wnt in enumerate(want):
        hd = plan.heads[i][..., :255].float().cpu()
        got = hd.view(*hd.shape[:3], 3, 85).permute(0, 3, 1, 2, 4).numpy()      # -> [N, A, H, W, K] like the oracle
        ref = wnt.numpy()
        assert got.shape == ref.shape
        err = np.abs(got - ref)
        rr = float(np.sqrt((err ** 2).mean()) / np.sqrt((ref ** 2).mean()))
        print(f"head{i}: ref rms {np.sqrt((ref ** 2).mean()):.2f} max {np.abs(ref).max():.1f} rel_rms {rr:.2e}")
        assert np.isfinite(got).all()
        assert rr < tol


def test_yolov5m_heads_widths_48_to_768():
    m, sd = _build(yolov5m, "m", _LIVELY["m"], size=(160, 160), score_thresh=0.2)
    _check_heads(m, sd, 2, 160, 128, 2e-2)


def test_yolov5l_heads_deep_c3_stacks():
    m, sd = _build(yolov5l, "l", _LIVELY["l"], size=(192, 192), score_thresh=0.2)
    _check_heads(m, sd, 2, 192, 160, 2e-2)


def test_yolov5x_heads_widths_80_to_1280():
    m, sd = _build(yolov5x, "x", _LIVELY["x"], size=(128, 128), score_thresh=0.2)
    _check_heads(m, sd, 1, 128, 128, 2e-2)


def test_yolov5m_bf16_heads():
    m, sd = _build(yolov5m, "m", _LIVELY["m"], dtype=torch.bfloat16, size=(160, 160), score_thresh=0.2)
    _check_heads(m, sd, 1, 160, 160, 1.2e-1)     # 8-bit mantissa through ~60 layers


def test_yolov5m_detections():
    m, sd = _build(yolov5m, "m", _STABLE["m"], size=(160, 160), score_thresh=0.2)
    ims = [util.synth_image_u8(120, 160, 1), util.synth_image_u8(160, 96, 2)]
    # measured 0.95 / 0.99 with the packed-half2 epilogue on shortcut layers, 0.917 / 0.99 with the (more accurate) fp32
    # epilogue they run now: on this random-weight fixture the match count moves with ANY rounding change, in either direction
    _check_dets(m, sd, ims, 0.90, score_thresh=0.2, size=(160, 160))


def test_yolov5l_detections_mixed_sizes():
    m, sd = _build(yolov5l, "l", _STABLE["l"], size=(192, 192), score_thresh=0.2)
    ims = [util.synth_image_u8(h, w, 10 + i) for i, (h, w) in enumerate([(150, 192), (192, 100), (97, 131)])]
    _check_dets(m, sd, ims, 0.96, score_thresh=0.2, size=(192, 192))      # measured 0.98 .. 0.993


def test_yolov5x_detections():
    m, sd = _build(yolov5x, "x", _STABLE["x"], size=(128, 128), score_thresh=0.2)
    ims = [util.synth_image_u8(128, 128, 5)]
    _check_dets(m, sd, ims, 0.97, score_thresh=0.2, size=(128, 128))      # measured 1.0


def test_yolov5x_1280_canvas_runs():
    """BASELINE.json configs[4] shape (1280x1280, 100 800 anchors): plumbing + output contract (no oracle: the CPU
    path needs ~0.8 TFLOP per image)."""
    m, _ = _build(yolov5x, "x", _STABLE["x"], size=(1280, 1280), score_thresh=0.3)
    out = m([torch.randint(0, 256, (3, 1280, 1280), dtype=torch.uint8, device=DEV)])
    assert len(out) == 1 and out[0]["boxes"].shape[1] == 4 and out[0]["boxes"].shape[0] <= 300
