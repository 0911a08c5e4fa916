"""The stage-wise checker (tests/stagewise.py) covers every model family: each op of each family's lowering has a
reference and the stem reference takes each family's stem module.  Lowered on the CPU, so that a new op kind, element
type or stem module cannot slip past the GPU check unnoticed."""
import pytest
import torch

import stagewise as S
from yolort_b200 import _C
from yolort_b200.engine import _Buf, _Op, _View, lower_darknet, lower_fp8, lower_lite, lower_yolo
from yolort_b200.models import darknet as D
from yolort_b200.models import yolov5n, yolov5n6, yolov5s, yolov5ts
from yolort_b200.models.yolo_lite import yolov5_mobilenet_v3_small_fpn

F16, CPU = torch.float16, torch.device("cpu")


def _yolo(m):
    m = m.eval().model
    return lower_yolo(m, F16, CPU)[0], m.backbone.body["0"]


def _fp8(m):
    """lower_fp8 with a synthetic calibration: amax 1.0 for every buffer of the fp16 lowering."""
    m = m.eval().model
    amax = {b.name: 1.0 for b in lower_yolo(m, F16, CPU)[0].bufs}
    return lower_fp8(m, F16, CPU, amax)[0], m.backbone.body["0"]


def _lite():
    m = yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False).eval()
    return lower_lite(m, F16, CPU)[0], m.backbone.body["0"]


def _darknet(m):
    m = m.eval()
    return lower_darknet(m, F16, CPU)[0], m.features[0]


FAMILIES = {
    "yolov5n_r6.0": lambda: _yolo(yolov5n()),
    "yolov5s_r4.0": lambda: _yolo(yolov5s(upstream_version="r4.0")),
    "yolov5s_r3.1": lambda: _yolo(yolov5s(upstream_version="r3.1")),
    "yolov5n6": lambda: _yolo(yolov5n6()),
    "yolov5ts": lambda: _yolo(yolov5ts()),
    "lite": _lite,
    "darknet_s_r6.0": lambda: _darknet(D.darknet_s_r6_0()),
    "darknet_s_r4.0": lambda: _darknet(D.darknet_s_r4_0()),
    "yolov5s_r6.0_fp8": lambda: _fp8(yolov5s()),
}


@pytest.mark.parametrize("family", list(FAMILIES))
def test_every_op_and_stem_has_a_stagewise_reference(family):
    L, stem = FAMILIES[family]()
    for op in L.ops:
        S.reference_for(op)
    stem_op = next(op for op in L.ops if op.pack > 1)
    canvas = torch.rand(2, 12, 20, 16).to(F16)        # [N, H/2, W/2, 16] space-to-depth input
    with torch.no_grad():
        ref = S.stem_reference(stem, canvas, F16)
    assert ref.shape == (2, stem_op.dst.C, 12, 20)


def test_unknown_kinds_raise():
    v = _View(_Buf("x", 1, 16), 0, 16)
    with pytest.raises(KeyError, match="no stage-wise reference"):
        S.reference_for(_Op(kind=_C.YB_OP_AVGPOOL, src=v, dst=v, dtype=_C.YB_F8E4M3))
    with pytest.raises(ValueError, match="activation"):
        S.act_ref(torch.zeros(1), 99)
    with pytest.raises(NotImplementedError, match="stem"):
        S.stem_reference(torch.nn.Conv2d(3, 16, 3), torch.zeros(1, 4, 4, 16), F16)
