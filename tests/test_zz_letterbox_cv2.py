"""The reference's own known-answer test for the letterbox (test/test_models_transform.py:40-73): YOLOTransform
must agree with the upstream OpenCV `letterbox` (yolort/v5/utils/augmentations.py:99-137) to atol 1e-2 on the same
five shapes x {auto, fixed} x {stride 32, 64}.  CPU: the oracle; GPU: the kernel."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate as R

cv2 = pytest.importorskip("cv2")

SHAPES = [(500, 500), (500, 1080), (720, 900), (1000, 950), (900, 720)]


def upstream_letterbox(im: np.ndarray, new_shape=(640, 640), auto=True, stride=32, color=(114, 114, 114)):
    """Restatement of augmentations.py:99-137 (scaleup=True, scale_fill=False): ratio, rounded unpadded size,
    padding modulo stride when `auto`, INTER_LINEAR resize, centred constant border."""
    h, w = im.shape[:2]
    r = min(new_shape[0] / h, new_shape[1] / w)
    unpad_w, unpad_h = int(round(w * r)), int(round(h * r))
    dw, dh = new_shape[1] - unpad_w, new_shape[0] - unpad_h
    if auto:
        dw, dh = dw % stride, dh % stride
    dw, dh = dw / 2, dh / 2
    if (w, h) != (unpad_w, unpad_h):
        im = cv2.resize(im, (unpad_w, unpad_h), interpolation=cv2.INTER_LINEAR)
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=color)


def _case(im_shape, seed):
    g = torch.Generator().manual_seed(seed)
    im = torch.randint(0, 255, (3, *im_shape), generator=g)          # the reference test's value range
    return im.to(torch.uint8), im.permute(1, 2, 0).numpy().astype("uint8")


def _want(im_numpy, auto, stride):
    out = upstream_letterbox(im_numpy, (640, 640), auto, stride).astype(np.float32)
    return np.transpose(out / 255.0, [2, 0, 1])


@pytest.mark.parametrize("im_shape", SHAPES[:3])
@pytest.mark.parametrize("auto", [True, False])
def test_restatement_equals_upstream_letterbox(im_shape, auto, golden_dir):
    """Bit-exact against the upstream letterbox: tests/golden/letterbox_upstream.json holds the SHA-256 of its output
    for each case (recorded from yolort.v5.letterbox on the same seeded inputs)."""
    with open(os.path.join(golden_dir, "letterbox_upstream.json")) as f:
        want = json.load(f)["cases"][f"{im_shape[0]}x{im_shape[1]}_auto{int(auto)}"]
    _, im_numpy = _case(im_shape, 1)
    got = upstream_letterbox(im_numpy, (640, 640), auto, 32)
    assert list(got.shape) == want["shape"] and str(got.dtype) == want["dtype"]
    assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == want["sha256"]


@pytest.mark.parametrize("im_shape", SHAPES)
@pytest.mark.parametrize("auto", [True, False])
@pytest.mark.parametrize("stride", [32, 64])
def test_oracle_letterbox_vs_opencv(im_shape, auto, stride):
    im_u8, im_numpy = _case(im_shape, 7)
    batch, _, _ = R.letterbox([im_u8], 640.0, 640.0, stride, None if auto else (640, 640))
    got, want = batch[0].numpy(), _want(im_numpy, auto, stride)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("im_shape", SHAPES)
@pytest.mark.parametrize("auto", [True, False])
@pytest.mark.parametrize("stride", [32, 64])
def test_gpu_letterbox_vs_opencv(im_shape, auto, stride):
    from yolort_b200.models.transform import YOLOTransform

    im_u8, im_numpy = _case(im_shape, 7)
    tr = YOLOTransform(640, 640, size_divisible=stride, fixed_shape=None if auto else (640, 640))
    nt, _ = tr([im_u8.to("cuda:0")])
    got, want = nt.tensors[0].cpu().numpy(), _want(im_numpy, auto, stride)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-2)
