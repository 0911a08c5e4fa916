"""YOLOv5's augmentations (yolort_b200.v5.utils.augmentations) on the CPU: the numpy restatement of the kernel
(oracle/restate_v5aug.py) against the reference's cv2 outputs recorded in tests/golden/v5aug.npz, the host draws and
box arithmetic against the same fixtures, and the input errors.  Where cv2 imports, the restatement is also compared
with it directly."""
import hashlib
import math
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5aug_cases as VC  # noqa: E402
from oracle import restate_v5aug as R  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.v5.utils import augmentations as A  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "v5aug.npz"))
NAMES = [c["name"] for c in VC.CASES]


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case(name):
    return next(c for c in VC.CASES if c["name"] == name)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_reference(name):
    c = case(name)
    im, _, extra = VC.inputs(c)
    plan, lab, r = VC.plan_case(c, im.shape)
    if c["fn"] == "mixup":
        out = R.mixup_pixels(im, extra[0], r)
    else:
        out = im if plan is None else VC.restate(plan, im)
    assert tuple(out.shape) == tuple(GOLD[f"{name}/shape"])
    if f"{name}/out" in GOLD:
        np.testing.assert_array_equal(out, GOLD[f"{name}/out"])
    assert sha(out) == str(GOLD[f"{name}/sha256"])
    np.testing.assert_array_equal(np.asarray(lab), GOLD[f"{name}/labels"])


@pytest.mark.parametrize("name", NAMES)
def test_draws_equal_reference(name):
    c = case(name)
    im, _, _ = VC.inputs(c)
    with VC.DrawLog() as log:
        VC.plan_case(c, im.shape)
    np.testing.assert_array_equal(np.array(log.values, np.float64), GOLD[f"{name}/draws"])
    assert log.kinds == [str(k) for k in GOLD[f"{name}/kinds"]]
    np.testing.assert_array_equal([random.random(), np.random.random()], GOLD[f"{name}/after"])


def test_zero_gains_draw_nothing():
    np.random.seed(0)
    state = np.random.get_state()[1].copy()
    assert A._hsv_draw(0, 0, 0) is None
    np.testing.assert_array_equal(np.random.get_state()[1], state)


def test_colour_tables_equal_reference():
    """The restated conversions over every input equal cv2's, in both channel orders; HSV->BGR on rows of 256 (its
    vector path) and of 1 pixel (its scalar path)."""
    bgr = R.all_bgr_image()
    for rgb in (False, True):
        tag = "rgb" if rgb else "bgr"
        hsv = R.to_hsv(bgr, rgb)
        assert sha(hsv) == str(GOLD[f"tables/to_hsv_{tag}"])
        assert sha(R.from_hsv(hsv, rgb)) == str(GOLD[f"tables/round_trip_{tag}"])
        for w in (256, 1):
            assert sha(R.from_hsv(R.all_hsv_image(w), rgb)) == str(GOLD[f"tables/from_hsv_{tag}_w{w}"])


def _random_map(rng, h, w, perspective):
    C = np.eye(3)
    C[0, 2], C[1, 2] = -w / 2, -h / 2
    P = np.eye(3)
    if perspective:
        P[2, 0], P[2, 1] = rng.uniform(-1e-3, 1e-3, 2)
    Rm = np.eye(3)
    Rm[:2] = A._rotation_matrix_2d(rng.uniform(-45, 45), rng.uniform(0.5, 1.5))
    S = np.eye(3)
    S[0, 1], S[1, 0] = (math.tan(v * math.pi / 180) for v in rng.uniform(-10, 10, 2))
    T = np.eye(3)
    T[0, 2], T[1, 2] = rng.uniform(0.4, 0.6) * w, rng.uniform(0.4, 0.6) * h
    return T @ S @ Rm @ P @ C


def test_restatement_equals_cv2_warps():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2024)
    for k in range(200):
        h, w = (int(v) for v in rng.integers(1, 90, 2))
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        perspective = k % 2 == 1
        M = _random_map(rng, h, w, perspective)
        oh, ow = max(1, h + int(rng.integers(-4, 40))), max(1, w + int(rng.integers(-4, 40)))
        if perspective:
            ref = cv2.warpPerspective(src, M, dsize=(ow, oh), borderValue=(114, 114, 114))
            out = R.warp(src, R.invert_perspective(M), oh, ow, True)
        else:
            ref = cv2.warpAffine(src, M[:2], dsize=(ow, oh), borderValue=(114, 114, 114))
            out = R.warp(src, R.invert_affine(M[:2]), oh, ow, False)
        np.testing.assert_array_equal(out, ref, err_msg=f"case {k}: {h}x{w} -> {oh}x{ow}, perspective {perspective}")


def test_rotation_matrix_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for a, s in zip(rng.uniform(-180, 180, 500), rng.uniform(0.1, 2, 500)):
        np.testing.assert_array_equal(A._rotation_matrix_2d(a, s), cv2.getRotationMatrix2D(angle=a, center=(0, 0),
                                                                                            scale=s))


def test_host_inverses_equal_restatement():
    rng = np.random.default_rng(9)
    for k in range(50):
        M = _random_map(rng, 480, 640, k % 2 == 1)
        np.testing.assert_array_equal(A._invert_affine(M), R.invert_affine(M[:2]))
        np.testing.assert_array_equal(A._invert_perspective(M), R.invert_perspective(M))


def test_box_candidates_is_the_reference_expression():
    rng = np.random.default_rng(3)
    b1 = rng.uniform(0, 100, (4, 50))
    b2 = rng.uniform(0, 100, (4, 50))
    w1, h1, w2, h2 = b1[2] - b1[0], b1[3] - b1[1], b2[2] - b2[0], b2[3] - b2[1]
    ar = np.maximum(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16))
    want = (w2 > 2) & (h2 > 2) & (w2 * h2 / (w1 * h1 + 1e-16) > 0.1) & (ar < 20)
    np.testing.assert_array_equal(A.box_candidates(b1, b2), want)


def test_input_errors():
    im = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(TypeError):
        A.augment_hsv(im)
    with pytest.raises(TypeError):
        A.cutout(im, np.zeros((0, 5)))
    try:
        from PIL import Image
    except ImportError:
        Image = None
    if Image is not None:
        with pytest.raises(TypeError):
            A.random_perspective(Image.fromarray(im))
    with pytest.raises(ValueError):
        A.augment_hsv(torch.zeros((8, 8, 3), dtype=torch.float32))
    with pytest.raises(ValueError):
        A.augment_hsv(torch.zeros((3, 8, 8, 1), dtype=torch.uint8))
    with pytest.raises(ValueError):
        A.random_perspective(torch.zeros((3, 8, 8), dtype=torch.uint8))
    with pytest.raises(_C.NativeLibraryError):
        A.augment_hsv(torch.zeros((8, 8, 3), dtype=torch.uint8))
    with pytest.raises(_C.NativeLibraryError):
        A.apply_batch([torch.zeros((8, 8, 3), dtype=torch.uint8)])
    with pytest.raises(NotImplementedError):
        A.random_perspective(torch.zeros((8, 8, 3), dtype=torch.uint8), segments=[np.ones((3, 2))])
    with pytest.raises(ValueError):
        A.apply_batch([torch.zeros((8, 8, 3), dtype=torch.uint8)], channel_order="hsv")


def test_apply_batch_draw_order_and_flips():
    """plan_batch draws random_perspective, augment_hsv, flipud, fliplr per image, in turn; flips mirror pixel
    xyxy boxes."""
    hyp = dict(A.HYP_SCRATCH, flipud=0.5, degrees=5.0, shear=2.0)
    sizes = [(48, 64), (33, 50), (40, 40)]
    labs = [VC.labels(k, h, w, 3) for k, (h, w) in enumerate(sizes)]
    random.seed(7)
    np.random.seed(7)
    plans, out = A.plan_batch(sizes, [lab.copy() for lab in labs], hyp)
    random.seed(7)
    np.random.seed(7)
    for (h, w), lab, plan, got in zip(sizes, labs, plans, out):
        M, s, height, width = A._perspective_draw((h, w), hyp["degrees"], hyp["translate"], hyp["scale"],
                                                  hyp["shear"], hyp["perspective"], (0, 0))
        want = A._warp_targets(lab.copy(), M, s, width, height, 0.0)
        np.testing.assert_array_equal(plan.lut, A._hsv_draw(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]))
        ud, lr = random.random() < hyp["flipud"], random.random() < hyp["fliplr"]
        assert (plan.flip_ud, plan.flip_lr) == (ud, lr)
        if ud:
            want[:, [2, 4]] = height - want[:, [4, 2]]
        if lr:
            want[:, [1, 3]] = width - want[:, [3, 1]]
        np.testing.assert_array_equal(got, want)
    assert any(p.flip_lr for p in plans) or any(p.flip_ud for p in plans)
