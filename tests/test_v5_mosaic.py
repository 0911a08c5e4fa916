"""YOLOv5's mosaic training batches (yolort_b200.v5.utils.datasets) on the CPU: the numpy restatement of the resize and
compose kernels (oracle/restate_v5mosaic.py) against cv2 and against upstream's loader recorded in
tests/golden/v5mosaic.npz, the host planner's draws and generator states against the same fixture, and the input
errors."""
import hashlib
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5mosaic_cases as MC  # noqa: E402
from oracle import restate_v5mosaic as R  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.v5.utils import datasets as D  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "v5mosaic.npz"))
NAMES = [c["name"] for c in MC.CASES]


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case(name):
    return next(c for c in MC.CASES if c["name"] == name)


def test_resize_restatement_equals_cv2():
    """300 seeded (h0, w0, s) load_image triples, with 1-pixel sides, exact 2x and 4x scales and upscales."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(640)
    for k in range(300):
        h0, w0 = (int(v) for v in rng.integers(1, 300, 2))
        if k % 10 == 0:
            h0 = 1
        elif k % 10 == 1:
            w0 = 1
        s = int(rng.integers(2, 400))
        if k % 10 == 2:                                  # exact 2x: INTER_AREA inside cv2
            s, h0, w0 = 2 * s, 4 * s, 4 * s * 3 // 4 // 2 * 2
        elif k % 10 == 3:                                # exact 4x
            h0, w0 = 4 * s, 4 * max(1, s // 3)
        r = s / max(h0, w0)
        h, w = int(h0 * r), int(w0 * r)
        if r == 1 or h < 1 or w < 1:
            continue
        im = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
        want = cv2.resize(im, (w, h), interpolation=cv2.INTER_LINEAR)
        np.testing.assert_array_equal(R.load_image(im, s)[0], want, err_msg=f"{h0}x{w0} at s={s}")


def test_long_side_left_one_short():
    """int(L * (s / L)) is s - 1 for these long sides; letterbox then resizes a second time by s / (s - 1)."""
    assert [L for L in range(1, 700) if int(L * (640 / L)) != 640] == [77, 154, 303, 308, 319, 581, 606, 616, 623,
                                                                       638]
    assert D.load_shape(98, 40, 64) == (63, 26)
    (nh, nw), _, _, _, out = D.letterbox_geometry(63, 26, 64)
    assert (nh, nw) == (64, 26) and out == (64, 64)


@pytest.mark.parametrize("k", range(len(MC.SHAPES)))
def test_load_image_restatement_equals_reference(k):
    ims, _ = MC.dataset()
    im = R.load_image(ims[k], MC.S)[0]
    assert tuple(im.shape) == tuple(GOLD[f"load/{k}/shape"])
    assert sha(im) == str(GOLD[f"load/{k}/sha256"])
    assert D.load_shape(*ims[k].shape[:2], MC.S) == im.shape[:2]


@pytest.mark.parametrize("name", NAMES)
def test_batch_restatement_equals_reference(name):
    ims, labs = MC.dataset()
    c = case(name)
    samples, targets = MC.plan(c, ims, labs)
    imgs = MC.restate(samples, ims)
    assert tuple(imgs.shape) == tuple(GOLD[f"{name}/shape"])
    assert sha(imgs) == str(GOLD[f"{name}/sha256"])
    np.testing.assert_array_equal(targets, GOLD[f"{name}/targets"])


@pytest.mark.parametrize("name", NAMES)
def test_planner_draws_and_states_equal_reference(name):
    ims, labs = MC.dataset()
    c = case(name)
    with MC.DrawLog() as log:
        MC.plan(c, ims, labs)
    np.testing.assert_array_equal(np.array(log.values, np.float64), GOLD[f"{name}/draws"])
    assert log.kinds == [str(k) for k in GOLD[f"{name}/kinds"]]
    py, npst = MC.generator_states()
    np.testing.assert_array_equal(py, GOLD[f"{name}/py_state"])
    np.testing.assert_array_equal(npst, GOLD[f"{name}/np_state"])


def test_cases_cover_every_branch():
    ims, labs = MC.dataset()
    kinds = set()
    for c in MC.CASES:
        for smp in MC.plan(c, ims, labs)[0]:
            kinds.add("mosaic" if smp.mosaic else "letterbox")
            kinds.add("mixup" if smp.r is not None else "single")
            kinds |= {"flip_ud"} if smp.flip_ud else set()
            kinds |= {"flip_lr"} if smp.flip_lr else set()
            kinds |= {"perspective"} if smp.canvases[0].perspective else set()
            kinds |= {"chain"} if any(isinstance(p[0], tuple) for cv in smp.canvases for p in cv.places) else set()
            kinds |= {"no_hsv"} if smp.lut is None else set()
    assert kinds >= {"mosaic", "letterbox", "mixup", "single", "flip_ud", "flip_lr", "perspective", "chain", "no_hsv"}


def test_load_mosaic_restatement_equals_reference():
    ims, labs = MC.dataset()
    random.seed(9)
    np.random.seed(9)
    planner = D.Planner([im.shape[:2] for im in ims], labs, MC.S, MC.SCRATCH)
    cv, labels4 = planner.mosaic(5)
    smp = D.Sample(*cv.out)
    smp.canvases = [cv]
    img4 = R.sample_pixels(smp, ims, MC.S, rgb=True).transpose(1, 2, 0)
    assert sha(img4) == str(GOLD["load_mosaic/sha256"])
    np.testing.assert_array_equal(labels4, GOLD["load_mosaic/labels"])


def test_input_errors():
    ims, labs = MC.dataset()
    with pytest.raises(TypeError):
        D.train_batch(ims, labs, [0])
    with pytest.raises(TypeError):
        D.load_image(ims[0], 64)
    with pytest.raises(ValueError):
        D.train_batch([torch.zeros((8, 8, 3), dtype=torch.float32)], [None], [0])
    with pytest.raises(ValueError):
        D.load_mosaic([torch.zeros((3, 8, 8), dtype=torch.uint8)], [None], 0)
    with pytest.raises(_C.NativeLibraryError):
        D.train_batch([torch.zeros((8, 8, 3), dtype=torch.uint8)], [None], [0], img_size=64)
    cpu = [torch.zeros((8, 8, 3), dtype=torch.uint8)]
    with pytest.raises(ValueError):
        D.train_batch(cpu, [None], [0], channel_order="hsv")
    with pytest.raises(NotImplementedError):
        D.train_batch(cpu, [None], [0], segments=[[np.ones((3, 2))]])
    with pytest.raises(NotImplementedError):
        D.load_mosaic(cpu, [None], 0, segments=[[np.ones((3, 2))]])
