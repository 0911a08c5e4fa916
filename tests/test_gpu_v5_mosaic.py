"""YOLOv5's mosaic training batches on the GPU (csrc/v5_augment.cu's resize and compose launches) against the numpy
restatement (oracle/restate_v5mosaic.py) and upstream's loader recorded in tests/golden/v5mosaic.npz, bit for bit."""
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
from v5aug_cases import image  # noqa: E402
from yolort_b200.v5.utils import datasets as D  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "v5mosaic.npz"))
NAMES = [c["name"] for c in MC.CASES]


def sha(a) -> str:
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case(name):
    return next(c for c in MC.CASES if c["name"] == name)


def layout(im: np.ndarray, how: str) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(im)).to(DEV)
    if how == "hwc_view":                        # [H, W, 3] view of planar [3, H, W] memory
        return t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
    if how == "strided":                         # every other column of a wider image
        wide = torch.zeros((im.shape[0], 2 * im.shape[1], 3), dtype=torch.uint8, device=DEV)
        wide[:, ::2] = t
        return wide[:, ::2]
    return t


def run(c, ims, labs, how="contiguous", channel_order="bgr", s=MC.S):
    srcs = [layout(im[..., ::-1] if channel_order == "rgb" else im, how) for im in ims]
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    return D.train_batch(srcs, labs, c["indices"], img_size=s, hyp=MC.hyp(c), channel_order=channel_order)


@pytest.mark.parametrize("name", NAMES)
def test_train_batch_equals_restatement_and_reference(name):
    ims, labs = MC.dataset()
    c = case(name)
    imgs, targets = run(c, ims, labs)
    assert imgs.shape == (len(c["indices"]), 3, MC.S, MC.S) and imgs.device == torch.device(DEV)
    samples, want_targets = MC.plan(c, ims, labs)
    np.testing.assert_array_equal(imgs.cpu().numpy(), MC.restate(samples, ims))
    assert sha(imgs) == str(GOLD[f"{name}/sha256"])
    np.testing.assert_array_equal(targets.cpu().numpy(), GOLD[f"{name}/targets"])
    assert targets.dtype == torch.float32 and targets.device == torch.device(DEV)


@pytest.mark.parametrize("how", ["hwc_view", "strided"])
@pytest.mark.parametrize("channel_order", ["bgr", "rgb"])
def test_strided_sources_and_channel_orders(how, channel_order):
    """RGB sources through COLOR_RGB2HSV give the same RGB batch as their BGR originals."""
    ims, labs = MC.dataset()
    for name in ("warp_flips", "letterbox"):
        imgs, _ = run(case(name), ims, labs, how, channel_order)
        assert sha(imgs) == str(GOLD[f"{name}/sha256"])


def test_load_image_and_load_mosaic_equal_reference():
    ims, labs = MC.dataset()
    for k, im in enumerate(ims):
        out, hw0, hw = D.load_image(layout(im, "strided"), MC.S)
        assert hw0 == im.shape[:2] and hw == tuple(GOLD[f"load/{k}/shape"][:2])
        assert sha(out) == str(GOLD[f"load/{k}/sha256"])
    random.seed(9)
    np.random.seed(9)
    img4, labels4 = D.load_mosaic([layout(im, "hwc_view") for im in ims], labs, 5, img_size=MC.S, hyp=MC.SCRATCH)
    assert sha(img4) == str(GOLD["load_mosaic/sha256"])
    np.testing.assert_array_equal(labels4, GOLD["load_mosaic/labels"])


def big_dataset(s: int, n: int):
    """Seeded 480 x 640 images and mixed sizes around s: downscales, upscales, exact 2x, and int() leaving the long
    side at s - 1 (319 -> 639 at s = 640)."""
    shapes = [(480, 640), (640, 480), (1280, 960), (319, 200), (300, 500), (700, 1200), (s, s // 2), (90, 160)]
    ims, labs = [], []
    rng = np.random.default_rng(s)
    for k in range(n):
        h, w = shapes[k % len(shapes)] if k % 2 else (480, 640)
        ims.append(image(1000 + k, h, w))
        m = k % 5
        labs.append(np.concatenate([rng.integers(0, 80, (m, 1)), rng.uniform(0.2, 0.8, (m, 2)),
                                    rng.uniform(0.05, 0.5, (m, 2))], 1).astype(np.float32))
    return ims, labs


@pytest.mark.parametrize("s,batch,extra", [(640, 1, {}), (640, 32, {}), (640, 64, dict(mosaic=0.5, mixup=0.3)),
                                           (640, 32, dict(mosaic=0.0, degrees=5.0, perspective=0.0003,
                                                          flipud=0.5)),
                                           (1280, 2, dict(mixup=1.0))])
def test_full_size_batches_equal_restatement(s, batch, extra):
    ims, labs = big_dataset(s, 16)
    c = dict(seed=s + batch, hyp=extra, indices=[(7 * k) % 16 for k in range(batch)])
    imgs, targets = run(c, ims, labs, s=s)
    samples, want_targets = MC.plan(c, ims, labs, s=s)
    np.testing.assert_array_equal(imgs.cpu().numpy(), MC.restate(samples, ims, s=s))
    np.testing.assert_array_equal(targets.cpu().numpy(), want_targets)


def test_decode_jpeg_output_goes_straight_in():
    from yolort_b200.io import decode_jpeg

    srcs, arrays = [], []
    for f in ("zidane.jpg", "bus.jpg"):
        data = torch.from_numpy(np.fromfile(os.path.join(ROOT, "tests", "golden", "jpeg", f), dtype=np.uint8))
        hwc = decode_jpeg(data, DEV).permute(1, 2, 0)            # the decoder's own HWC memory, RGB
        srcs.append(hwc)
        arrays.append(hwc.cpu().numpy().copy())
    labs = [np.array([[0, 0.5, 0.5, 0.2, 0.3]], np.float32)] * 2
    c = dict(seed=21, hyp=dict(mosaic=0.5, mixup=0.5), indices=[0, 1, 1, 0, 0, 1])
    random.seed(21)
    np.random.seed(21)
    imgs, _ = D.train_batch(srcs, labs, c["indices"], img_size=640, hyp=MC.hyp(c), channel_order="rgb")
    samples, _ = MC.plan(c, arrays, labs, s=640)
    np.testing.assert_array_equal(imgs.cpu().numpy(), MC.restate(samples, arrays, s=640, rgb=True))


def test_repeated_calls_give_identical_bits():
    ims, labs = big_dataset(640, 16)
    c = dict(seed=3, hyp=dict(mixup=0.5), indices=list(range(16)))
    runs = [run(c, ims, labs, s=640) for _ in range(3)]
    for imgs, targets in runs[1:]:
        assert torch.equal(imgs, runs[0][0]) and torch.equal(targets, runs[0][1])


def test_training_step_on_train_batch():
    from parity_util import layouts, synth_state_dict
    from yolort_b200.models import yolov5n
    from yolort_b200.models.box_head import SetCriterion

    m = yolov5n(size=(640, 640), score_thresh=0.15)
    m.load_state_dict(synth_state_dict(layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0))
    model = m.model
    model.compute_loss = SetCriterion(model.anchor_generator.strides, model.anchor_generator.anchor_grids,
                                      model.num_classes)
    model = model.to(DEV).train()
    model.backbone.requires_grad_(False)
    ims, labs = big_dataset(640, 16)
    random.seed(0)
    np.random.seed(0)
    imgs, targets = D.train_batch([torch.from_numpy(im).to(DEV) for im in ims], labs, range(16), img_size=640)
    assert len(targets) > 0
    losses = model(imgs.float() / 255, targets)
    loss = sum(losses.values())
    assert bool(torch.isfinite(loss))
    loss.backward()
    grads = [p.grad for p in model.parameters() if p.requires_grad]
    assert grads and all(g is not None and bool(torch.isfinite(g).all()) for g in grads)
    model.compute_loss = None
    model.eval()
