"""YOLOv5's augmentations on the GPU (csrc/v5_augment.cu) against the numpy restatement (oracle/restate_v5aug.py)
and the reference's cv2 digests in tests/golden/v5aug.npz, bit for bit."""
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

import v5aug_cases as VC  # noqa: E402
from oracle import restate_v5aug as R  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.v5.utils import augmentations as A  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "v5aug.npz"))


def sha(a) -> str:
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_case(c, src: torch.Tensor):
    im, lab, extra = VC.inputs(c)
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    if c["fn"] == "augment_hsv":
        A.augment_hsv(src, **c["kw"])
        return src, lab
    if c["fn"] == "random_perspective":
        return A.random_perspective(src, lab.copy(), **c["kw"])
    if c["fn"] == "cutout":
        out = A.cutout(src, lab.copy(), **c["kw"])
        return src, out
    return A.mixup(src, lab.copy(), torch.from_numpy(extra[0]).to(DEV), extra[1])


@pytest.mark.parametrize("name", [c["name"] for c in VC.CASES])
def test_each_function_equals_restatement_and_reference(name):
    c = next(c for c in VC.CASES if c["name"] == name)
    im, _, extra = VC.inputs(c)
    out, lab = run_case(c, torch.from_numpy(im.copy()).to(DEV))
    got = out.cpu().numpy()
    plan, want_lab, r = VC.plan_case(c, im.shape)
    want = R.mixup_pixels(im, extra[0], r) if c["fn"] == "mixup" else im if plan is None else VC.restate(plan, im)
    np.testing.assert_array_equal(got, want)
    assert sha(got) == str(GOLD[f"{name}/sha256"])
    np.testing.assert_array_equal(np.asarray(lab), GOLD[f"{name}/labels"])


@pytest.mark.parametrize("layout", ["contiguous", "hwc_view", "strided"])
def test_strided_sources(layout):
    c = next(c for c in VC.CASES if c["name"] == "affine")
    im, _, _ = VC.inputs(c)
    t = torch.from_numpy(im.copy()).to(DEV)
    if layout == "hwc_view":            # [H, W, 3] view of planar [3, H, W] memory
        t = t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
    elif layout == "strided":           # every other column of a wider image
        wide = torch.zeros((im.shape[0], 2 * im.shape[1], 3), dtype=torch.uint8, device=DEV)
        wide[:, ::2] = t
        t = wide[:, ::2]
    out, _ = run_case(c, t)
    assert sha(out) == str(GOLD[f"{c['name']}/sha256"])
    c = next(c for c in VC.CASES if c["name"] == "hsv_odd")
    im, _, _ = VC.inputs(c)
    t = torch.from_numpy(im.copy()).to(DEV).permute(2, 0, 1).contiguous().permute(1, 2, 0)
    out, _ = run_case(c, t)
    assert sha(out) == str(GOLD[f"{c['name']}/sha256"])


def test_decode_jpeg_output_goes_straight_in():
    from yolort_b200.io import decode_jpeg

    path = os.path.join(ROOT, "tests", "golden", "jpeg", "zidane.jpg")
    data = torch.from_numpy(np.fromfile(path, dtype=np.uint8))
    chw = decode_jpeg(data, DEV)
    hwc = chw.permute(1, 2, 0)                       # the decoder's own HWC memory
    src = hwc.cpu().numpy().copy()
    random.seed(3)
    np.random.seed(3)
    outs, _ = A.apply_batch([hwc], None, channel_order="rgb")
    random.seed(3)
    np.random.seed(3)
    plans, _ = A.plan_batch([src.shape[:2]], [None], A.HYP_SCRATCH)
    np.testing.assert_array_equal(outs[0].cpu().numpy(), VC.restate(plans[0], src, rgb=True))


@pytest.mark.parametrize("channel_order", ["bgr", "rgb"])
def test_apply_batch_equals_restatement(channel_order):
    hyp = dict(A.HYP_SCRATCH, degrees=8.0, shear=3.0, flipud=0.5, perspective=0.0)
    sizes = [(48, 64), (37, 53), (1, 40), (30, 1), (64, 96), (40, 33)]
    ims = [VC.image(20 + k, h, w) for k, (h, w) in enumerate(sizes)]
    labs = [VC.labels(20 + k, h, w, 3) for k, (h, w) in enumerate(sizes)]
    targets = [{"boxes": torch.from_numpy(l[:, 1:].copy()).to(DEV), "labels": torch.from_numpy(l[:, 0]).long().to(DEV),
                "image_id": k} for k, l in enumerate(labs)]
    for persp in (0.0, 0.001):
        hyp["perspective"] = persp
        random.seed(11)
        np.random.seed(11)
        outs, tgs = A.apply_batch([torch.from_numpy(im).to(DEV) for im in ims], targets, hyp,
                                  channel_order=channel_order)
        random.seed(11)
        np.random.seed(11)
        plans, want_labs = A.plan_batch(sizes, [l.copy() for l in labs], hyp)
        assert any(p.flip_lr for p in plans)
        for im, o, p, t, wl in zip(ims, outs, plans, tgs, want_labs):
            np.testing.assert_array_equal(o.cpu().numpy(), VC.restate(p, im, rgb=channel_order == "rgb"))
            np.testing.assert_array_equal(t["boxes"].cpu().numpy(), wl[:, 1:5])
            assert t["boxes"].device == torch.device(DEV) and t["labels"].dtype == torch.int64
        assert [t["image_id"] for t in tgs] == list(range(len(sizes)))


def _one_op(src: np.ndarray, ops: int, lut=None) -> np.ndarray:
    t = torch.from_numpy(src).to(DEV)
    out = torch.empty_like(t)
    plan = A._Plan(int(t.shape[0]), int(t.shape[1]))
    descs = (_C.V5Image * 1)()
    A._fill(descs[0], t, out, plan, False)
    descs[0].ops = ops
    if lut is not None:
        np.ctypeslib.as_array(descs[0].lut)[...] = lut
    _C.v5_augment(descs, [t, out], t.device)
    return out.cpu().numpy()


def test_kernel_colour_tables_equal_reference():
    bgr = R.all_bgr_image()
    ident = np.tile(np.arange(256, dtype=np.uint8), (3, 1))
    for rgb in (False, True):
        tag, bit = ("rgb", _C.YB_V5_RGB) if rgb else ("bgr", 0)
        assert sha(_one_op(bgr, _C.YB_V5_TO_HSV | bit)) == str(GOLD[f"tables/to_hsv_{tag}"])
        for w in (256, 1):
            got = _one_op(R.all_hsv_image(w), _C.YB_V5_FROM_HSV | bit)
            assert sha(got) == str(GOLD[f"tables/from_hsv_{tag}_w{w}"])
        ops = _C.YB_V5_TO_HSV | _C.YB_V5_LUT | _C.YB_V5_FROM_HSV | bit
        assert sha(_one_op(bgr, ops, ident)) == str(GOLD[f"tables/round_trip_{tag}"])


def test_augment_hsv_writes_in_place_and_identity_returns_the_input():
    im = torch.from_numpy(VC.image(5, 40, 50)).to(DEV)
    before, ptr = im.clone(), im.data_ptr()
    np.random.seed(0)
    assert A.augment_hsv(im) is None
    assert im.data_ptr() == ptr and not torch.equal(im, before)
    out, lab = A.random_perspective(im, np.zeros((0, 5)), degrees=0, translate=0, scale=0, shear=0)
    assert out is im and lab.shape == (0, 5)


def test_repeated_calls_give_identical_bits():
    ims = [torch.from_numpy(VC.image(30 + k, 480, 640)).to(DEV) for k in range(4)]
    runs = []
    for _ in range(3):
        random.seed(4)
        np.random.seed(4)
        runs.append([o.clone() for o in A.apply_batch(ims, None, A.HYP_SCRATCH)[0]])
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


def test_training_step_on_augmented_batch():
    from parity_util import layouts, synth_state_dict
    from yolort_b200.models import yolov5n
    from yolort_b200.models.box_head import SetCriterion

    m = yolov5n(size=(640, 640), score_thresh=0.15)
    m.load_state_dict(synth_state_dict(layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0))
    model = m.model
    model.compute_loss = SetCriterion(model.anchor_generator.strides, model.anchor_generator.anchor_grids,
                                      model.num_classes)
    m = m.to(DEV).train()
    model.backbone.requires_grad_(False)
    ims = [torch.from_numpy(VC.image(100 + k, 480, 640)).to(DEV) for k in range(32)]
    targets = []
    for k in range(32):
        l = VC.labels(100 + k, 480, 640, 4)
        targets.append({"boxes": torch.from_numpy(l[:, 1:].copy()).to(DEV),
                        "labels": torch.from_numpy(l[:, 0]).long().to(DEV)})
    random.seed(0)
    np.random.seed(0)
    outs, tgs = A.apply_batch(ims, targets, A.HYP_SCRATCH, channel_order="rgb")
    losses = m([o.permute(2, 0, 1) for o in outs], tgs)
    loss = sum(losses.values())
    assert bool(torch.isfinite(loss))
    loss.backward()
    grads = [p.grad for p in model.parameters() if p.requires_grad]
    assert grads and all(g is not None and bool(torch.isfinite(g).all()) for g in grads)
    model.compute_loss = None
    m.eval()
