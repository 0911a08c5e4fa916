"""The training augmentations on the device (yolort_b200.data.transforms, csrc/augment.cu): every op alone and the
default pipeline bit-identical to oracle/restate_augment.py and to the reference's fixtures (tests/golden/augment.npz),
on mixed-size batches (1x1 crops, a 4x zoom of 1280x720, odd widths, HWC-strided sources, images without boxes);
contrast on large images; repeated calls; the fused float output; the input checks; the YOLOTransform target batch and
the YOLOv5 training step."""
import os

import numpy as np
import pytest
import torch
import torchvision.transforms._functional_tensor as TF

import augment_cases as AC
from oracle import restate_augment as R
from yolort_b200 import _C
from yolort_b200.data import transforms as T
from yolort_b200.models.transform import YOLOTransform

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "augment.npz"))


def state(hw, recipe):
    """A planned image from a recipe in restate_augment's notation."""
    st = T._State(hw, None)
    h, w = hw
    kinds = {"brightness": _C.YB_AUG_BRIGHTNESS, "contrast": _C.YB_AUG_CONTRAST, "saturation": _C.YB_AUG_SATURATION,
             "hue": _C.YB_AUG_HUE}
    for op in recipe:
        if op[0] in kinds:
            st.ops.append((kinds[op[0]], (0, h, w) if op[0] == "contrast" else (), float(op[1])))
        elif op[0] == "permute":
            st.ops.append((_C.YB_AUG_PERMUTE, op[1], None))
        elif op[0] == "zoom":
            _, ch, cw, top, left, f = op
            st.ops.append((_C.YB_AUG_ZOOM_OUT, (top, left, h, w, ch, cw, f[0] | f[1] << 8 | f[2] << 16), None))
            h, w = ch, cw
        elif op[0] == "crop":
            _, top, left, h, w = op
            st.ops.append((_C.YB_AUG_CROP, (top, left, h, w), None))
        elif op[0] == "hflip":
            st.ops.append((_C.YB_AUG_HFLIP, (w,), None))
        elif op[0] == "float":
            st.float_out = True
    st.h, st.w = h, w
    return st


def synth(h, w, seed, hwc=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g)
    if hwc:       # [3, H, W] view of interleaved memory, as decode_jpeg returns
        return x.permute(1, 2, 0).contiguous().to(DEV).permute(2, 0, 1)
    return x.to(DEV)


# (h, w, recipe) per image of one batch: each op alone with both ends of its range, then chains
MIXED = [
    (37, 53, [("brightness", 0.875)]),
    (64, 81, [("brightness", 1.125)]),
    (29, 33, [("contrast", 0.5)]),
    (40, 41, [("contrast", 1.5)]),
    (31, 77, [("saturation", 0.5)]),
    (50, 23, [("saturation", 1.5)]),
    (45, 45, [("hue", -0.05)]),
    (33, 47, [("hue", 0.05)]),
    (21, 99, [("hue", 0.0)]),
    (19, 17, [("permute", (2, 0, 1))]),
    (720, 1280, [("zoom", 2880, 5120, 1000, 3000, (0, 0, 0))]),
    (30, 31, [("zoom", 61, 97, 7, 60, (12, 200, 7))]),
    (41, 59, [("crop", 40, 58, 1, 1)]),
    (41, 59, [("crop", 3, 5, 30, 51)]),
    (23, 71, [("hflip",)]),
    (33, 47, [("brightness", 1.0625), ("contrast", 0.75), ("saturation", 1.25), ("hue", 0.0312), ("permute", (1, 2, 0)),
              ("zoom", 70, 100, 20, 31, (0, 0, 0)), ("crop", 10, 20, 45, 61), ("hflip",)]),
    # colour after geometry: the fill and the flip are seen by the contrast mean
    (27, 35, [("zoom", 54, 71, 3, 30, (9, 99, 200)), ("hflip",), ("contrast", 1.3), ("crop", 2, 1, 50, 69),
              ("saturation", 0.7), ("contrast", 0.6)]),
]


@pytest.mark.parametrize("float_out", [False, True])
def test_each_op_and_chains_equal_the_restatement(float_out):
    images, states, want = [], [], []
    for k, (h, w, recipe) in enumerate(MIXED):
        if float_out:
            recipe = recipe + [("float",)]
        im = synth(h, w, k, hwc=k % 3 == 1)
        images.append(im)
        states.append(state((h, w), recipe))
        want.append(R.apply_recipe(im.cpu().numpy(), recipe))
    got = T.run_recipes(images, states)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == (torch.float32 if float_out else torch.uint8)
        assert np.array_equal(g.cpu().numpy(), w), (k, MIXED[k][2])


def test_contrast_on_large_images():
    """Grayscale sums beyond 2^24: torch's fp32 sum rounds, the kernel's integer sum does not."""
    h, w = 720, 1280
    im = synth(h, w, 7)
    for f in (0.5, 1.5):
        got = T.run_recipes([im], [state((h, w), [("contrast", f)])])[0].cpu()
        ref = TF.adjust_contrast(im.cpu(), f)
        diff = (got.int() - ref.int()).abs()
        assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) <= 1e-4
        exact = float(R.gray_mean(im.cpu().numpy()))
        torch_mean = float(TF.rgb_to_grayscale(im.cpu()).float().mean())
        assert abs(exact - torch_mean) <= 1e-5 * exact
        assert np.array_equal(got.numpy(), R.contrast(im.cpu().numpy(), f))


@pytest.mark.parametrize("device_targets", [False, True])
@pytest.mark.parametrize("seed", AC.SEEDS)
def test_default_pipeline_is_the_reference(seed, device_targets):
    images, targets = AC.batch(seed)
    images = [im.to(DEV) for im in images]
    if device_targets:
        targets = [{k: v.to(DEV) for k, v in t.items()} for t in targets]
    torch.manual_seed(seed)
    outs, tg = T.default_train_transforms().apply_batch(images, targets)
    assert np.array_equal(torch.rand(1).numpy(), GOLD[f"s{seed}/rand_after"])
    for k, (o, t) in enumerate(zip(outs, tg)):
        a = o.cpu().numpy()
        assert o.dtype == torch.float32 and a.shape == tuple(GOLD[f"s{seed}/{k}/shape"])
        assert R.digest(a) == str(GOLD[f"s{seed}/{k}/sha256"])
        assert t["boxes"].device.type == ("cuda" if device_targets else "cpu")
        assert np.array_equal(t["boxes"].cpu().numpy(), GOLD[f"s{seed}/{k}/boxes"])
        assert np.array_equal(t["labels"].cpu().numpy(), GOLD[f"s{seed}/{k}/labels"])
    # image by image through Compose.__call__ is the same computation
    torch.manual_seed(seed)
    pipe = T.default_train_transforms()
    for k, (im, t) in enumerate(zip(images, targets)):
        o, _ = pipe(im, t)
        assert R.digest(o.cpu().numpy()) == str(GOLD[f"s{seed}/{k}/sha256"])
    # the fixture's target batch from the augmented batch
    _, tb = YOLOTransform(*AC.LETTERBOX)(outs, tg)
    assert tb.device.type == "cuda" and np.array_equal(tb.cpu().numpy(), GOLD[f"s{seed}/targets_batched"])


def test_repeated_call_and_float_output():
    images, targets = AC.batch(3)
    images = [im.to(DEV) for im in images]
    runs = []
    for pipe in (T.default_train_transforms(), T.default_train_transforms()):
        torch.manual_seed(11)
        runs.append(pipe.apply_batch(images, targets)[0])
    u8 = T.Compose(T.default_train_transforms().transforms[:-1])
    torch.manual_seed(11)
    bytes_out = u8.apply_batch(images, targets)[0]
    for a, b, c in zip(*runs, bytes_out):
        assert torch.equal(a, b)
        assert c.dtype == torch.uint8 and torch.equal(a.cpu(), c.cpu().to(torch.float32) / 255.0)


def test_single_transforms_and_errors():
    im = synth(40, 50, 1)
    t = {"boxes": torch.tensor([[0.0, 0.0, 50.0, 40.0]]), "labels": torch.tensor([1]), "image_id": torch.tensor(7)}
    torch.manual_seed(0)
    o, tt = T.RandomHorizontalFlip(p=1.0)(im, t)
    assert torch.equal(o.cpu(), im.cpu().flip(-1)) and tt["image_id"] is t["image_id"]
    o, _ = T.ToTensor()(im, None)
    assert torch.equal(o.cpu(), im.cpu().float() / 255.0)
    o, _ = T.PILToTensor()(im, None)
    assert torch.equal(o, im)
    from PIL import Image

    with pytest.raises(TypeError):
        T.RandomZoomOut()(Image.new("RGB", (8, 8)), t)
    with pytest.raises(ValueError):
        T.RandomZoomOut()(im.float(), t)
    with pytest.raises(ValueError):
        T.RandomZoomOut()(im[0], t)
    with pytest.raises(_C.NativeLibraryError):
        T.RandomZoomOut()(im.cpu(), t)
    with pytest.raises(NotImplementedError):
        T.RandomZoomOut()(im, dict(t, masks=torch.zeros(1, 40, 50)))
    # the device is still usable
    o, _ = T.PILToTensor()(im, None)
    torch.cuda.synchronize()


def test_yolov5_training_step_returns_the_criterion_dict():
    from parity_util import layouts, synth_state_dict
    from yolort_b200.models import yolov5n
    from yolort_b200.models.box_head import SetCriterion

    m = yolov5n(size=(128, 128), score_thresh=0.15)
    m.load_state_dict(synth_state_dict(layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0))
    model = m.model
    model.compute_loss = SetCriterion(model.anchor_generator.strides, model.anchor_generator.anchor_grids,
                                      model.num_classes)
    m = m.to(DEV).train()
    images, targets = AC.batch(2)
    torch.manual_seed(2)
    images, targets = T.default_train_transforms().apply_batch([im.to(DEV) for im in images], targets)
    got = m(images, targets)
    samples, _ = m.transform(images, None)                       # the letterbox by hand
    tb = R.normalize_targets(targets, [tuple(im.shape[1:]) for im in images]).to(DEV)
    want = model(samples.tensors, tb)
    assert list(got) == ["cls_logits", "bbox_regression", "objectness"]
    for k in got:
        assert torch.equal(got[k], want[k]) and bool(torch.isfinite(got[k]).all())
    model.compute_loss = None
    with pytest.raises(NotImplementedError):
        m(images, targets)
    m.eval()
