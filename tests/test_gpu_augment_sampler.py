"""The device parameter sampler (`Compose.apply_batch(..., generator=)`, csrc/augment_sample.cu) against its
restatement oracle/sample_augment.py fed the same key: descriptors, boxes, labels and counts bit for bit, on the CPU
test's cases and on 32 seeded 640x480 images; pixels bit-identical to oracle/restate_augment.apply_recipe on the
sampled recipes; seeds; torch's default generators untouched; errors before anything is drawn; the training step."""
import ctypes

import numpy as np
import pytest
import torch

import augment_cases as AC
from oracle import restate_augment as R
from oracle import sample_augment as S
from augment_sampler_cases import CASES
from yolort_b200 import _C
from yolort_b200.data import transforms as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def synth(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g).to(DEV)


def key_of(seed):
    """The key a call with a generator seeded `seed` draws (the call draws it the same way)."""
    g = torch.Generator(DEV).manual_seed(seed)
    return [int(v) for v in T._draw_key(g, torch.device(DEV)).cpu()]


def desc_of(im, recipe):
    """The yb_aug_image the host sampler fills for `recipe` (restate_augment notation) on image `im`."""
    st = T._State(tuple(im.shape[1:]), None)
    h, w = st.h, st.w
    kinds = {"brightness": _C.YB_AUG_BRIGHTNESS, "contrast": _C.YB_AUG_CONTRAST, "saturation": _C.YB_AUG_SATURATION,
             "hue": _C.YB_AUG_HUE}
    for op in recipe:
        if op[0] in kinds:
            st.ops.append((kinds[op[0]], (0, h, w) if op[0] == "contrast" else (), op[1]))
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
    st.h, st.w = h, w
    d = _C.AugImage()
    T._fill_desc(d, im, st)
    return d


def check_against_restatement(transforms, images, targets, seed):
    pipe = T.Compose(transforms)
    host = [None if t is None else {k: v.cpu() for k, v in t.items()} for t in targets]
    want = S.sample(transforms, [tuple(im.shape[1:]) for im in images], host, key_of(seed))
    g = torch.Generator(DEV).manual_seed(seed)
    descs, got = pipe.sample(images, targets, g)
    for k, (im, d, t, w) in enumerate(zip(images, descs, got, want)):
        e = desc_of(im, [op for op in w["recipe"] if op[0] != "float"])
        assert ctypes.string_at(ctypes.addressof(d), ctypes.sizeof(d)) == \
            ctypes.string_at(ctypes.addressof(e), ctypes.sizeof(e)), (k, w["recipe"])
        assert (d.out_h, d.out_w) == w["hw"]
        if t is None:
            assert w["boxes"] is None
            continue
        assert t["boxes"].dtype == torch.float32 and t["labels"].dtype == torch.int64
        assert np.array_equal(t["boxes"].cpu().numpy(), w["boxes"]), k
        assert np.array_equal(t["labels"].cpu().numpy(), w["labels"]), k
    return want


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_descriptors_and_boxes_equal_the_restatement(case, seed):
    _, transforms, sizes, targets = case
    images = [synth(h, w, k) for k, (h, w) in enumerate(sizes)]
    check_against_restatement(transforms, images, targets, seed)


def coco_like(n=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    images = [torch.randint(0, 256, (3, 480, 640), dtype=torch.uint8, generator=g).to(DEV) for _ in range(n)]
    targets = []
    for _ in range(n):
        k = int(torch.randint(1, 8, (1,), generator=g))
        xy = torch.rand(k, 2, generator=g) * torch.tensor([500.0, 360.0])
        wh = torch.rand(k, 2, generator=g) * torch.tensor([140.0, 120.0]) + 4
        targets.append({"boxes": torch.cat([xy, xy + wh], 1), "labels": torch.randint(0, 80, (k,), generator=g),
                        "image_id": torch.tensor(len(targets))})
    return images, targets


@pytest.mark.parametrize("device_targets", [False, True])
def test_32_images_and_pixels_equal_the_restatement(device_targets):
    images, targets = coco_like()
    if device_targets:
        targets = [{k: v.to(DEV) for k, v in t.items()} for t in targets]
    pipe = T.default_train_transforms()
    want = check_against_restatement(pipe.transforms, images, targets, 42)
    outs, got = pipe.apply_batch(images, targets, generator=torch.Generator(DEV).manual_seed(42))
    for im, o, t, t0, w in zip(images, outs, got, targets, want):
        assert o.dtype == torch.float32
        assert np.array_equal(o.cpu().numpy(), R.apply_recipe(im.cpu().numpy(), w["recipe"]))
        assert t["boxes"].device == t0["boxes"].device and t["labels"].device == t0["labels"].device
        assert t["image_id"] is t0["image_id"]
        assert np.array_equal(t["boxes"].cpu().numpy(), w["boxes"])
    assert sum("crop" in [op[0] for op in w["recipe"]] for w in want) > 0


@pytest.mark.parametrize("device_targets", [False, True])
def test_images_without_targets_keep_the_rows_of_the_others(device_targets):
    """Without RandomIoUCrop a target may be None; the other images' boxes stay in their rows."""
    images, targets = AC.batch(4)
    images = [im.to(DEV) for im in images]
    if device_targets:
        targets = [{k: v.to(DEV) for k, v in t.items()} for t in targets]
    targets[0] = targets[2] = None
    transforms = [T.RandomPhotometricDistort(), T.RandomZoomOut(p=0.9), T.RandomHorizontalFlip(p=0.6)]
    want = check_against_restatement(transforms, images, targets, 8)
    _, got = T.Compose(transforms).apply_batch(images, targets, generator=torch.Generator(DEV).manual_seed(8))
    assert got[0] is None and got[2] is None
    for k in (1, 3):
        assert np.array_equal(got[k]["boxes"].cpu().numpy(), want[k]["boxes"])
        assert got[k]["boxes"].device == targets[k]["boxes"].device


def test_pixels_of_the_other_cases_equal_the_restatement():
    for name, transforms, sizes, targets in CASES[-2:]:
        images = [synth(h, w, k) for k, (h, w) in enumerate(sizes)]
        want = S.sample(transforms, sizes, targets, key_of(3))
        outs, _ = T.Compose(transforms).apply_batch(images, targets, generator=torch.Generator(DEV).manual_seed(3))
        for im, o, w in zip(images, outs, want):
            assert o.dtype == (torch.float32 if w["recipe"][-1:] == [("float",)] else torch.uint8)
            assert np.array_equal(o.cpu().numpy(), R.apply_recipe(im.cpu().numpy(), w["recipe"])), name


def test_seeds_streams_and_default_generators():
    images, targets = coco_like(8, seed=1)
    pipe = T.default_train_transforms()
    cpu_state, cuda_state = torch.get_rng_state(), torch.cuda.get_rng_state(DEV)
    g = torch.Generator(DEV)
    runs = []
    for seed in (5, 5, 6):
        g.manual_seed(seed)
        runs.append(pipe.apply_batch(images, targets, generator=g))
    nxt = pipe.apply_batch(images, targets, generator=g)          # the next call draws a fresh key
    assert torch.equal(torch.get_rng_state(), cpu_state) and torch.equal(torch.cuda.get_rng_state(DEV), cuda_state)

    def same(a, b):
        return all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(a[0], b[0])) and all(
            torch.equal(s["boxes"], t["boxes"]) and torch.equal(s["labels"], t["labels"]) for s, t in zip(a[1], b[1]))

    assert same(runs[0], runs[1])
    assert not same(runs[0], runs[2]) and not same(runs[2], nxt)


def test_input_errors_are_raised_before_anything_is_drawn():
    im = synth(40, 50, 1)
    t = {"boxes": torch.tensor([[1.0, 1.0, 30.0, 20.0]]), "labels": torch.tensor([3])}
    whole = {"boxes": torch.tensor([[0.0, 0.0, 50.0, 40.0]]), "labels": torch.tensor([3])}
    pipe = T.default_train_transforms()
    g = torch.Generator(DEV).manual_seed(0)
    state = g.get_state()
    with pytest.raises(ValueError):
        pipe.apply_batch([im], [t], generator=torch.Generator())
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            pipe.apply_batch([im], [t], generator=torch.Generator("cuda:1"))
    with pytest.raises(TypeError):
        T.Compose([T.RandomHorizontalFlip(), object()]).apply_batch([im], [t], generator=g)
    with pytest.raises(ValueError):
        pipe.apply_batch([im], [None], generator=g)
    with pytest.raises(ValueError):
        pipe.apply_batch([im], [{"boxes": t["boxes"].half(), "labels": t["labels"]}], generator=g)
    with pytest.raises(ValueError):
        pipe.apply_batch([im], [{"boxes": t["boxes"], "labels": t["labels"].to(torch.int32)}], generator=g)
    with pytest.raises(NotImplementedError):
        T.Compose([T.RandomPhotometricDistort()] * 5).apply_batch([im], [t], generator=g)
    with pytest.raises(ValueError):
        pipe.apply_batch([im.float()], [t], generator=g)
    with pytest.raises(_C.NativeLibraryError):
        pipe.apply_batch([im.cpu()], [t], generator=g)
    assert torch.equal(g.get_state(), state)
    # an IoU crop that can never accept a window (no boxes, no option of 1.0) gives up and names the image
    none = {"boxes": torch.zeros(0, 4), "labels": torch.zeros(0, dtype=torch.int64)}
    with pytest.raises(RuntimeError, match=r"\[1\]"):
        T.Compose([T.RandomIoUCrop(sampler_options=[0.5])]).apply_batch([im, im], [whole, none], generator=g)
    o, tt = T.Compose([T.RandomHorizontalFlip(p=1.0)]).apply_batch([im], [t], generator=g)
    assert torch.equal(o[0].cpu(), im.cpu().flip(-1))
    assert torch.equal(tt[0]["boxes"], torch.tensor([[20.0, 1.0, 49.0, 20.0]]))


def test_yolov5_training_step_on_a_sampled_batch():
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
    images, targets = T.default_train_transforms().apply_batch(
        [im.to(DEV) for im in images], [{k: v.to(DEV) for k, v in t.items()} for t in targets],
        generator=torch.Generator(DEV).manual_seed(9))
    got = m(images, targets)
    assert list(got) == ["cls_logits", "bbox_regression", "objectness"]
    for k in got:
        assert bool(torch.isfinite(got[k]).all())
    m.eval()
