"""The training augmentations without a GPU: oracle/restate_augment.py bit-identical to torchvision's CPU tensor
functions and to the unmodified reference (tests/golden/augment.npz); the product's parameter sampler
(yolort_b200.data.transforms, host side) drawing the reference's random numbers in the reference's order; the
YOLOTransform target batch; the input checks that need no device."""
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

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "augment.npz"))
F32 = np.float32


def every_byte_image(h=256, w=259, seed=0):
    """Random bytes, with every value in each channel and every (v, v, v) gray triple."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g)
    v = torch.arange(256, dtype=torch.uint8)
    x[0, 0, :256], x[1, 1, :256], x[2, 2, :256] = v, v, v
    x[:, 3, :256] = v
    return x


def ends(lo, hi):
    return [lo, hi, float(F32(lo + (hi - lo) * 0.37))]


@pytest.mark.parametrize("factor", ends(0.875, 1.125))
def test_brightness_is_torchvision(factor):
    x = every_byte_image()
    assert np.array_equal(R.brightness(x.numpy(), factor), TF.adjust_brightness(x, factor).numpy())


@pytest.mark.parametrize("factor", ends(0.5, 1.5))
def test_contrast_and_saturation_are_torchvision(factor):
    x = every_byte_image()
    assert np.array_equal(R.contrast(x.numpy(), factor), TF.adjust_contrast(x, factor).numpy())
    assert np.array_equal(R.saturation(x.numpy(), factor), TF.adjust_saturation(x, factor).numpy())


@pytest.mark.parametrize("factor", [-0.05, 0.05, 0.0, float(F32(0.0123)), float(F32(-0.0377))])
def test_hue_is_torchvision(factor):
    x = every_byte_image()
    assert np.array_equal(R.hue(x.numpy(), factor), TF.adjust_hue(x, factor).numpy())


def test_geometry_and_float_are_torchvision():
    x = every_byte_image()[:, :37, :53].contiguous()
    xn = x.numpy()
    for perm in ([0, 1, 2], [2, 0, 1], [1, 2, 0]):
        assert np.array_equal(R.permute(xn, perm), x[perm].numpy())
    # zoom-out: F.pad with fill 0, then the border overwritten with the fill colour (transforms.py:261-267)
    top, left, ch, cw, fill = 5, 9, 61, 70, (12, 200, 7)
    ref = TF.pad(x, [left, top, cw - left - 53, ch - top - 37], fill=0)
    v = torch.tensor(fill, dtype=torch.uint8).view(-1, 1, 1)
    ref[..., :top, :] = ref[..., :, :left] = ref[..., top + 37:, :] = ref[..., :, left + 53:] = v
    assert np.array_equal(R.zoom_out(xn, ch, cw, top, left, fill), ref.numpy())
    assert np.array_equal(R.crop(xn, 3, 4, 20, 1), TF.crop(x, 3, 4, 20, 1).numpy())
    assert np.array_equal(R.hflip(xn), TF.hflip(x).numpy())
    assert np.array_equal(R.to_float(xn), TF.convert_image_dtype(x, torch.float).numpy())


@pytest.mark.parametrize("seed", AC.SEEDS)
def test_restatement_reproduces_the_reference(seed):
    images, targets = AC.batch(seed)
    torch.manual_seed(seed)
    outs = []
    for k, (im, t) in enumerate(zip(images, targets)):
        recipe, boxes, labels = R.sample_default((im.shape[1], im.shape[2]), t["boxes"], t["labels"])
        out = R.apply_recipe(im.numpy(), recipe)
        assert R.digest(out) == str(GOLD[f"s{seed}/{k}/sha256"])
        if f"s{seed}/{k}/u8" in GOLD:
            assert np.array_equal(np.round(out * 255).astype(np.uint8), GOLD[f"s{seed}/{k}/u8"])
        assert np.array_equal(boxes.numpy(), GOLD[f"s{seed}/{k}/boxes"])
        assert np.array_equal(labels.numpy(), GOLD[f"s{seed}/{k}/labels"])
        outs.append((out.shape, {"boxes": boxes, "labels": labels}))
    assert np.array_equal(torch.rand(1).numpy(), GOLD[f"s{seed}/rand_after"])
    tb = R.normalize_targets([t for _, t in outs], [s[1:] for s, _ in outs])
    assert np.array_equal(tb.numpy(), GOLD[f"s{seed}/targets_batched"])


@pytest.mark.parametrize("seed", AC.SEEDS)
def test_product_sampler_draws_what_the_reference_draws(seed):
    images, targets = AC.batch(seed)
    torch.manual_seed(seed)
    with AC.DrawLog() as log:
        states = T.default_train_transforms().plan([(im.shape[1], im.shape[2]) for im in images],
                                                   [dict(t) for t in targets])
    assert list(log.kinds) == list(GOLD[f"s{seed}/kinds"])
    assert np.array_equal(np.array(log.values), GOLD[f"s{seed}/draws"])
    assert np.array_equal(torch.rand(1).numpy(), GOLD[f"s{seed}/rand_after"])     # the generator's state after it
    for k, (im, st) in enumerate(zip(images, states)):
        assert (3, st.h, st.w) == tuple(GOLD[f"s{seed}/{k}/shape"])
        assert np.array_equal(st.target["boxes"].numpy(), GOLD[f"s{seed}/{k}/boxes"])
        assert np.array_equal(st.target["labels"].numpy(), GOLD[f"s{seed}/{k}/labels"])
        assert R.digest(R.apply_recipe(im.numpy(), T.recipe_of(st))) == str(GOLD[f"s{seed}/{k}/sha256"])
    for t, t0 in zip(targets, AC.batch(seed)[1]):               # the caller's targets are left as they were
        assert torch.equal(t["boxes"], t0["boxes"]) and torch.equal(t["labels"], t0["labels"])


@pytest.mark.parametrize("seed", AC.SEEDS)
def test_target_batch_is_the_reference(seed):
    sizes = [tuple(GOLD[f"s{seed}/{k}/shape"]) for k in range(len(AC.SIZES))]
    targets = [{"boxes": torch.from_numpy(GOLD[f"s{seed}/{k}/boxes"]),
                "labels": torch.from_numpy(GOLD[f"s{seed}/{k}/labels"])} for k in range(len(AC.SIZES))]
    got = YOLOTransform(*AC.LETTERBOX).batch_targets([torch.empty(s) for s in sizes], targets)
    assert got.dtype == torch.float32 and np.array_equal(got.numpy(), GOLD[f"s{seed}/targets_batched"])
    empty = [{"boxes": torch.zeros(0, 4), "labels": torch.zeros(0, dtype=torch.int64)}] * 2
    assert YOLOTransform(*AC.LETTERBOX).batch_targets([torch.empty(3, 8, 8)] * 2, empty).shape == (0, 6)


def test_reference_names_and_signatures():
    import inspect

    for name in T.__all__:
        assert hasattr(T, name)
    sig = inspect.signature(T.RandomIoUCrop)
    assert list(sig.parameters) == ["min_scale", "max_scale", "min_aspect_ratio", "max_aspect_ratio",
                                    "sampler_options", "trials"]
    assert list(inspect.signature(T.RandomZoomOut).parameters) == ["fill", "side_range", "p"]
    assert list(inspect.signature(T.RandomPhotometricDistort).parameters) == ["contrast", "saturation", "hue",
                                                                              "brightness", "p"]
    assert [type(t).__name__ for t in T.default_train_transforms().transforms] == [
        "RandomPhotometricDistort", "RandomZoomOut", "RandomIoUCrop", "RandomHorizontalFlip", "PILToTensor",
        "ConvertImageDtype"]
    assert isinstance(T.default_val_transforms(), T.ToTensor) and T.ToTensor().dtype == torch.float32
    assert T.collate_fn([(1, "a"), (2, "b")]) == ((1, 2), ("a", "b"))


def test_input_checks_without_a_device():
    from PIL import Image

    pipe = T.default_train_transforms()
    t = {"boxes": torch.tensor([[1.0, 1.0, 5.0, 5.0]]), "labels": torch.tensor([3])}
    with pytest.raises(TypeError):
        pipe(Image.new("RGB", (8, 8)), t)
    with pytest.raises(ValueError):
        pipe(torch.rand(3, 8, 8), t)
    with pytest.raises(ValueError):
        pipe(torch.zeros(8, 8, dtype=torch.uint8), t)
    with pytest.raises(_C.NativeLibraryError):
        pipe(torch.zeros(3, 8, 8, dtype=torch.uint8), t)
    with pytest.raises(NotImplementedError):
        T.Compose([T.ToTensor(), T.RandomHorizontalFlip()]).plan([(8, 8)], [None])
    with pytest.raises(ValueError):
        T.Compose([T.RandomIoUCrop()]).plan([(8, 8)], [None])
