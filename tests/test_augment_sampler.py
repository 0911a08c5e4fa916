"""The device parameter sampler of the training augmentations without a GPU: oracle/sample_augment.py's Philox4x32-10
against Random123's known answers; the restated sampler's invariants (crop windows inside their canvas, within the
aspect bounds and accepted by the IoU rule; kept boxes inside the output; labels following their boxes) on seeded
batches; its distributions against the reference's sampler (oracle/restate_augment.sample_default); the input checks
of `Compose.apply_batch(..., generator=)`."""
import numpy as np
import pytest
import torch
import torchvision
from scipy import stats

import augment_cases as AC
from augment_sampler_cases import CASES, many_boxes
from oracle import restate_augment as R
from oracle import sample_augment as S
from yolort_b200.data import transforms as T

F32 = np.float32


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    assert " ".join(f"{int(w):08x}" for w in S.philox(ctr, key)) == want


def test_words_to_numbers():
    assert S.uniform(0) == 0 and S.uniform(0xFFFFFFFF) == F32(1 - 2.0 ** -24)
    assert int(S.below(0xFFFFFFFF, 6)) == 5 and int(S.below(0x80000000, 6)) == 3
    assert S.PERMS[0] == (0, 1, 2) and S.PERMS[5] == (2, 1, 0)


def replay_box(box, recipe, hw):
    """A box of the input through the geometric ops of a recipe, in the host sampler's fp32 operations."""
    b = np.array(box, dtype=F32)
    h, w = hw
    for op in recipe:
        if op[0] == "zoom":
            _, h, w, top, left, _ = op
            b += np.array([left, top, left, top], dtype=F32)
        elif op[0] == "crop":
            _, top, left, h, w = op
            b = b - np.array([left, top, left, top], dtype=F32)
            b = np.minimum(np.maximum(b, F32(0)), np.array([w, h, w, h], dtype=F32))
        elif op[0] == "hflip":
            b = np.array([F32(w) - b[2], b[1], F32(w) - b[0], b[3]], dtype=F32)
    return b


@pytest.mark.parametrize("key", [(0, 0), (0x12345678, 0x9ABCDEF0), (7, 1 << 31)])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restated_sampler_invariants(case, key):
    _, transforms, sizes, targets = case
    crops = {id(t): t for t in transforms if isinstance(t, T.RandomIoUCrop)}
    out = S.sample(transforms, sizes, targets, key)
    for hw, tg, o in zip(sizes, targets, out):
        assert o["status"] == 0
        for c in o["crops"]:
            ch, cw = c["canvas"]
            top, left, nh, nw = c["window"]
            assert 0 <= top and 0 <= left and top + nh <= ch and left + nw <= cw and nh > 0 and nw > 0
            assert any(t.min_aspect_ratio <= nw / nh <= t.max_aspect_ratio for t in crops.values())
            b = torch.from_numpy(c["boxes"])
            cx, cy = 0.5 * (b[:, 0] + b[:, 2]), 0.5 * (b[:, 1] + b[:, 3])
            keep = (left < cx) & (cx < left + nw) & (top < cy) & (cy < top + nh)
            assert np.array_equal(keep.numpy(), c["keep"]) and bool(keep.any())
            win = torch.tensor([[left, top, left + nw, top + nh]], dtype=torch.float32)
            assert float(torchvision.ops.box_iou(b[keep], win).max()) >= c["option"]
        h, w = o["hw"]
        boxes, labels = o["boxes"], o["labels"]
        assert boxes.shape == (len(labels), 4)
        assert (boxes >= 0).all() and (boxes[:, 0::2] <= w).all() and (boxes[:, 1::2] <= h).all()
        # every kept label names its input box, which the recipe's geometry carries to the kept box
        src = {int(l): k for k, l in enumerate(tg["labels"])}
        assert list(labels) == sorted(labels, key=lambda l: src[int(l)])
        for b, l in zip(boxes, labels):
            assert np.array_equal(b, replay_box(tg["boxes"][src[int(l)]].numpy(), o["recipe"], hw))


def test_an_image_without_an_accepted_window_reports_its_status():
    out = S.sample([T.RandomIoUCrop(sampler_options=[0.5])], [(40, 50), (40, 50)],
                   [{"boxes": torch.zeros(0, 4), "labels": torch.zeros(0, dtype=torch.int64)},
                    {"boxes": torch.tensor([[0.0, 0.0, 50.0, 40.0]]), "labels": torch.tensor([3])}], (5, 6))
    assert out[0]["status"] == S.ST_CROP_ROUNDS and out[0]["recipe"] == [] and out[1]["status"] == 0


# -- distributions against the reference's sampler ---------------------------------------------------------------------
N_IMAGES = 4096
BOX_SETS = {
    "three boxes": ((480, 640), torch.tensor([[20.0, 30.0, 200.0, 260.0], [300.0, 100.0, 420.0, 180.0],
                                              [500.0, 300.0, 630.0, 470.0]])),
    "twenty boxes": ((300, 400), many_boxes(300, 400, 20, seed=5)["boxes"]),
}
KINDS = ("brightness", "contrast", "saturation", "hue", "permute", "zoom", "crop", "hflip")


def summary(recipes, hw, n_in, kept):
    rates = {k: np.mean([any(op[0] == k for op in r) for r in recipes]) for k in KINDS}
    zoom, area = [], []
    for r in recipes:
        h, w = hw
        for op in r:
            if op[0] == "zoom":
                zoom.append(op[2] / w)
                h, w = op[1], op[2]
            elif op[0] == "crop":
                area.append(op[3] * op[4] / (h * w))
    return rates, np.array(zoom), np.array(area), np.array(kept) / n_in


def ks_critical(n, m, alpha=1e-3):
    return np.sqrt(-np.log(alpha / 2) / 2) * np.sqrt((n + m) / (n * m))


@pytest.mark.parametrize("box_set", list(BOX_SETS))
def test_distributions_match_the_reference(box_set):
    hw, boxes = BOX_SETS[box_set]
    labels = torch.arange(len(boxes))
    torch.manual_seed(1234)
    ref = [R.sample_default(hw, boxes, labels) for _ in range(N_IMAGES)]
    ours = S.sample(T.default_train_transforms().transforms, [hw] * N_IMAGES,
                    [{"boxes": boxes, "labels": labels}] * N_IMAGES, (0x2468ACE0, 0x13579BDF))
    a = summary([r for r, _, _ in ref], hw, len(boxes), [len(l) for _, _, l in ref])
    b = summary([o["recipe"] for o in ours], hw, len(boxes), [len(o["labels"]) for o in ours])
    for k in KINDS:
        p = (a[0][k] + b[0][k]) / 2
        sd = np.sqrt(p * (1 - p) * 2 / N_IMAGES)
        assert abs(a[0][k] - b[0][k]) <= 4.5 * sd + 1e-12, (k, a[0][k], b[0][k])
    for what, x, y in zip(("zoom ratio", "crop area", "kept fraction"), a[1:], b[1:]):
        assert len(x) > 500 and len(y) > 500, what
        d = stats.ks_2samp(x, y).statistic
        assert d < ks_critical(len(x), len(y)), (what, d)


# -- input checks ------------------------------------------------------------------------------------------------------
def test_input_errors_without_a_device():
    im = torch.zeros(3, 8, 8, dtype=torch.uint8)
    t = {"boxes": torch.tensor([[1.0, 1.0, 5.0, 5.0]]), "labels": torch.tensor([3])}
    pipe = T.default_train_transforms()
    g = torch.Generator()                                 # a CPU generator
    with pytest.raises(ValueError, match="CUDA torch.Generator"):
        pipe.apply_batch([im], [t], generator=g)
    with pytest.raises(ValueError, match="CUDA torch.Generator"):
        pipe.apply_batch([im], [t], generator=1234)

    class Other(T._Transform):
        def _draw(self, st):
            pass

    with pytest.raises(TypeError):
        T.Compose([Other()]).apply_batch([im], [t], generator=g)
    with pytest.raises(TypeError):
        T.Compose([lambda x: x]).apply_batch([im], [t], generator=g)
    with pytest.raises(ValueError, match="RandomIoUCrop"):
        pipe.apply_batch([im], [None], generator=g)
    for bad in ({"boxes": t["boxes"].double(), "labels": t["labels"]}, {"boxes": t["boxes"][0], "labels": t["labels"]},
                {"boxes": t["boxes"], "labels": t["labels"].int()}, {"boxes": t["boxes"], "labels": torch.tensor([1, 2])}):
        with pytest.raises(ValueError, match="boxes|labels"):
            pipe.apply_batch([im], [bad], generator=g)
    with pytest.raises(NotImplementedError, match="contrast"):
        T.Compose([T.RandomPhotometricDistort()] * 5).apply_batch([im], [t], generator=g)
    with pytest.raises(NotImplementedError, match="ops"):
        T.Compose([T.RandomPhotometricDistort(contrast=(1, 1))] * 4 + [T.RandomHorizontalFlip()]).apply_batch(
            [im], [t], generator=g)
    with pytest.raises(NotImplementedError):
        T.Compose([T.ToTensor(), T.RandomHorizontalFlip()]).apply_batch([im], [t], generator=g)
    # the bound is static: four photometric distorts without contrast (16 ops) pass it
    assert len(T.Compose([T.RandomPhotometricDistort(contrast=(1, 1))] * 4)._sampler_table()) == 4


def test_sampler_table_of_the_default_pipeline():
    table = T.default_train_transforms()._sampler_table()
    kinds = [s.kind for s in table]
    assert kinds == [T._C.YB_AUG_S_PHOTOMETRIC, T._C.YB_AUG_S_ZOOM_OUT, T._C.YB_AUG_S_IOU_CROP, T._C.YB_AUG_S_HFLIP,
                     T._C.YB_AUG_S_NONE, T._C.YB_AUG_S_NONE]
    ph, zo, cr, fl = table[0], table[1], table[2], table[3]
    assert ph.jitter == 15 and ph.p == 0.5 and list(ph.lo) == [F32(0.875), 0.5, 0.5, F32(-0.05)]
    assert list(ph.span) == [0.25, 1.0, 1.0, F32(0.05 - -0.05)]
    assert (zo.lo[0], zo.span[0], zo.p, zo.fill) == (1.0, 3.0, 0.5, 0)
    assert (cr.lo[0], cr.span[0], cr.min_aspect, cr.max_aspect) == (F32(0.3), F32(0.7), 0.5, 2.0)
    assert (cr.trials, cr.n_options, list(cr.options[:7])) == (40, 7, [0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 1.0])
    assert fl.p == 0.5
