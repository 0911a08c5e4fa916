"""Seeded cases of YOLOv5's augmentations (oracle/make_golden_v5aug.py writes tests/golden/v5aug.npz from them)."""
import random

import numpy as np

# name, function, seed, image size, keyword arguments, boxes
CASES = [
    dict(name="hsv_odd", fn="augment_hsv", seed=1, hw=(37, 53), kw={}),
    dict(name="hsv_scratch", fn="augment_hsv", seed=2, hw=(48, 70), kw=dict(hgain=0.015, sgain=0.7, vgain=0.4)),
    dict(name="hsv_zero", fn="augment_hsv", seed=3, hw=(20, 30), kw=dict(hgain=0, sgain=0, vgain=0)),
    dict(name="hsv_row", fn="augment_hsv", seed=4, hw=(1, 77), kw={}),
    dict(name="affine", fn="random_perspective", seed=5, hw=(45, 61), kw={}, boxes=6),
    dict(name="affine_scratch", fn="random_perspective", seed=6, hw=(48, 64),
         kw=dict(degrees=0.0, translate=0.1, scale=0.5, shear=0.0), boxes=5),
    dict(name="perspective", fn="random_perspective", seed=7, hw=(33, 47), kw=dict(perspective=0.001), boxes=4),
    dict(name="perspective_wide", fn="random_perspective", seed=8, hw=(24, 150),
         kw=dict(degrees=30, shear=5, perspective=0.0005), boxes=3),
    dict(name="border", fn="random_perspective", seed=9, hw=(40, 50), kw=dict(border=(6, 9)), boxes=4),
    dict(name="border_negative", fn="random_perspective", seed=10, hw=(60, 64), kw=dict(border=(-8, -10)), boxes=4),
    dict(name="identity", fn="random_perspective", seed=11, hw=(30, 40),
         kw=dict(degrees=0, translate=0, scale=0, shear=0), boxes=3),
    dict(name="one_row", fn="random_perspective", seed=12, hw=(1, 40), kw={}),
    dict(name="one_column", fn="random_perspective", seed=13, hw=(30, 1), kw={}),
    dict(name="no_boxes", fn="random_perspective", seed=14, hw=(40, 40), kw={}, boxes=0),
    dict(name="large", fn="random_perspective", seed=15, hw=(3000, 4000),
         kw=dict(degrees=0.0, translate=0.1, scale=0.5, shear=0.0), boxes=8),
    dict(name="cutout", fn="cutout", seed=16, hw=(60, 80), kw=dict(p=1.0), boxes=6),
    dict(name="cutout_skip", fn="cutout", seed=17, hw=(20, 20), kw=dict(p=0.0), boxes=2),
    dict(name="mixup", fn="mixup", seed=18, hw=(30, 41), kw={}, boxes=2),
]


def image(seed: int, h: int, w: int) -> np.ndarray:
    """A uint8 [h, w, 3] image with smooth gradients and noise (bilinear taps see both)."""
    rng = np.random.default_rng(seed)
    y = np.arange(h)[:, None, None]
    x = np.arange(w)[None, :, None]
    base = (y * 7 + x * 3 + np.array([0, 85, 170])) % 256
    return ((base + rng.integers(0, 40, (h, w, 3))) % 256).astype(np.uint8)


def labels(seed: int, h: int, w: int, n: int) -> np.ndarray:
    """[n, 5] float32 (cls, x1, y1, x2, y2); the first box touches the image's border."""
    if n == 0:
        return np.zeros((0, 5), np.float32)
    rng = np.random.default_rng(seed + 1000)
    x1 = rng.uniform(0, w * 0.6, n)
    y1 = rng.uniform(0, h * 0.6, n)
    x2 = np.minimum(w, x1 + rng.uniform(2, max(2.0, w * 0.5), n))
    y2 = np.minimum(h, y1 + rng.uniform(2, max(2.0, h * 0.5), n))
    out = np.stack([rng.integers(0, 80, n).astype(np.float64), x1, y1, x2, y2], 1).astype(np.float32)
    out[0, 1:] = (0, 0, w, min(h, max(3, h // 2)))
    return out


def inputs(case):
    """(image, labels, extra) of a case; extra is (image2, labels2) for mixup."""
    h, w = case["hw"]
    im = image(case["seed"], h, w)
    lab = labels(case["seed"], h, w, case.get("boxes", 0))
    extra = None
    if case["fn"] == "mixup":
        extra = (image(case["seed"] + 500, h, w), labels(case["seed"] + 500, h, w, 1))
    return im, lab, extra


class DrawLog:
    """Records every value drawn from `random` and `np.random` inside the block (the calls the reference makes)."""

    def __enter__(self):
        self.values, self.kinds, self._saved = [], [], []
        for mod, names in ((random, ("random", "uniform", "randint")), (np.random, ("uniform", "beta"))):
            for n in names:
                f = getattr(mod, n)
                self._saved.append((mod, n, f))
                setattr(mod, n, self._wrap(f, f"{mod.__name__}.{n}"))
        return self

    def _wrap(self, f, kind):
        def g(*a, **k):
            v = f(*a, **k)
            for x in np.ravel(v):
                self.values.append(float(x))
                self.kinds.append(kind)
            return v
        return g

    def __exit__(self, *exc):
        for mod, n, f in self._saved:
            setattr(mod, n, f)


def plan_case(case, im_shape):
    """The package's host draws for a case, after random.seed / np.random.seed: (plan, labels, mixup ratio).
    The plan is None where the function leaves the image as it is."""
    from yolort_b200.v5.utils import augmentations as A

    h, w = im_shape[:2]
    _, lab, extra = inputs(case)
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    kw, fn = case["kw"], case["fn"]
    plan, r = None, None
    if fn == "augment_hsv":
        lut = A._hsv_draw(kw.get("hgain", 0.5), kw.get("sgain", 0.5), kw.get("vgain", 0.5))
        if lut is not None:
            plan = A._Plan(h, w)
            plan.lut = lut
    elif fn == "random_perspective":
        args = dict(degrees=10, translate=0.1, scale=0.1, shear=10, perspective=0.0, border=(0, 0))
        args.update(kw)
        M, s, height, width = A._perspective_draw((h, w), args["degrees"], args["translate"], args["scale"],
                                                  args["shear"], args["perspective"], args["border"])
        p = A._Plan(height, width)
        A._warp_plan(p, M, args["border"], args["perspective"])
        plan = p if p.inv is not None else None
        lab = A._warp_targets(lab.copy(), M, s, width, height, args["perspective"])
    elif fn == "cutout":
        rects, lab = A._cutout_draw(h, w, lab.copy(), kw.get("p", 0.5))
        if rects is not None:
            plan = A._Plan(h, w)
            plan.rects = rects
    else:
        r = np.random.beta(32.0, 32.0)
        lab = np.concatenate((lab, extra[1]), 0)
    return plan, lab, r


def restate(plan, src: np.ndarray, rgb: bool = False) -> np.ndarray:
    """oracle/restate_v5aug.py's pipeline for a plan."""
    from oracle import restate_v5aug as R

    return R.pipeline(src, plan.out_h, plan.out_w, inv=plan.inv, perspective=plan.perspective, lut=plan.lut,
                      flip_ud=plan.flip_ud, flip_lr=plan.flip_lr, rects=plan.rects, rgb=rgb)
