"""Seeded datasets and cases of YOLOv5's mosaic loader (oracle/make_golden_v5mosaic.py writes
tests/golden/v5mosaic.npz from them)."""
import random

import numpy as np

from v5aug_cases import image

S = 64
# load_image at s = 64: upscale, downscale, exact 2x (INTER_AREA), int() leaving the long side at 63 (98 * (64 / 98)
# is 63.99...: letterbox resizes a second time), portrait, landscape, and an image already 64 long
SHAPES = [(20, 30), (100, 150), (128, 96), (98, 40), (90, 50), (40, 70), (64, 40), (1, 33)]
SCRATCH = {"hsv_h": 0.015, "hsv_s": 0.7, "hsv_v": 0.4, "degrees": 0.0, "translate": 0.1, "scale": 0.5, "shear": 0.0,
           "perspective": 0.0, "flipud": 0.0, "fliplr": 0.5, "mosaic": 1.0, "mixup": 0.0, "copy_paste": 0.0}
CASES = [
    dict(name="mosaic", seed=1, hyp={}, indices=[0, 1, 2, 3, 4, 5, 6, 7]),
    dict(name="mosaic_half", seed=2, hyp=dict(mosaic=0.5), indices=[3, 0, 7, 1, 2, 6, 5, 4, 3, 3]),
    dict(name="letterbox", seed=3, hyp=dict(mosaic=0.0), indices=[0, 1, 2, 3, 4, 5, 6, 7]),
    dict(name="mixup", seed=4, hyp=dict(mixup=1.0), indices=[1, 5, 2, 0]),
    dict(name="warp_flips", seed=5, hyp=dict(mosaic=0.5, mixup=0.5, degrees=10.0, shear=5.0, perspective=0.0005,
                                             flipud=1.0, fliplr=1.0), indices=[0, 1, 2, 3, 4, 5, 6, 7]),
    dict(name="no_hsv_affine", seed=6, hyp=dict(mosaic=0.5, hsv_h=0.0, hsv_s=0.0, hsv_v=0.0, degrees=5.0),
         indices=[2, 3, 3, 7]),
]


def dataset(seed: int = 0):
    """The images (uint8 [h, w, 3], BGR) and upstream-style labels (float32 [n, 5] normalised cls, x, y, w, h)."""
    ims, labs = [], []
    rng = np.random.default_rng(seed + 77)
    for k, (h, w) in enumerate(SHAPES):
        ims.append(image(seed * 100 + k, h, w))
        n = k % 4
        xy = rng.uniform(0.2, 0.8, (n, 2))
        wh = rng.uniform(0.05, 0.6, (n, 2))
        cls = rng.integers(0, 80, (n, 1)).astype(np.float64)
        labs.append(np.concatenate([cls, xy, wh], 1).astype(np.float32))
    return ims, labs


def hyp(case):
    return dict(SCRATCH, **case["hyp"])


class DrawLog:
    """Records every value drawn from `random` and `np.random` inside the block, random.choices' picks and
    random.shuffle's permutations included."""

    def __enter__(self):
        self.values, self.kinds, self._saved = [], [], []
        for mod, names in ((random, ("random", "uniform", "randint", "choices")), (np.random, ("uniform", "beta"))):
            for n in names:
                f = getattr(mod, n)
                self._saved.append((mod, n, f))
                setattr(mod, n, self._wrap(f, f"{mod.__name__}.{n}"))
        f = random.shuffle
        self._saved.append((random, "shuffle", f))

        def shuffle(x, *a):
            f(x, *a)
            self._log(list(x), "random.shuffle")
        random.shuffle = shuffle
        return self

    def _log(self, v, kind):
        for x in np.ravel(np.asarray(v, np.float64)):
            self.values.append(float(x))
            self.kinds.append(kind)

    def _wrap(self, f, kind):
        def g(*a, **k):
            v = f(*a, **k)
            self._log(v, kind)
            return v
        return g

    def __exit__(self, *exc):
        for mod, n, f in self._saved:
            setattr(mod, n, f)


def generator_states():
    """random.getstate() and np.random.get_state() as arrays."""
    version, internal, gauss = random.getstate()
    st = np.random.get_state()
    return (np.array([version, *internal], np.int64), np.concatenate([st[1].astype(np.int64), [st[2]]]))


def plan(case, ims, labs, s=S):
    """The package's host draws for a case after its seeds: (samples, targets [n, 6] float32)."""
    from yolort_b200.v5.utils import datasets as D

    random.seed(case["seed"])
    np.random.seed(case["seed"])
    planner = D.Planner([im.shape[:2] for im in ims], labs, s, hyp(case))
    samples = [planner.sample(i) for i in case["indices"]]
    rows = []
    for n, smp in enumerate(samples):
        lab = np.zeros((len(smp.labels), 6), np.float32)
        lab[:, 1:] = smp.labels
        lab[:, 0] = n
        rows.append(lab)
    return samples, np.concatenate(rows, 0)


def restate(samples, ims, s=S, rgb=False):
    """oracle/restate_v5mosaic.py's pixels of a batch: uint8 [N, 3, s, s] RGB."""
    from oracle import restate_v5mosaic as R

    return np.stack([R.sample_pixels(smp, ims, s, rgb) for smp in samples])
