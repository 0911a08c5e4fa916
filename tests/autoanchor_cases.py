"""Seeded synthetic datasets for the AutoAnchor fixtures (oracle/make_golden_autoanchor.py) and tests: objects with
.shapes (float64 [M, 2], (w, h)) and .labels (float32 [n_i, 5], normalised (cls, x, y, w, h)), the attributes
yolort/v5/utils/autoanchor.py reads."""
import numpy as np


class Dataset:
    def __init__(self, shapes, labels):
        self.shapes, self.labels = shapes, labels


def make(seed: int, images: int, per_image: int, scale: float = 0.1, sigma: float = 0.6, tiny: int = 0) -> Dataset:
    """Log-normal box sizes around `scale` of the image side; `tiny` labels per image are 0.5 to 2.5 px wide."""
    rng = np.random.default_rng(seed)
    shapes = rng.integers(240, 1280, size=(images, 2)).astype(np.float64)
    labels = []
    for i in range(images):
        n = int(rng.integers(max(per_image // 2, 1), per_image + 1))
        wh = np.clip(scale * rng.lognormal(0.0, sigma, size=(n, 2)), 1e-4, 1.0)
        if tiny:
            wh[:tiny] = rng.uniform(0.5, 2.5, size=(min(tiny, n), 2)) / shapes[i].max()
        xy = rng.uniform(0.2, 0.8, size=(n, 2))
        cls = rng.integers(0, 80, size=(n, 1))
        labels.append(np.concatenate([cls, xy, wh], 1).astype(np.float32))
    return Dataset(shapes, labels)


def duplicated(seed: int, distinct: int, copies: int) -> Dataset:
    """Only `distinct` different label sizes: k-means with more codes empties clusters and returns fewer."""
    rng = np.random.default_rng(seed)
    wh = np.stack([rng.uniform(0.6, 0.9, distinct), rng.uniform(0.01, 0.02, distinct)], 1)   # far from every anchor
    lab = np.concatenate([np.zeros((distinct, 1)), np.full((distinct, 2), 0.5), wh], 1).astype(np.float32)
    return Dataset(np.full((copies, 2), 640.0), [lab.copy() for _ in range(copies)])


# name -> (dataset, call, kwargs, seed); call "check" runs check_anchors on a model with the P5 anchors.  The seeds of
# the cases that evolve were chosen so that every decision of the evolution is pinned (restate_autoanchor.decision_pinned;
# oracle/make_golden_autoanchor.py asserts it).
CASES = {
    "good_fit": (lambda: make(1, 60, 12, scale=0.08, sigma=0.5), "check", {"anchors": "p5"}, 11),
    "poor9": (lambda: make(2, 30, 20, scale=0.3, sigma=0.9), "kmean", {"n": 9, "gen": 1000}, 26),
    "poor12": (lambda: make(3, 30, 20, scale=0.25, sigma=0.9), "kmean", {"n": 12, "gen": 1000}, 25),
    "poor_check": (lambda: make(4, 30, 16, scale=0.3, sigma=1.2), "check", {"anchors": "p5"}, 22),   # BPR < 0.98
    "tiny": (lambda: make(5, 25, 16, scale=0.2, sigma=0.8, tiny=3), "kmean", {"n": 9, "gen": 300}, 22),
    "few_clusters": (lambda: duplicated(6, 5, 20), "check", {"anchors": "p5"}, 16),
    "few_points": (lambda: duplicated(7, 4, 1), "check", {"anchors": "p5"}, 17),
}

P5_STRIDES = [8, 16, 32]
P5_ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
