"""YOLOv5's AutoAnchor (yolort/v5/utils/autoanchor.py:18-174) on the GPU.

The host makes every random draw in the reference's order -- check_anchors' scale draw, k-means' 30 starting books
(scipy's _kpoints on numpy's global RandomState) and the table of `gen` mutation vectors -- and builds the label sizes
with the reference's numpy expressions.  The device computes the ratio metric, the 30 k-means trials at once and all
generations of the evolution in one cooperative launch (csrc/autoanchor.cu).  After `random.seed(s); np.random.seed(s)`
the anchors and both generators' states equal the reference's (DESIGN.md, "AutoAnchor", states where the fitness of a
generation may differ from the reference's own float32 sum).
"""
import logging
import math
import random
from typing import List, Tuple

import numpy as np
import torch

from ... import _C

LOGGER = logging.getLogger(__name__)
PREFIX = "\033[34m\033[1mAutoAnchor: \033[0m"       # colorstr("AutoAnchor: ")
KMEANS_TRIALS = 30                                    # kmeans(wh / s, n, iter=30)


def _yolo(model):
    """The YOLO that owns the anchors of `model`: a YOLO, a YOLOv5 (its .model) or a wrapper with .module."""
    from ...models.yolo import YOLO

    m = model.module if hasattr(model, "module") else model
    m = getattr(m, "model", m)
    if not isinstance(m, YOLO):
        raise TypeError(f"expected a YOLO or YOLOv5 model (or a wrapper with .module), got {type(model).__name__}")
    return m


def _device():
    if not torch.cuda.is_available():
        raise _C.NativeLibraryError("AutoAnchor runs on sm_90a GPUs only (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _strides_units(m) -> Tuple[np.ndarray, np.ndarray]:
    """(anchors in stride units [nl, na, 2] as upstream's Detect holds them, strides [nl]), float32."""
    ag = m.anchor_generator
    strides = np.array(ag.strides, dtype=np.float32)
    a = np.array(ag.anchor_grids, dtype=np.float32).reshape(ag.num_layers, ag.num_anchors, 2)
    return a / strides[:, None, None], strides


def check_anchor_order(model) -> None:
    """Reverse the anchors' level order when their area order differs from the stride order (autoanchor.py:18-28)."""
    m = _yolo(model)
    su, strides = _strides_units(m)
    a = su.prod(-1).reshape(-1)
    da = a[-1] - a[0]
    ds = strides[-1] - strides[0]
    if np.sign(da) != np.sign(ds):
        LOGGER.info(f"{PREFIX}Reversing anchor order")
        flipped = su[::-1] * strides[:, None, None]         # float32: exact for power-of-two strides
        m.set_anchor_grids(flipped.reshape(len(strides), -1).tolist())


def _check_dataset(dataset) -> Tuple[np.ndarray, List[np.ndarray]]:
    if isinstance(dataset, str):
        raise NotImplementedError("kmean_anchors(dataset=<yaml path>) needs a dataset loader, which yolort_b200 has "
                                  "not; pass an object with .shapes and .labels")
    shapes, labels = getattr(dataset, "shapes", None), getattr(dataset, "labels", None)
    if not isinstance(shapes, np.ndarray) or shapes.dtype != np.float64 or shapes.ndim != 2 or shapes.shape[1] != 2:
        raise ValueError("dataset.shapes must be a float64 ndarray [M, 2] of (w, h)")
    if not np.isfinite(shapes).all() or (shapes <= 0).any():
        raise ValueError("dataset.shapes must be positive and finite")
    labels = list(labels) if labels is not None else None
    if labels is None or len(labels) != shapes.shape[0]:
        raise ValueError("dataset.labels must be a list of one array per image (len(labels) == len(shapes))")
    for i, l in enumerate(labels):
        if not isinstance(l, np.ndarray) or l.dtype != np.float32 or l.ndim != 2 or l.shape[1] != 5:
            raise ValueError(f"dataset.labels[{i}] must be a float32 ndarray [n, 5] of (cls, x, y, w, h)")
        if not np.isfinite(l).all() or (l[:, 3:5] < 0).any():
            raise ValueError(f"dataset.labels[{i}] has negative or non-finite sizes")
    return shapes, labels


def _check_thr(thr) -> float:
    thr = float(thr)
    if not math.isfinite(thr) or thr <= 0.0:
        raise ValueError(f"thr must be positive and finite (the metric compares with 1 / thr), got {thr}")
    return thr


def _metric(wh32: torch.Tensor, k: np.ndarray, thr: float, f64: bool):
    counts, sums = _C.anchor_metric(wh32, torch.from_numpy(np.ascontiguousarray(k, dtype=np.float64)), thr, f64)
    c, s = counts.tolist(), sums.tolist()
    return (c[0], c[1], s[0], s[1], s[2])


def _results(k: np.ndarray, wh0: torch.Tensor, thr: float, n: int, img_size: int, verbose: bool) -> np.ndarray:
    """print_results (autoanchor.py:107-122): k sorted small to large, the float64 metric of wh0 logged."""
    k = k[np.argsort(k.prod(1))]
    if verbose:
        n_best, n_x, s_x, s_best, s_past = _metric(wh0, k, thr, True)
        m = int(wh0.shape[0])
        bpr = np.float32(np.float32(n_best) / np.float32(m))
        aat = np.float32(np.float32(np.float32(n_x) / np.float32(m * n)) * np.float32(n))
        past = s_past / n_x if n_x else float("nan")
        s = (f"{PREFIX}thr={thr:.2f}: {float(bpr):.4f} best possible recall, {float(aat):.2f} anchors past thr\n"
             f"{PREFIX}n={n}, img_size={img_size}, metric_all={s_x / (m * n):.3f}/{s_best / m:.3f}-mean/best, "
             f"past_thr={past:.3f}-mean: ")
        for x in k:
            s += "%i,%i, " % (round(x[0]), round(x[1]))
        LOGGER.info(s[:-2])
    return k


def draw_mutations(n: int, gen: int, mp: float = 0.9, s: float = 0.1) -> np.ndarray:
    """The `gen` mutation vectors of autoanchor.py:163-165, drawn in the reference's order: npr.random, random.random,
    npr.randn, redrawn while all ones; float64 [gen, n, 2]."""
    npr = np.random
    sh = (n, 2)
    out = np.empty((gen, n, 2))
    for g in range(gen):
        v = np.ones(sh)
        while (v == 1).all():
            v = ((npr.random(sh) < mp) * random.random() * npr.randn(*sh) * s + 1).clip(0.3, 3.0)
        out[g] = v
    return out


def kmeans_device(obs: np.ndarray, n: int, trials: int = KMEANS_TRIALS) -> Tuple[np.ndarray, float]:
    """scipy.cluster.vq.kmeans(obs, n, iter=trials) on the device, bit for bit: the starting books are drawn here from
    numpy's global RandomState (choice(len(obs), n, replace=False) per trial), the trials run at once, the best is
    taken by strict < in trial order."""
    if not np.isfinite(obs).all():
        raise ValueError("array must not contain infs or NaNs")          # scipy's check_finite
    idx = np.stack([np.random.choice(obs.shape[0], size=int(n), replace=False) for _ in range(trials)])
    if n > _C.YB_AA_MAX_ANCHORS:
        raise ValueError(f"at most {_C.YB_AA_MAX_ANCHORS} anchors, got {n}")
    dev = _device()
    d_obs = torch.from_numpy(np.ascontiguousarray(obs)).to(dev)
    books, sizes, dist, _ = _C.kmeans(d_obs, d_obs[torch.from_numpy(idx).to(dev)])
    books, sizes, dist = books.cpu().numpy(), sizes.cpu().tolist(), dist.cpu().numpy()
    best, best_dist = None, math.inf
    for t in range(trials):
        if dist[t] < best_dist:
            best, best_dist = books[t, :sizes[t]].copy(), float(dist[t])
    return best, best_dist


def evolve_anchors(wh: torch.Tensor, k: np.ndarray, v: np.ndarray, thr: float):
    """kmean_anchors' genetic evolution (autoanchor.py:157-171) on the device for the float32 label sizes wh [N, 2]
    (on the device), the starting anchors k and the mutation table v; thr is the ratio 1 / hyp['anchor_t'].
    Returns (k, fitness float32 [gen + 1] after each generation, accepted generations).  With thr >= 1 no ratio
    (at most 1) passes it: every fitness is 0 and no generation is kept, as in the reference."""
    if thr >= 1.0:
        return k.copy(), np.zeros(v.shape[0] + 1, dtype=np.float32), []
    e = math.floor(math.log2(np.float32(thr))) - 23
    if int(wh.shape[0]) >= 2 ** (63 + e):
        raise ValueError(f"{int(wh.shape[0])} labels overflow the exact fitness sum at thr={thr}")
    kk, fit, acc = _C.anchor_evolve(wh, torch.from_numpy(k), torch.from_numpy(v), thr, e)
    return kk.cpu().numpy(), fit.cpu().numpy(), np.nonzero(acc.cpu().numpy())[0].tolist()


def kmean_anchors(dataset="./data/coco128.yaml", n=9, img_size=640, thr=4.0, gen=1000, verbose=True):
    """Creates kmeans-evolved anchors from a loaded dataset (.shapes float64 [M, 2], .labels float32 [n_i, 5] each).
    Returns the float64 [n, 2] anchors sorted small to large, as the reference does (autoanchor.py:74-174)."""
    shapes, labels = _check_dataset(dataset)
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not 1 <= n <= _C.YB_AA_MAX_ANCHORS:
        raise ValueError(f"n must be an integer in [1, {_C.YB_AA_MAX_ANCHORS}], got {n!r}")
    if isinstance(gen, bool) or not isinstance(gen, (int, np.integer)) or gen < 0:
        raise ValueError(f"gen must be a non-negative integer, got {gen!r}")
    thr = 1 / _check_thr(thr)
    n, gen = int(n), int(gen)

    shapes = img_size * shapes / shapes.max(1, keepdims=True)
    wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, labels)])
    i = (wh0 < 3.0).any(1).sum()
    if i:
        LOGGER.info(f"{PREFIX}WARNING: Extremely small objects found. {i} of {len(wh0)} labels are < 3 pixels in size.")
    wh = wh0[(wh0 >= 2.0).any(1)]
    LOGGER.info(f"{PREFIX}Running kmeans for {n} anchors on {len(wh)} points...")
    s = wh.std(0)
    k, _ = kmeans_device(wh / s, n)
    assert len(k) == n, f"{PREFIX}ERROR: scipy.cluster.vq.kmeans requested {n} points but returned only {len(k)}"
    k *= s
    dev = _device()
    wh_d = torch.from_numpy(wh.astype(np.float32)).to(dev)
    wh0_d = torch.from_numpy(wh0.astype(np.float32)).to(dev)
    k = _results(k, wh0_d, thr, n, img_size, verbose=False)

    v = draw_mutations(n, gen)
    k_end, fit, acc = evolve_anchors(wh_d, k, v, thr)
    kc = k
    for g in acc:                    # the accepted anchors, replayed on the host with the device's decisions
        kc = (kc.copy() * v[g]).clip(min=2.0)
        LOGGER.debug(f"{PREFIX}generation {g}: fitness = {float(fit[g + 1]):.4f}")
        if verbose:
            _results(kc, wh0_d, thr, n, img_size, verbose)
    assert np.array_equal(kc, k_end)
    return _results(k_end, wh0_d, thr, n, img_size, verbose=True)


def check_anchors(dataset, model, thr=4.0, imgsz=640) -> None:
    """Check the anchors' fit to the data and replace them with kmean_anchors' when that raises the best possible
    recall (autoanchor.py:31-71).  The model's anchors change through YOLO.set_anchor_grids only."""
    m = _yolo(model)
    shapes, labels = _check_dataset(dataset)
    thr = _check_thr(thr)
    shapes = imgsz * shapes / shapes.max(1, keepdims=True)
    scale = np.random.uniform(0.9, 1.1, size=(shapes.shape[0], 1))
    wh = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes * scale, labels)]).astype(np.float32)
    if wh.shape[0] == 0:
        raise ValueError("the dataset has no labels")
    dev = _device()
    wh_d = torch.from_numpy(wh).to(dev)
    n_wh = wh.shape[0]

    current = np.array(m.anchor_generator.anchors_px(), dtype=np.float32).reshape(-1, 2)
    n_best, n_x, *_ = _metric(wh_d, current, 1 / thr, False)
    bpr = np.float32(np.float32(n_best) / np.float32(n_wh))
    aat = np.float32(np.float32(n_x) / np.float32(n_wh))
    s = f"\n{PREFIX}{float(aat):.2f} anchors/target, {float(bpr):.3f} Best Possible Recall (BPR). "
    if bpr > np.float32(0.98):
        LOGGER.info(f"{s}Current anchors are a good fit to dataset ✅")
        return
    LOGGER.info(f"{s}Anchors are a poor fit to dataset ⚠️, attempting to improve...")
    na = current.shape[0]
    anchors = None
    try:
        anchors = kmean_anchors(dataset, n=na, img_size=imgsz, thr=thr, gen=1000, verbose=False)
    except Exception as e:
        LOGGER.info(f"{PREFIX}ERROR: {e}")
    new_bpr = bpr
    if anchors is not None:
        nb = _metric(wh_d, anchors, 1 / thr, True)[0]
        new_bpr = np.float32(np.float32(nb) / np.float32(n_wh))
    if new_bpr > bpr:
        k32 = anchors.astype(np.float32).reshape(m.anchor_generator.num_layers, -1)
        m.set_anchor_grids(k32.tolist())
        check_anchor_order(m)
        LOGGER.info(f"{PREFIX}New anchors saved to model. Update model *.yaml to use these anchors in the future.")
    else:
        LOGGER.info(f"{PREFIX}Original anchors better than new anchors. Proceeding with original anchors.")
