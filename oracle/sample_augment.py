"""Numpy restatement of the device parameter sampler of the training augmentations (`Compose.apply_batch(images,
targets, generator=g)`, csrc/augment_sample.cu), written from the rules below.  TEST INFRASTRUCTURE ONLY.

The sampler keeps the reference's transforms, parameter distributions and acceptance rules (yolort/data/transforms.py,
restated draw for draw in oracle/restate_augment.py) but draws from its own counter-based stream, so a batch is
reproducible from one key and every image can be sampled in parallel.

Rule 1 (generator).  Philox4x32-10 with curand's constants; key = the call's two 32-bit words; counter =
    (image index, transform index in the Compose, a, b).  Photometric distort: blocks (0, 0), (0, 1), (0, 2), words 0-6
    its seven decisions, 7-10 the brightness, contrast, saturation and hue factors, 11 the channel permutation.
    Zoom-out: block (0, 0) = apply, ratio, left, top.  Flip: block (0, 0) word 0.  IoU crop: block (round, 0xffffffff)
    word 0 the round's option, block (round, trial) the trial's width scale, height scale, left and top.
Rule 2 (words to numbers).  A uniform is (x >> 8) * 2^-24 in fp32 (exact, in [0, 1)); an integer in [0, n) is
    (x * n) >> 32 in 64 bits; the channel permutation is one of the 6 permutations of (0, 1, 2) in lexicographic order.
    A value drawn from a range (lo, hi) is fp32(lo) + u * fp32(hi - lo), the difference taken in double.  A transform
    with probability p applies when u < fp32(p).  The reference's randperm(4) inside a single-factor ColorJitter has no
    effect on the result and has no counterpart.
Rule 3 (geometry, the host sampler's fp32 operations in its order).  Zoom-out: canvas = int(fp32(w) * r), offsets
    int(fp32(canvas - w) * u); boxes + offset.  IoU crop: window = int(fp32(w) * r); the aspect test nw / nh in double;
    offsets int(fp32(w - nw) * u); a box is kept when its fp32 centre 0.5 * (x0 + x1) lies strictly inside the window;
    IoU = inter / ((area1 + area2) - inter) in fp32 (torchvision's box_iou), and a trial is accepted unless the largest
    IoU of its kept boxes, in double, is below the round's option; kept boxes are shifted, clamped to the window and
    kept in order.  Flip: x0' = fp32(w) - x1.
Rule 4 (IoU-crop rounds).  An option of 1.0 or more leaves the image as it is; otherwise the first accepted trial of
    the round in trial order wins, and a round without one is followed by the next.  After 1024 rounds the image's
    status is set (the call raises) and it is left uncropped.
"""
import itertools
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

F32 = np.float32
U64 = np.uint64
MASK = U64(0xFFFFFFFF)
M0, M1, W0, W1 = U64(0xD2511F53), U64(0xCD9E8D57), U64(0x9E3779B9), U64(0xBB67AE85)
ROUNDS = 1024
OPTION_BLOCK = 0xFFFFFFFF
ST_CROP_ROUNDS = 1
PERMS = list(itertools.permutations(range(3)))


# -- rules 1-2 -------------------------------------------------------------------------------------------------------
def philox(ctr, key) -> Tuple[np.ndarray, ...]:
    """Philox4x32-10 of the counters `ctr` (four broadcastable integer arrays) under `key` (two words): four uint32
    arrays."""
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, dtype=U64) & MASK for c in ctr))
    k0, k1 = U64(int(key[0]) & 0xFFFFFFFF), U64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = c0 * M0, c2 * M1
        c0, c1, c2, c3 = (p1 >> U64(32)) ^ c1 ^ k0, p1 & MASK, (p0 >> U64(32)) ^ c3 ^ k1, p0 & MASK
    return tuple(np.asarray(c, dtype=np.uint32) for c in (c0, c1, c2, c3))


def uniform(x):
    return (np.asarray(x, dtype=np.uint32) >> np.uint32(8)).astype(F32) * F32(2.0 ** -24)


def below(x, n: int):
    return (np.asarray(x, dtype=U64) * U64(n)) >> U64(32)


def from_range(lo: float, hi: float, x):
    return F32(lo) + uniform(x) * F32(hi - lo)


# -- the transforms ---------------------------------------------------------------------------------------------------
class _Image:
    def __init__(self, hw, boxes, labels):
        self.h, self.w = hw
        self.boxes = np.asarray(boxes, dtype=F32).reshape(-1, 4).copy()
        self.labels = np.asarray(labels, dtype=np.int64).reshape(-1).copy()
        self.recipe: List[tuple] = []
        self.status = 0
        self.crops: List[dict] = []        # what each accepted IoU crop saw (for invariant checks)


def _photometric(tr, key, i, t, im: _Image):
    x = np.concatenate([np.array(philox((i, t, 0, j), key), dtype=np.uint32) for j in range(3)])
    r = uniform(x[:7])
    p = F32(tr.p)

    def jitter(name, rng, word):
        if rng is not None:
            im.recipe.append((name, float(from_range(rng[0], rng[1], x[word]))))

    if r[0] < p:
        jitter("brightness", tr.brightness, 7)
    before = r[1] < F32(0.5)
    if before and r[2] < p:
        jitter("contrast", tr.contrast, 8)
    if r[3] < p:
        jitter("saturation", tr.saturation, 9)
    if r[4] < p:
        jitter("hue", tr.hue, 10)
    if not before and r[5] < p:
        jitter("contrast", tr.contrast, 8)
    if r[6] < p:
        im.recipe.append(("permute", PERMS[int(below(x[11], 6))]))


def _zoom_out(tr, key, i, t, im: _Image):
    x = philox((i, t, 0, 0), key)
    if not uniform(x[0]) < F32(tr.p):
        return
    r = from_range(tr.side_range[0], tr.side_range[1], x[1])
    cw, ch = int(F32(im.w) * r), int(F32(im.h) * r)
    left, top = int(F32(cw - im.w) * uniform(x[2])), int(F32(ch - im.h) * uniform(x[3]))
    fill = tuple(torch.tensor(tr.fill, dtype=torch.uint8).expand(3).tolist())
    im.recipe.append(("zoom", ch, cw, top, left, fill))
    im.boxes[:, 0::2] += F32(left)
    im.boxes[:, 1::2] += F32(top)
    im.h, im.w = ch, cw


def _hflip(tr, key, i, t, im: _Image):
    if uniform(philox((i, t, 0, 0), key)[0]) < F32(tr.p):
        im.recipe.append(("hflip",))
        x0 = im.boxes[:, 0].copy()
        im.boxes[:, 0] = F32(im.w) - im.boxes[:, 2]
        im.boxes[:, 2] = F32(im.w) - x0


def _inside(b: np.ndarray, l, t, r, btm):
    """[trials, boxes]: fp32 box centres strictly inside each window (l, t, r, btm as fp32 [trials, 1])."""
    cx, cy = F32(0.5) * (b[:, 0] + b[:, 2]), F32(0.5) * (b[:, 1] + b[:, 3])
    return (l < cx) & (cx < r) & (t < cy) & (cy < btm)


def _iou_crop(tr, key, i, t, im: _Image):
    opts = [float(o) for o in tr.options]
    trials = np.arange(int(tr.trials), dtype=U64)
    b = im.boxes
    for rnd in range(ROUNDS):
        jac = opts[int(below(philox((i, t, rnd, OPTION_BLOCK), key)[0], len(opts)))]
        if jac >= 1.0:
            return
        if not len(trials):
            continue
        x = philox((i, t, rnd, trials), key)
        nw = (F32(im.w) * from_range(tr.min_scale, tr.max_scale, x[0])).astype(np.int64)
        nh = (F32(im.h) * from_range(tr.min_scale, tr.max_scale, x[1])).astype(np.int64)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = nw.astype(np.float64) / nh.astype(np.float64)
        left = ((im.w - nw).astype(F32) * uniform(x[2])).astype(np.int64)
        top = ((im.h - nh).astype(F32) * uniform(x[3])).astype(np.int64)
        ok = (tr.min_aspect_ratio <= q) & (q <= tr.max_aspect_ratio) & (nw != 0) & (nh != 0)
        lf, tf = left.astype(F32)[:, None], top.astype(F32)[:, None]
        rf, bf = (left + nw).astype(F32)[:, None], (top + nh).astype(F32)[:, None]
        inside = _inside(b, lf, tf, rf, bf)
        area1 = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        area2 = (rf - lf) * (bf - tf)
        iw = np.maximum(np.minimum(b[:, 2], rf) - np.maximum(b[:, 0], lf), F32(0))
        ih = np.maximum(np.minimum(b[:, 3], bf) - np.maximum(b[:, 1], tf), F32(0))
        inter = iw * ih
        with np.errstate(divide="ignore", invalid="ignore"):
            iou = inter / ((area1 + area2) - inter)
        best = np.where(inside, iou, F32(-np.inf)).max(1, initial=F32(-np.inf))
        ok &= inside.any(1) & ~(best.astype(np.float64) < jac)
        if not ok.any():
            continue
        k = int(np.argmax(ok))
        keep = inside[k]
        kept = b[keep].copy()
        kept[:, 0::2] = np.minimum(np.maximum(kept[:, 0::2] - F32(left[k]), F32(0)), F32(nw[k]))
        kept[:, 1::2] = np.minimum(np.maximum(kept[:, 1::2] - F32(top[k]), F32(0)), F32(nh[k]))
        im.crops.append({"canvas": (im.h, im.w), "window": (int(top[k]), int(left[k]), int(nh[k]), int(nw[k])),
                         "option": jac, "boxes": b.copy(), "keep": keep})
        im.recipe.append(("crop", int(top[k]), int(left[k]), int(nh[k]), int(nw[k])))
        im.boxes, im.labels = kept, im.labels[keep]
        im.h, im.w = int(nh[k]), int(nw[k])
        return
    im.status |= ST_CROP_ROUNDS


_SAMPLERS = {"RandomPhotometricDistort": _photometric, "RandomZoomOut": _zoom_out, "RandomIoUCrop": _iou_crop,
             "RandomHorizontalFlip": _hflip, "PILToTensor": None, "ConvertImageDtype": None, "ToTensor": None}


def sample(transforms: Sequence, sizes: Sequence[Tuple[int, int]], targets: Sequence[Optional[dict]], key) -> List[dict]:
    """Every image of a batch through `transforms` (objects with the reference's class and attribute names) under the
    64-bit key `key` (two 32-bit words).  Per image: recipe (oracle/restate_augment.py notation, with ("float",) when a
    float conversion ends the list), hw, boxes fp32 [k, 4], labels int64 [k] (None without a target), status and the
    accepted IoU crops."""
    out = []
    float_out = False
    for tr in transforms:
        if type(tr).__name__ in ("ConvertImageDtype", "ToTensor"):
            float_out = tr.dtype == torch.float32
    for i, (hw, tg) in enumerate(zip(sizes, targets)):
        im = _Image(hw, np.zeros((0, 4)) if tg is None else tg["boxes"], np.zeros(0) if tg is None else tg["labels"])
        for t, tr in enumerate(transforms):
            fn = _SAMPLERS[type(tr).__name__]
            if fn is not None:
                fn(tr, key, i, t, im)
        if float_out:
            im.recipe.append(("float",))
        out.append({"recipe": im.recipe, "hw": (im.h, im.w), "boxes": None if tg is None else im.boxes,
                    "labels": None if tg is None else im.labels, "status": im.status, "crops": im.crops})
    return out
