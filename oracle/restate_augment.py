"""Numpy / torch-CPU restatement of the reference's training augmentations (yolort/data/transforms.py:21-336) on uint8
tensor images, written from the rules below and checked against torchvision's CPU tensor functions and against the
unmodified reference by tests/golden/augment.npz (oracle/make_golden_augment.py).  TEST INFRASTRUCTURE ONLY.

The parity target is torchvision's tensor arithmetic (torchvision/transforms/_functional_tensor.py), not PIL's.

Rule 1 (blend, _functional_tensor.py `_blend`).  out = trunc(clamp(fp32(r) * x + fp32(1.0 - r) * y, 0, 255)): the factor
    r is an fp32 value held as a Python double; `1.0 - r` is computed in double and rounded to fp32 when it meets the
    tensor; each product is rounded, then the sum; `.to(uint8)` truncates.
Rule 2 (grayscale, `rgb_to_grayscale`).  gray = trunc((0.2989 r + 0.587 g) + 0.114 b), each coefficient rounded to fp32,
    each product and sum rounded in fp32.
Rule 3 (brightness / saturation / contrast, `adjust_*`).  brightness blends with 0, saturation with gray, contrast with
    the fp32 mean of gray over the whole image: mean = fp32(sum) / fp32(n), where the integer sum is exact (torch's fp32
    sum equals it while it stays below 2^24).
Rule 4 (hue, `adjust_hue`, `_rgb2hsv`, `_hsv2rgb`).  x = byte / 255 (fp32 IEEE division); HSV as torchvision computes it,
    including h = fmod(h / 6 + 1, 1); h' = remainder(h + factor, 1) (torch's floating remainder: fmod, plus 1 when
    negative); i = floor(6 h'), f = 6 h' - i, p, q, t clamped to [0, 1]; back to bytes as trunc(x * fp32(255.999)).
Rule 5 (permutation, zoom-out, crop, flip).  Channel gather; a canvas of the fill value (uint8) with the image at
    (top, left); a window; a mirror of the columns.
Rule 6 (float output, `convert_image_dtype`).  byte / 255.0 in fp32 with IEEE division.
Rule 7 (parameters, transforms.py:59-336 and torchvision ColorJitter.get_params).  Drawn from torch's default CPU
    generator in the reference's order, with the reference's fp32 tensor arithmetic for sizes and offsets; boxes
    follow the reference's fp32 operations in its order.
"""
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torchvision

F32 = np.float32


# -- rules 1-4: colour -----------------------------------------------------------------------------------------------
def blend(x: np.ndarray, y, ratio: float) -> np.ndarray:
    r = F32(ratio)
    omr = F32(1.0 - float(ratio))
    v = r * x.astype(F32) + omr * np.asarray(y, dtype=F32)
    return np.clip(v, F32(0), F32(255)).astype(np.uint8)


def gray(x: np.ndarray) -> np.ndarray:
    r, g, b = (c.astype(F32) for c in x)
    return ((F32(0.2989) * r + F32(0.587) * g) + F32(0.114) * b).astype(np.uint8)


def gray_mean(x: np.ndarray) -> np.float32:
    gr = gray(x)
    return F32(int(gr.astype(np.int64).sum())) / F32(gr.size)


def brightness(x, f):
    return blend(x, F32(0), f)


def contrast(x, f):
    return blend(x, gray_mean(x), f)


def saturation(x, f):
    return blend(x, gray(x)[None], f)


def _remainder1(a: np.ndarray) -> np.ndarray:
    m = np.fmod(a, F32(1))
    return np.where(m < 0, m + F32(1), m).astype(F32)


def hue(x: np.ndarray, f: float) -> np.ndarray:
    v3 = x.astype(F32) / F32(255)
    r, g, b = v3
    maxc, minc = v3.max(0), v3.min(0)
    eqc = maxc == minc
    cr = maxc - minc
    s = cr / np.where(eqc, F32(1), maxc)
    crd = np.where(eqc, F32(1), cr)
    rc, gc, bc = (maxc - r) / crd, (maxc - g) / crd, (maxc - b) / crd
    h = np.where(maxc == r, bc - gc, np.where(maxc == g, (F32(2) + rc) - bc, (F32(4) + gc) - rc)).astype(F32)
    h = np.fmod(h / F32(6) + F32(1), F32(1))
    h = _remainder1(h + F32(f))
    h6 = h * F32(6)
    i = np.floor(h6)
    fr = h6 - i
    i = i.astype(np.int32) % 6
    v = maxc
    p = np.clip(v * (F32(1) - s), F32(0), F32(1))
    q = np.clip(v * (F32(1) - s * fr), F32(0), F32(1))
    t = np.clip(v * (F32(1) - s * (F32(1) - fr)), F32(0), F32(1))
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    out = np.empty_like(v3)
    for k, (a0, a1, a2) in enumerate(table):
        m = i == k
        out[0][m], out[1][m], out[2][m] = a0[m], a1[m], a2[m]
    return (out * F32(255.999)).astype(np.uint8)


# -- rule 5: geometry ------------------------------------------------------------------------------------------------
def permute(x, perm):
    return x[list(perm)]


def zoom_out(x, canvas_h, canvas_w, top, left, fill):
    out = np.empty((3, canvas_h, canvas_w), np.uint8)
    out[:] = np.asarray(fill, np.uint8).reshape(3, 1, 1)
    out[:, top:top + x.shape[1], left:left + x.shape[2]] = x
    return out


def crop(x, top, left, h, w):
    return x[:, top:top + h, left:left + w].copy()


def hflip(x):
    return x[:, :, ::-1].copy()


def to_float(x):
    return x.astype(F32) / F32(255)


# -- recipes ---------------------------------------------------------------------------------------------------------
# A recipe is the list of ops one image's transforms drew, in call order:
#   ("brightness" | "contrast" | "saturation" | "hue", factor), ("permute", (a, b, c)),
#   ("zoom", canvas_h, canvas_w, top, left, fill[3]), ("crop", top, left, h, w), ("hflip",), ("float",)
_OPS = {"brightness": brightness, "contrast": contrast, "saturation": saturation, "hue": hue, "permute": permute,
        "zoom": zoom_out, "crop": crop, "hflip": lambda x: hflip(x), "float": to_float}


def apply_recipe(x: np.ndarray, recipe) -> np.ndarray:
    for op in recipe:
        x = _OPS[op[0]](x, *op[1:])
    return x


# -- rule 7: the parameter sampler of default_train_transforms ----------------------------------------------------
def _jitter(lo, hi) -> float:
    torch.randperm(4)
    return float(torch.empty(1).uniform_(lo, hi))


def sample_photometric(recipe, p=0.5):
    r = torch.rand(7)
    if r[0] < p:
        recipe.append(("brightness", _jitter(0.875, 1.125)))
    before = r[1] < 0.5
    if before and r[2] < p:
        recipe.append(("contrast", _jitter(0.5, 1.5)))
    if r[3] < p:
        recipe.append(("saturation", _jitter(0.5, 1.5)))
    if r[4] < p:
        recipe.append(("hue", _jitter(-0.05, 0.05)))
    if not before and r[5] < p:
        recipe.append(("contrast", _jitter(0.5, 1.5)))
    if r[6] < p:
        recipe.append(("permute", tuple(torch.randperm(3).tolist())))


def sample_zoom_out(recipe, hw, boxes, fill=(0.0, 0.0, 0.0), side=(1.0, 4.0), p=0.5):
    if torch.rand(1) >= p:
        return hw, boxes
    h, w = hw
    r = side[0] + torch.rand(1) * (side[1] - side[0])
    cw, ch = int(w * r), int(h * r)
    r = torch.rand(2)
    left, top = int((cw - w) * r[0]), int((ch - h) * r[1])
    recipe.append(("zoom", ch, cw, top, left, tuple(torch.tensor(fill, dtype=torch.uint8).tolist())))
    boxes = boxes.clone()
    boxes[:, 0::2] += left
    boxes[:, 1::2] += top
    return (ch, cw), boxes


def sample_iou_crop(recipe, hw, boxes, labels, options=(0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 1.0), trials=40):
    h, w = hw
    while True:
        jac = options[int(torch.randint(low=0, high=len(options), size=(1,)))]
        if jac >= 1.0:
            return hw, boxes, labels
        for _ in range(trials):
            r = 0.3 + (1.0 - 0.3) * torch.rand(2)
            nw, nh = int(w * r[0]), int(h * r[1])
            if not 0.5 <= nw / nh <= 2.0:
                continue
            r = torch.rand(2)
            left, top = int((w - nw) * r[0]), int((h - nh) * r[1])
            if nw == 0 or nh == 0:
                continue
            cx = 0.5 * (boxes[:, 0] + boxes[:, 2])
            cy = 0.5 * (boxes[:, 1] + boxes[:, 3])
            keep = (left < cx) & (cx < left + nw) & (top < cy) & (cy < top + nh)
            if not keep.any():
                continue
            kept = boxes[keep]
            win = torch.tensor([[left, top, left + nw, top + nh]], dtype=kept.dtype)
            if torchvision.ops.box_iou(kept, win).max() < jac:
                continue
            kept[:, 0::2] -= left
            kept[:, 1::2] -= top
            kept[:, 0::2].clamp_(min=0, max=nw)
            kept[:, 1::2].clamp_(min=0, max=nh)
            recipe.append(("crop", top, left, nh, nw))
            return (nh, nw), kept, labels[keep]


def sample_hflip(recipe, hw, boxes, p=0.5):
    if torch.rand(1) < p:
        recipe.append(("hflip",))
        boxes = boxes.clone()
        boxes[:, [0, 2]] = hw[1] - boxes[:, [2, 0]]
    return boxes


def sample_default(hw: Tuple[int, int], boxes: torch.Tensor, labels: torch.Tensor, hflip_prob: float = 0.5):
    """One image through default_train_transforms(hflip_prob): (recipe, boxes, labels), boxes in fp32 on the host."""
    recipe: List[tuple] = []
    sample_photometric(recipe)
    hw, boxes = sample_zoom_out(recipe, hw, boxes)
    hw, boxes, labels = sample_iou_crop(recipe, hw, boxes, labels)
    boxes = sample_hflip(recipe, hw, boxes, hflip_prob)
    recipe.append(("float",))
    return recipe, boxes, labels


def normalize_targets(targets: List[Dict[str, torch.Tensor]], sizes: List[Tuple[int, int]]) -> torch.Tensor:
    """YOLOTransform's target batch (yolort/models/transform.py:205-219, :232-250, :370-381): boxes divided by the
    pre-resize (h, w) in fp32, xyxy to cxcywh, rows (image, label, cx, cy, w, h)."""
    rows = []
    for i, (t, (h, w)) in enumerate(zip(targets, sizes)):
        b = t["boxes"].to(torch.float32)
        th, tw = torch.tensor(h, dtype=torch.float32), torch.tensor(w, dtype=torch.float32)
        x0, y0 = b[:, 0] / tw, b[:, 1] / th
        x1, y1 = b[:, 2] / tw, b[:, 3] / th
        cx, cy = (x0 + x1) / 2, (y0 + y1) / 2
        r = torch.stack([torch.full_like(cx, i), t["labels"].to(torch.float32), cx, cy, x1 - x0, y1 - y0], 1)
        rows.append(r)
    return torch.cat(rows) if rows else torch.zeros((0, 6))


def digest(a: np.ndarray) -> str:
    import hashlib

    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
