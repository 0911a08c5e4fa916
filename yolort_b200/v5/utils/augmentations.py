"""YOLOv5's own augmentations (yolort/v5/utils/augmentations.py:53-324) on the GPU.

Same names, signatures, defaults and return values as the reference: `augment_hsv`, `random_perspective`,
`box_candidates`, `mixup`, `cutout`.  Images are CUDA uint8 [H, W, 3] tensors (cv2's layout, any strides: the HWC
views `yolort_b200.io.decode_jpeg` returns go straight in); labels stay numpy [n, 5] arrays of (cls, x1, y1, x2, y2) in
pixels.  A numpy or PIL image raises TypeError, a CPU tensor NativeLibraryError, a wrong dtype or rank ValueError,
non-empty `segments` NotImplementedError.

Every parameter is drawn on the host from Python's `random` and numpy's global generator in the reference's order, so
after `random.seed(s); np.random.seed(s)` the draws, and the pixels and boxes, are the reference's.  Box arithmetic
runs on the host in the reference's own numpy expressions.  The pixels are csrc/v5_augment.cu's: OpenCV 4.x's
fixed-point warpAffine / warpPerspective (border 114), its BGR<->HSV conversions and the gains' LUTs, bit for bit
(oracle/restate_v5aug.py states each step; HSV->BGR follows the row split of OpenCV's x86 AVX2 build).

`apply_batch(images, targets, hyp)` runs YOLOv5's non-mosaic training recipe on a batch in one launch: per image
random_perspective -> augment_hsv -> flipud -> fliplr with the keys of hyp.scratch.yaml.
"""
import math
import random
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from ... import _C

__all__ = ["augment_hsv", "random_perspective", "box_candidates", "bbox_ioa", "mixup", "cutout", "apply_batch",
           "letterbox", "HYP_SCRATCH"]

# yolort/v5/data/hyps/hyp.scratch.yaml: the augmentation keys
HYP_SCRATCH = {"hsv_h": 0.015, "hsv_s": 0.7, "hsv_v": 0.4, "degrees": 0.0, "translate": 0.1, "scale": 0.5,
               "shear": 0.0, "perspective": 0.0, "flipud": 0.0, "fliplr": 0.5, "mixup": 0.0}
_HSV = _C.YB_V5_TO_HSV | _C.YB_V5_LUT | _C.YB_V5_FROM_HSV


def _check_image(im, what: str) -> None:
    if not isinstance(im, Tensor):
        raise TypeError(f"{what}: images must be uint8 [H, W, 3] CUDA tensors, got {type(im).__name__} (decode to a "
                        "tensor, e.g. with yolort_b200.io.decode_jpeg)")
    if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
        raise ValueError(f"{what}: images must be uint8 [H, W, 3] tensors, got {im.dtype} {tuple(im.shape)}")
    _C.require_cuda(im, what)


class _Plan:
    """One image's draws as the kernel takes them: output size, inverse map, LUT, flips, cutout rectangles."""

    def __init__(self, h: int, w: int):
        self.out_h, self.out_w = h, w
        self.inv: Optional[np.ndarray] = None
        self.perspective = False
        self.lut: Optional[np.ndarray] = None
        self.flip_ud = self.flip_lr = False
        self.rects: List[tuple] = []

    def ops(self, rgb: bool) -> int:
        ops = _C.YB_V5_RGB if rgb else 0
        if self.inv is not None:
            ops |= _C.YB_V5_PERSPECTIVE if self.perspective else _C.YB_V5_AFFINE
        if self.lut is not None:
            ops |= _HSV
        if self.flip_ud:
            ops |= _C.YB_V5_FLIP_UD
        if self.flip_lr:
            ops |= _C.YB_V5_FLIP_LR
        return ops


def _fill(d: "_C.V5Image", src: Tensor, dst: Tensor, plan: _Plan, rgb: bool) -> None:
    d.src, d.dst = src.data_ptr(), dst.data_ptr()
    d.src_stride_y, d.src_stride_x, d.src_stride_c = (int(v) for v in src.stride())
    d.dst_stride_y, d.dst_stride_x, d.dst_stride_c = (int(v) for v in dst.stride())
    d.src_h, d.src_w = int(src.shape[0]), int(src.shape[1])
    d.out_h, d.out_w = plan.out_h, plan.out_w
    d.ops = plan.ops(rgb)
    if plan.inv is not None:
        for j, v in enumerate(plan.inv):
            d.inv[j] = float(v)
    if plan.lut is not None:
        ctypes_lut = np.ctypeslib.as_array(d.lut)
        ctypes_lut[...] = plan.lut
    if len(plan.rects) > _C.YB_V5_MAX_RECTS:
        raise NotImplementedError(f"{len(plan.rects)} cutout rectangles (at most {_C.YB_V5_MAX_RECTS})")
    d.n_rects = len(plan.rects)
    for j, (y0, x0, y1, x1, c) in enumerate(plan.rects):
        d.rects[j][0], d.rects[j][1], d.rects[j][2], d.rects[j][3] = y0, x0, y1, x1
        d.rect_color[j] = int(c[0]) | (int(c[1]) << 8) | (int(c[2]) << 16)


def _run_one(src: Tensor, dst: Tensor, plan: _Plan, rgb: bool = False) -> None:
    descs = (_C.V5Image * 1)()
    _fill(descs[0], src, dst, plan, rgb)
    _C.v5_augment(descs, [src, dst], src.device)


# -- draws (the reference's expressions and order) -----------------------------------------------------------------
def _hsv_draw(hgain, sgain, vgain) -> Optional[np.ndarray]:
    """augment_hsv's gains and LUTs ([3, 256] uint8), or None when every gain is zero (nothing is drawn)."""
    if not (hgain or sgain or vgain):
        return None
    r = np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1  # random gains
    x = np.arange(0, 256, dtype=r.dtype)
    lut_hue = ((x * r[0]) % 180).astype(np.uint8)
    lut_sat = np.clip(x * r[1], 0, 255).astype(np.uint8)
    lut_val = np.clip(x * r[2], 0, 255).astype(np.uint8)
    return np.stack([lut_hue, lut_sat, lut_val])


def _rotation_matrix_2d(angle: float, scale: float) -> np.ndarray:
    """cv2.getRotationMatrix2D(angle=angle, center=(0, 0), scale=scale)."""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    return np.array([[alpha, beta, (1 - alpha) * 0.0 - beta * 0.0], [-beta, alpha, beta * 0.0 + (1 - alpha) * 0.0]])


def _perspective_draw(shape, degrees, translate, scale, shear, perspective, border):
    """random_perspective's draws: (M, s, height, width)."""
    height = shape[0] + border[0] * 2  # shape(h,w,c)
    width = shape[1] + border[1] * 2
    C = np.eye(3)
    C[0, 2] = -shape[1] / 2  # x translation (pixels)
    C[1, 2] = -shape[0] / 2  # y translation (pixels)
    P = np.eye(3)
    P[2, 0] = random.uniform(-perspective, perspective)  # x perspective (about y)
    P[2, 1] = random.uniform(-perspective, perspective)  # y perspective (about x)
    R = np.eye(3)
    a = random.uniform(-degrees, degrees)
    s = random.uniform(1 - scale, 1 + scale)
    R[:2] = _rotation_matrix_2d(a, s)
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-shear, shear) * math.pi / 180)  # x shear (deg)
    S[1, 0] = math.tan(random.uniform(-shear, shear) * math.pi / 180)  # y shear (deg)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - translate, 0.5 + translate) * width  # x translation (pixels)
    T[1, 2] = random.uniform(0.5 - translate, 0.5 + translate) * height  # y translation (pixels)
    M = T @ S @ R @ P @ C  # order of operations (right to left) is IMPORTANT
    return M, s, height, width


def _invert_affine(M) -> np.ndarray:
    """cv2.warpAffine's inverse of the 2x3 map M[:2] (invertAffineTransform's arithmetic): 6 doubles."""
    m = [float(v) for v in M[:2].reshape(-1)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m[4] * D, m[0] * D
    m[0], m[1], m[3], m[4] = a11, m[1] * -D, m[3] * -D, a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    return np.array([m[0], m[1], b1, m[3], m[4], b2])


def _invert_perspective(M) -> np.ndarray:
    """cv2.warpPerspective's inverse of M: cv::invert(DECOMP_LU)'s closed form for 3x3 doubles, 9 doubles."""
    s = [[float(v) for v in row] for row in M]
    d = (s[0][0] * (s[1][1] * s[2][2] - s[1][2] * s[2][1]) - s[0][1] * (s[1][0] * s[2][2] - s[1][2] * s[2][0]) +
         s[0][2] * (s[1][0] * s[2][1] - s[1][1] * s[2][0]))
    if d == 0.0:
        return np.zeros(9)
    d = 1.0 / d
    return np.array([(s[1][1] * s[2][2] - s[1][2] * s[2][1]) * d, (s[0][2] * s[2][1] - s[0][1] * s[2][2]) * d,
                     (s[0][1] * s[1][2] - s[0][2] * s[1][1]) * d, (s[1][2] * s[2][0] - s[1][0] * s[2][2]) * d,
                     (s[0][0] * s[2][2] - s[0][2] * s[2][0]) * d, (s[0][2] * s[1][0] - s[0][0] * s[1][2]) * d,
                     (s[1][0] * s[2][1] - s[1][1] * s[2][0]) * d, (s[0][1] * s[2][0] - s[0][0] * s[2][1]) * d,
                     (s[0][0] * s[1][1] - s[0][1] * s[1][0]) * d])


def _warp_plan(plan: _Plan, M, border, perspective) -> None:
    """Sets the plan's warp when random_perspective changes the image (it returns the input otherwise)."""
    if (border[0] != 0) or (border[1] != 0) or (M != np.eye(3)).any():  # image changed
        plan.perspective = bool(perspective)
        plan.inv = _invert_perspective(M) if perspective else _invert_affine(M)


def _warp_targets(targets, M, s, width, height, perspective):
    """random_perspective's box arithmetic, the reference's expressions."""
    n = len(targets)
    if n:
        xy = np.ones((n * 4, 3))
        xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)  # x1y1, x2y2, x1y2, x2y1
        xy = xy @ M.T  # transform
        xy = (xy[:, :2] / xy[:, 2:3] if perspective else xy[:, :2]).reshape(n, 8)  # perspective rescale or affine
        x = xy[:, [0, 2, 4, 6]]
        y = xy[:, [1, 3, 5, 7]]
        new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
        new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
        new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
        i = box_candidates(box1=targets[:, 1:5].T * s, box2=new.T, area_thr=0.10)
        targets = targets[i]
        targets[:, 1:5] = new[i]
    return targets


# -- the reference's functions ------------------------------------------------------------------------------------
def augment_hsv(im, hgain=0.5, sgain=0.5, vgain=0.5):
    """HSV colour-space augmentation of the BGR image `im`, in place (cv2's COLOR_BGR2HSV, LUT, COLOR_HSV2BGR)."""
    _check_image(im, "augment_hsv")
    lut = _hsv_draw(hgain, sgain, vgain)
    if lut is not None:
        plan = _Plan(int(im.shape[0]), int(im.shape[1]))
        plan.lut = lut
        _run_one(im, im, plan)


def random_perspective(im, targets=(), segments=(), degrees=10, translate=0.1, scale=0.1, shear=10,
                       perspective=0.0, border=(0, 0)):
    """Rotation, scale, shear, translation and perspective (cv2.warpAffine / warpPerspective, border 114) of `im`,
    and of the [n, 5] (cls, xyxy) `targets`; returns (im, targets).  `im` itself comes back when the map is the
    identity and there is no border."""
    if any(np.asarray(x).any() for x in segments):
        raise NotImplementedError("random_perspective: segments are not supported on the GPU")
    _check_image(im, "random_perspective")
    M, s, height, width = _perspective_draw(im.shape, degrees, translate, scale, shear, perspective, border)
    plan = _Plan(height, width)
    _warp_plan(plan, M, border, perspective)
    if plan.inv is not None:
        if height <= 0 or width <= 0:
            raise ValueError(f"random_perspective: border {tuple(border)} leaves no output pixel")
        out = torch.empty((height, width, 3), dtype=torch.uint8, device=im.device)
        _run_one(im, out, plan)
        im = out
    return im, _warp_targets(targets, M, s, width, height, perspective)


def _cutout_draw(h: int, w: int, labels, p):
    """cutout's draws: the rectangles (y0, x0, y1, x1, colour) in order (None when it does not apply) and the kept
    labels."""
    if not random.random() < p:
        return None, labels
    rects = []
    scales = [0.5] * 1 + [0.25] * 2 + [0.125] * 4 + [0.0625] * 8 + [0.03125] * 16  # image size fraction
    for s in scales:
        mask_h = random.randint(1, int(h * s))  # create random masks
        mask_w = random.randint(1, int(w * s))
        xmin = max(0, random.randint(0, w) - mask_w // 2)
        ymin = max(0, random.randint(0, h) - mask_h // 2)
        xmax = min(w, xmin + mask_w)
        ymax = min(h, ymin + mask_h)
        rects.append((ymin, xmin, ymax, xmax, [random.randint(64, 191) for _ in range(3)]))
        if len(labels) and s > 0.03:
            box = np.array([xmin, ymin, xmax, ymax], dtype=np.float32)
            ioa = bbox_ioa(box, labels[:, 1:5])  # intersection over area
            labels = labels[ioa < 0.60]  # remove >60% obscured labels
    return rects, labels


def cutout(im, labels, p=0.5):
    """Cutout (https://arxiv.org/abs/1708.04552): 31 random-colour rectangles written into `im` in place, the last
    one over a pixel setting it; returns the labels less than 60 % obscured."""
    _check_image(im, "cutout")
    h, w = int(im.shape[0]), int(im.shape[1])
    rects, labels = _cutout_draw(h, w, labels, p)
    if rects is not None:
        plan = _Plan(h, w)
        plan.rects = rects
        _run_one(im, im, plan)
    return labels


def mixup(im, labels, im2, labels2):
    """MixUp (https://arxiv.org/pdf/1710.09412.pdf): returns (uint8(im * r + im2 * (1 - r)), both label sets)."""
    _check_image(im, "mixup")
    _check_image(im2, "mixup")
    if im.shape != im2.shape or im.device != im2.device:
        raise ValueError(f"mixup: images of {tuple(im.shape)} on {im.device} and {tuple(im2.shape)} on {im2.device}")
    r = np.random.beta(32.0, 32.0)  # mixup ratio, alpha=beta=32.0
    im = _C.v5_mixup(im.contiguous(), im2.contiguous(), r)
    labels = np.concatenate((labels, labels2), 0)
    return im, labels


def box_candidates(box1, box2, wh_thr=2, ar_thr=20, area_thr=0.1, eps=1e-16):  # box1(4,n), box2(4,n)
    # Compute candidate boxes: box1 before augment, box2 after augment, wh_thr (pixels), aspect_ratio_thr, area_ratio
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))  # aspect ratio
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)  # candidates


def bbox_ioa(box1, box2, eps=1e-7):
    """Intersection over box2's area of box1 (4,) and box2 (n, 4), xyxy (yolort/v5/utils/metrics.py)."""
    box2 = box2.transpose()
    b1_x1, b1_y1, b1_x2, b1_y2 = box1[0], box1[1], box1[2], box1[3]
    b2_x1, b2_y1, b2_x2, b2_y2 = box2[0], box2[1], box2[2], box2[3]
    inter_area = (np.minimum(b1_x2, b2_x2) - np.maximum(b1_x1, b2_x1)).clip(0) * (
        np.minimum(b1_y2, b2_y2) - np.maximum(b1_y1, b2_y1)
    ).clip(0)
    box2_area = (b2_x2 - b2_x1) * (b2_y2 - b2_y1) + eps
    return inter_area / box2_area


# -- the batch ----------------------------------------------------------------------------------------------------
def plan_batch(sizes, targets, hyp: Dict[str, float]):
    """Draws every image's parameters in turn (random_perspective, augment_hsv, flipud, fliplr) and carries its
    labels through them on the host.  `targets` are [n, 5] float32 (cls, xyxy) arrays (or None).  Returns the plans
    and the new label arrays; no device work."""
    plans, out = [], []
    for (h, w), t in zip(sizes, targets):
        lab = np.zeros((0, 5), np.float32) if t is None else t
        M, s, height, width = _perspective_draw((h, w), hyp["degrees"], hyp["translate"], hyp["scale"],
                                                hyp["shear"], hyp["perspective"], (0, 0))
        plan = _Plan(height, width)
        _warp_plan(plan, M, (0, 0), hyp["perspective"])
        lab = _warp_targets(lab, M, s, width, height, hyp["perspective"])
        plan.lut = _hsv_draw(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
        if random.random() < hyp["flipud"]:
            plan.flip_ud = True
            lab[:, [2, 4]] = height - lab[:, [4, 2]]
        if random.random() < hyp["fliplr"]:
            plan.flip_lr = True
            lab[:, [1, 3]] = width - lab[:, [3, 1]]
        plans.append(plan)
        out.append(lab)
    return plans, out


def apply_batch(images: Sequence[Tensor], targets: Optional[Sequence[Optional[Dict[str, Tensor]]]] = None,
                hyp: Optional[Dict[str, float]] = None, channel_order: str = "bgr"):
    """YOLOv5's non-mosaic training augmentations on a batch: for each image in order random_perspective ->
    augment_hsv -> flipud -> fliplr, drawn as `plan_batch` draws them, then every pixel in one launch.  `targets`
    are yolort-style {"boxes": [n, 4] xyxy pixels, "labels": [n]} dicts; `hyp` has the keys of hyp.scratch.yaml
    (HYP_SCRATCH by default).  channel_order "rgb" converts with COLOR_RGB2HSV / HSV2RGB, so decode_jpeg output goes
    straight in.  Returns (images, targets): the images are [H, W, 3] views into one buffer, the targets keep their
    other keys and come back on the device they came from."""
    if channel_order not in ("bgr", "rgb"):
        raise ValueError(f"channel_order must be 'bgr' or 'rgb', got {channel_order!r}")
    hyp = dict(HYP_SCRATCH if hyp is None else hyp)
    images = list(images)
    if not images:
        return [], []
    targets = [None] * len(images) if targets is None else list(targets)
    if len(targets) != len(images):
        raise ValueError(f"{len(images)} images and {len(targets)} targets")
    for im in images:
        _check_image(im, "apply_batch")
    dev = images[0].device
    if any(im.device != dev for im in images):
        raise ValueError("apply_batch: every image must be on the same device")
    arrays, where = [], []
    for t in targets:
        if t is None:
            arrays.append(None)
            where.append(None)
            continue
        if "boxes" not in t or "labels" not in t:
            raise ValueError("a target must hold 'boxes' and 'labels'")
        b, l = t["boxes"], t["labels"]
        where.append((b.device, l.device, l.dtype))
        arrays.append(np.concatenate([l.detach().cpu().numpy().astype(np.float32).reshape(-1, 1),
                                      b.detach().cpu().numpy().astype(np.float32).reshape(-1, 4)], 1))
    plans, labs = plan_batch([(int(im.shape[0]), int(im.shape[1])) for im in images], arrays, hyp)
    offsets, total = [], 0
    for p in plans:
        offsets.append(total)
        total += -(-3 * p.out_h * p.out_w // 16) * 16     # every image starts 16-byte aligned
    buf = torch.empty((total,), dtype=torch.uint8, device=dev)
    outs = [buf[o: o + 3 * p.out_h * p.out_w].view(p.out_h, p.out_w, 3) for o, p in zip(offsets, plans)]
    descs = (_C.V5Image * len(images))()
    for d, im, o, p in zip(descs, images, outs, plans):
        _fill(d, im, o, p, channel_order == "rgb")
    _C.v5_augment(descs, images, dev)
    out_targets = []
    for t, lab, wh in zip(targets, labs, where):
        if t is None:
            out_targets.append(None)
            continue
        t = dict(t)
        t["boxes"] = torch.from_numpy(np.ascontiguousarray(lab[:, 1:5])).to(wh[0])
        t["labels"] = torch.from_numpy(lab[:, 0].copy()).to(wh[2]).to(wh[1])
        out_targets.append(t)
    return outs, out_targets


def letterbox(im, new_shape=(640, 640), color=(114, 114, 114), auto=True, scale_fill=False, scaleup=True, stride=32):
    """letterbox (yolort/v5/utils/augmentations.py:99-137) of a CUDA uint8 [H, W, 3] image: resize with
    cv2.resize(INTER_LINEAR) when the size changes, then a constant border of `color` with the reference's
    int(round(d -/+ 0.1)) pads.  Returns (im [h, w, 3] uint8 in the image's channel order, ratio, (dw, dh)), with
    ratio and (dw, dh) the reference's values."""
    from .datasets import letterbox_image

    return letterbox_image(im, new_shape, color, auto, scale_fill, scaleup, stride)
