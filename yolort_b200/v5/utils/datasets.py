"""YOLOv5's mosaic training batches on the GPU: the augment=True, rect=False branch of upstream YOLOv5 v6.0's
`LoadImagesAndLabels.__getitem__` (load_image, load_mosaic or the letterbox branch, random_perspective, mixup,
augment_hsv, flipud, fliplr) followed by `collate_fn`.

    load_image(im, img_size)                      -> (im, (h0, w0), (h, w))
    load_mosaic(images, labels, index, img_size, hyp) -> (img4 [s, s, 3], labels4 [n, 5] (cls, xyxy))
    train_batch(images, labels, indices, img_size, hyp, channel_order)
                                                  -> (imgs uint8 [N, 3, s, s] RGB, targets float32 [n, 6])

`images` are the dataset's CUDA uint8 [H, W, 3] tensors (cv2's layout, any strides; the HWC views of
`yolort_b200.io.decode_jpeg` go straight in with channel_order="rgb"), `labels` upstream's per-image float32 [n, 5]
(cls, x, y, w, h) normalised arrays.  Every parameter is drawn on the host from Python's `random` and numpy's global
generator in upstream's order, and the boxes go through upstream's numpy expressions, so after
`random.seed(k); np.random.seed(k)` the draws, the generators' states, the labels and the pixels are upstream's.

The pixels come from two launches of csrc/v5_augment.cu: cv2.resize(INTER_LINEAR) of the images load_image scales
(OpenCV's 8-bit fixed-point arithmetic, and its INTER_AREA average for an exact 2x downscale), then one launch for the
whole batch that warps each sample from a virtual canvas (the mosaic's four placements, or the letterbox's one, and 114
elsewhere; the 2s x 2s canvas is never written), blends mixup in IEEE double, runs the HSV steps and the flips and
stores CHW RGB.  oracle/restate_v5mosaic.py restates every step.  Segments (copy_paste) are not supported.
"""
import random
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from ... import _C
from . import augmentations as _aug

__all__ = ["load_image", "load_mosaic", "train_batch", "xywhn2xyxy", "xyxy2xywhn", "HYP_SCRATCH"]

# yolort/v5/data/hyps/hyp.scratch.yaml: the augmentation keys of augmentations.HYP_SCRATCH and the loader's own
HYP_SCRATCH = dict(_aug.HYP_SCRATCH, mosaic=1.0, mixup=0.0, copy_paste=0.0)


# -- upstream's box expressions (yolort/v5/utils/general.py) -------------------------------------------------------
def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
    """nx4 boxes from normalised [x, y, w, h] to pixel [x1, y1, x2, y2]."""
    y = np.copy(x)
    y[:, 0] = w * (x[:, 0] - x[:, 2] / 2) + padw  # top left x
    y[:, 1] = h * (x[:, 1] - x[:, 3] / 2) + padh  # top left y
    y[:, 2] = w * (x[:, 0] + x[:, 2] / 2) + padw  # bottom right x
    y[:, 3] = h * (x[:, 1] + x[:, 3] / 2) + padh  # bottom right y
    return y


def xyxy2xywhn(x, w=640, h=640, clip=False, eps=0.0):
    """nx4 boxes from pixel [x1, y1, x2, y2] to normalised [x, y, w, h]; `clip` clips x in place first."""
    if clip:
        x[:, [0, 2]] = x[:, [0, 2]].clip(0, w - eps)  # x1, x2
        x[:, [1, 3]] = x[:, [1, 3]].clip(0, h - eps)  # y1, y2
    y = np.copy(x)
    y[:, 0] = ((x[:, 0] + x[:, 2]) / 2) / w  # x center
    y[:, 1] = ((x[:, 1] + x[:, 3]) / 2) / h  # y center
    y[:, 2] = (x[:, 2] - x[:, 0]) / w  # width
    y[:, 3] = (x[:, 3] - x[:, 1]) / h  # height
    return y


# -- geometry ------------------------------------------------------------------------------------------------------
def load_shape(h0: int, w0: int, img_size: int) -> Tuple[int, int]:
    """load_image's output size: int(h0 * r), int(w0 * r) with r = img_size / max(h0, w0) (the input's when r == 1).
    int() can leave the long side at img_size - 1."""
    r = img_size / max(h0, w0)
    if r == 1:
        return h0, w0
    h, w = int(h0 * r), int(w0 * r)
    if h < 1 or w < 1:
        raise ValueError(f"load_image: a {h0}x{w0} image resizes to {h}x{w} at img_size {img_size}")
    return h, w


def mosaic_place(i: int, s: int, xc: int, yc: int, h: int, w: int):
    """Upstream's rectangles of quadrant i (top-left, top-right, bottom-left, bottom-right) of the 2s x 2s canvas:
    (x1a, y1a, x2a, y2a) on the canvas, (x1b, y1b, x2b, y2b) in the image."""
    if i == 0:  # top left
        x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc  # xmin, ymin, xmax, ymax (large image)
        x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h  # xmin, ymin, xmax, ymax (small image)
    elif i == 1:  # top right
        x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
        x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
    elif i == 2:  # bottom left
        x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, w, min(y2a - y1a, h)
    else:  # bottom right
        x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
    return (x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b)


def letterbox_geometry(h: int, w: int, s: int):
    """letterbox(im, s, auto=False, scaleup=True) of an h x w image: ((nh, nw), ratio, (dw, dh), (top, left),
    (out_h, out_w))."""
    r = min(s / h, s / w)
    ratio = r, r  # width, height ratios
    new_unpad = int(round(w * r)), int(round(h * r))
    dw, dh = s - new_unpad[0], s - new_unpad[1]  # wh padding
    dw /= 2  # divide padding into 2 sides
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    out = (new_unpad[1] + top + bottom, new_unpad[0] + left + right)
    return (new_unpad[1], new_unpad[0]), ratio, (dw, dh), (top, left), out


class Canvas:
    """A virtual canvas: placements (key, y0, x0, y1, x1, oy, ox) -- canvas [y0, y1) x [x0, x1) reads the loaded
    image `key` at (y - oy, x - ox), 114 elsewhere -- and the inverse warp that reads it (inv None: no warp)."""

    def __init__(self, h: int, w: int):
        self.h, self.w = h, w
        self.places: List[tuple] = []
        self.inv: Optional[np.ndarray] = None
        self.perspective = False


class Sample:
    """One training sample's draws: its canvases (two with mixup, ratio r), LUT, flips and normalised labels."""

    def __init__(self, out_h: int, out_w: int):
        self.out_h, self.out_w = out_h, out_w
        self.canvases: List[Canvas] = []
        self.r: Optional[float] = None
        self.lut: Optional[np.ndarray] = None
        self.flip_ud = self.flip_lr = False
        self.mosaic = False
        self.labels = np.zeros((0, 5), np.float32)


class Planner:
    """Upstream's draws for a dataset of images of `shapes` [(h0, w0)] and normalised `labels`, on the host.  The
    loaded images are keys: an index (load_image), or ("letterbox", index) (letterbox's second resize of a load_image
    output whose long side int() left at img_size - 1); `loads` maps each key to (source key or index, (h, w))."""

    def __init__(self, shapes, labels, img_size: int, hyp: Dict[str, float]):
        self.shapes, self.labels, self.s, self.hyp = list(shapes), list(labels), int(img_size), hyp
        self.n = len(self.shapes)
        self.loads: Dict[object, tuple] = {}

    def load(self, index: int) -> Tuple[int, int]:
        h0, w0 = self.shapes[index]
        hw = load_shape(h0, w0, self.s)
        if hw != (h0, w0):
            self.loads[index] = (None, hw)
        return hw

    def mosaic(self, index: int):
        """load_mosaic's draws: (canvas, labels4 xyxy)."""
        s, hyp = self.s, self.hyp
        border = [-s // 2, -s // 2]
        yc, xc = (int(random.uniform(-x, 2 * s + x)) for x in border)  # mosaic center x, y
        indices = [index] + random.choices(range(self.n), k=3)  # 3 additional image indices
        random.shuffle(indices)
        cv = Canvas(2 * s, 2 * s)
        labels4 = []
        for i, idx in enumerate(indices):
            h, w = self.load(idx)
            (x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b) = mosaic_place(i, s, xc, yc, h, w)
            padw, padh = x1a - x1b, y1a - y1b
            if y2a > y1a and x2a > x1a:
                cv.places.append((idx, y1a, x1a, y2a, x2a, padh, padw))
            labels = self.labels[idx].copy()
            if labels.size:
                labels[:, 1:] = xywhn2xyxy(labels[:, 1:], w, h, padw, padh)  # normalized xywh to pixel xyxy format
            labels4.append(labels)
        labels4 = np.concatenate(labels4, 0)
        np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
        # copy_paste draws nothing without segments
        labels4 = self._perspective(cv, labels4, border)
        return cv, labels4

    def _perspective(self, cv: Canvas, labels, border):
        hyp = self.hyp
        M, sc, height, width = _aug._perspective_draw((cv.h, cv.w), hyp["degrees"], hyp["translate"], hyp["scale"],
                                                      hyp["shear"], hyp["perspective"], border)
        plan = _aug._Plan(height, width)
        _aug._warp_plan(plan, M, border, hyp["perspective"])
        cv.inv, cv.perspective = plan.inv, plan.perspective
        cv.out = (height, width)
        return _aug._warp_targets(labels, M, sc, width, height, hyp["perspective"])

    def letterbox(self, index: int):
        """The letterbox branch's draws: (canvas, labels xyxy)."""
        s = self.s
        h, w = self.load(index)
        (nh, nw), ratio, pad, (top, left), out = letterbox_geometry(h, w, s)
        key = index
        if (nh, nw) != (h, w):
            key = ("letterbox", index)
            self.loads[key] = (index, (nh, nw))
        cv = Canvas(*out)
        cv.places.append((key, top, left, top + nh, left + nw, top, left))
        labels = self.labels[index].copy()
        if labels.size:  # normalized xywh to pixel xyxy format
            labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
        labels = self._perspective(cv, labels, (0, 0))
        return cv, labels

    def sample(self, index: int) -> Sample:
        hyp = self.hyp
        if random.random() < hyp["mosaic"]:
            cv, labels = self.mosaic(index)
            canvases, r = [cv], None
            if random.random() < hyp["mixup"]:
                cv2_, labels2 = self.mosaic(random.randint(0, self.n - 1))
                r = np.random.beta(32.0, 32.0)  # mixup ratio, alpha=beta=32.0
                labels = np.concatenate((labels, labels2), 0)
                canvases.append(cv2_)
            mosaic = True
        else:
            cv, labels = self.letterbox(index)
            canvases, r, mosaic = [cv], None, False
        out_h, out_w = canvases[0].out
        nl = len(labels)  # number of labels
        if nl:
            labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=out_w, h=out_h, clip=True, eps=1E-3)
        smp = Sample(out_h, out_w)
        smp.canvases, smp.r, smp.mosaic = canvases, r, mosaic
        smp.lut = _aug._hsv_draw(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
        if random.random() < hyp["flipud"]:
            smp.flip_ud = True
            if nl:
                labels[:, 2] = 1 - labels[:, 2]
        if random.random() < hyp["fliplr"]:
            smp.flip_lr = True
            if nl:
                labels[:, 1] = 1 - labels[:, 1]
        smp.labels = labels
        return smp


# -- device work ---------------------------------------------------------------------------------------------------
def _check_inputs(images, labels, segments, hyp, what: str):
    if segments is not None and any(len(sg) for sg in segments):
        raise NotImplementedError(f"{what}: segments (copy_paste) are not supported on the GPU")
    for im in images:
        _aug._check_image(im, what)
    if not images:
        raise ValueError(f"{what}: no images")
    dev = images[0].device
    if any(im.device != dev for im in images):
        raise ValueError(f"{what}: every image must be on the same device")
    if len(labels) != len(images):
        raise ValueError(f"{what}: {len(images)} images and {len(labels)} label arrays")
    out = []
    for lab in labels:
        lab = np.zeros((0, 5), np.float32) if lab is None else np.asarray(lab)
        if lab.ndim != 2 or lab.shape[1] != 5:
            raise ValueError(f"{what}: labels must be [n, 5] (cls, x, y, w, h) arrays, got {lab.shape}")
        out.append(lab)
    for k in ("mosaic", "mixup", "copy_paste"):
        if k not in hyp:
            raise ValueError(f"{what}: hyp has no {k!r}")
    return dev, out


def _views(t: Tensor):
    return t.data_ptr(), [int(v) for v in t.stride()]


def _run_loads(planner: Planner, images: Sequence[Tensor], dev) -> Dict[object, Tensor]:
    """Every loaded image the plans read: the dataset image itself, or a resize into one scratch buffer (load_image's
    first, then letterbox's second resize in a launch of their own)."""
    loaded: Dict[object, Tensor] = {}
    levels = [[k for k, v in planner.loads.items() if v[0] is None], [k for k, v in planner.loads.items()
                                                                        if v[0] is not None]]
    sizes = {k: 3 * hw[0] * hw[1] for k, (_, hw) in planner.loads.items()}
    total = sum(-(-n // 16) * 16 for n in sizes.values())
    buf = torch.empty((max(total, 1),), dtype=torch.uint8, device=dev) if planner.loads else None
    off = 0
    for keys in levels:
        if not keys:
            continue
        jobs = (_C.V5ResizeJob * len(keys))()
        srcs = []
        for j, k in zip(jobs, keys):
            src_key, (h, w) = planner.loads[k]
            src = images[k] if src_key is None else loaded.get(src_key, images[src_key])
            dst = buf[off: off + 3 * h * w].view(h, w, 3)
            off += -(-3 * h * w // 16) * 16
            j.src, (j.src_stride_y, j.src_stride_x, j.src_stride_c) = _views(src)
            j.dst = dst.data_ptr()
            j.src_h, j.src_w, j.dst_h, j.dst_w = int(src.shape[0]), int(src.shape[1]), h, w
            loaded[k] = dst
            srcs += [src, dst]
        _C.v5_resize(jobs, srcs, dev)
    return loaded


def _fill_sample(d, smp: Sample, images, loaded, dst: Tensor, dst_strides, rgb: bool, colour: bool) -> None:
    d.dst = dst.data_ptr()
    d.dst_stride_y, d.dst_stride_x, d.dst_stride_c = dst_strides
    d.out_h, d.out_w = smp.out_h, smp.out_w
    ops = _C.YB_V5_RGB if rgb else 0
    if colour:
        if smp.lut is not None:
            ops |= _aug._HSV
            np.ctypeslib.as_array(d.lut)[...] = smp.lut
        if smp.flip_ud:
            ops |= _C.YB_V5_FLIP_UD
        if smp.flip_lr:
            ops |= _C.YB_V5_FLIP_LR
    d.ops = ops
    d.n_canvases = len(smp.canvases)
    if smp.r is not None:
        d.mix_r, d.mix_omr = float(smp.r), float(1 - smp.r)
    for c, cv in zip(d.canvas, smp.canvases):
        if cv.inv is not None:
            c.warp = _C.YB_V5_PERSPECTIVE if cv.perspective else _C.YB_V5_AFFINE
            for j, v in enumerate(cv.inv):
                c.inv[j] = float(v)
        c.n_places = len(cv.places)
        for p, (key, y0, x0, y1, x1, oy, ox) in zip(c.places, cv.places):
            src = loaded.get(key, images[key] if isinstance(key, int) else None)
            p.src, (p.stride_y, p.stride_x, p.stride_c) = _views(src)
            p.y0, p.x0, p.y1, p.x1, p.oy, p.ox = y0, x0, y1, x1, oy, ox


def _compose(samples: List[Sample], images, loaded, outs: Sequence[Tensor], strides, rgb: bool, colour: bool, dev):
    descs = (_C.V5Sample * len(samples))()
    for d, smp, o, st in zip(descs, samples, outs, strides):
        _fill_sample(d, smp, images, loaded, o, st, rgb, colour)
    _C.v5_compose(descs, list(images) + list(loaded.values()) + list(outs), dev)


# -- upstream's functions ------------------------------------------------------------------------------------------
def load_image(im, img_size: int):
    """load_image (v6.0, augment=True): `im` resized by r = img_size / max(h0, w0) with cv2.resize(INTER_LINEAR) to
    (int(h0 * r), int(w0 * r)) when r != 1, else `im` itself; returns (im, (h0, w0), (h, w))."""
    _aug._check_image(im, "load_image")
    h0, w0 = int(im.shape[0]), int(im.shape[1])
    planner = Planner([(h0, w0)], [None], img_size, HYP_SCRATCH)
    h, w = planner.load(0)
    if (h, w) == (h0, w0):
        return im, (h0, w0), (h, w)
    return _run_loads(planner, [im], im.device)[0], (h0, w0), (h, w)


def load_mosaic(images: Sequence[Tensor], labels, index: int, img_size: int = 640, hyp=None, segments=None):
    """load_mosaic (v6.0) of dataset item `index`: four load_image outputs on a 2s x 2s canvas of 114 around a random
    centre, then random_perspective with border (-s // 2, -s // 2).  Returns (img4 uint8 [s, s, 3] in the images'
    channel order, labels4 [n, 5] (cls, xyxy) pixels)."""
    images = list(images)
    hyp = dict(HYP_SCRATCH if hyp is None else hyp)
    dev, labels = _check_inputs(images, list(labels), segments, hyp, "load_mosaic")
    if int(img_size) % 2:
        raise ValueError(f"load_mosaic: img_size {img_size} must be even")
    planner = Planner([(int(im.shape[0]), int(im.shape[1])) for im in images], labels, img_size, hyp)
    cv, labels4 = planner.mosaic(int(index))
    smp = Sample(*cv.out)
    smp.canvases = [cv]
    loaded = _run_loads(planner, images, dev)
    out = torch.empty((smp.out_h, smp.out_w, 3), dtype=torch.uint8, device=dev)
    _compose([smp], images, loaded, [out], [tuple(int(v) for v in out.stride())], False, False, dev)
    return out, labels4


def train_batch(images: Sequence[Tensor], labels, indices: Sequence[int], img_size: int = 640, hyp=None,
                channel_order: str = "bgr", segments=None):
    """`collate_fn([dataset[i] for i in indices])[:2]` of upstream's LoadImagesAndLabels(augment=True, rect=False):
    per index, mosaic (probability hyp["mosaic"], with mixup of a second mosaic at hyp["mixup"]) or letterbox, then
    random_perspective, augment_hsv, flipud and fliplr.  Returns (imgs uint8 [N, 3, s, s] RGB, targets float32
    [n, 6] (image, cls, x, y, w, h normalised)) on the images' device; `YOLO.train()(imgs / 255, targets)` takes them
    as they are.  channel_order "rgb" takes RGB images (decode_jpeg's) through COLOR_RGB2HSV / HSV2RGB."""
    if channel_order not in ("bgr", "rgb"):
        raise ValueError(f"channel_order must be 'bgr' or 'rgb', got {channel_order!r}")
    images = list(images)
    hyp = dict(HYP_SCRATCH if hyp is None else hyp)
    dev, labels = _check_inputs(images, list(labels), segments, hyp, "train_batch")
    indices = [int(i) for i in indices]
    if not indices:
        raise ValueError("train_batch: no indices")
    if any(i < 0 or i >= len(images) for i in indices):
        raise IndexError(f"train_batch: an index outside 0..{len(images) - 1}")
    s = int(img_size)
    if s < 2 or s % 2:
        raise ValueError(f"train_batch: img_size {img_size} must be even")
    planner = Planner([(int(im.shape[0]), int(im.shape[1])) for im in images], labels, s, hyp)
    samples = [planner.sample(i) for i in indices]
    loaded = _run_loads(planner, images, dev)
    imgs = torch.empty((len(samples), 3, s, s), dtype=torch.uint8, device=dev)
    rgb = channel_order == "rgb"
    plane = s * s
    # channel k of the sample lands in plane k (RGB) or 2 - k (BGR)
    outs = [imgs[n] if rgb else imgs[n, 2] for n in range(len(samples))]
    strides = [(s, 1, plane if rgb else -plane)] * len(samples)
    _compose(samples, images, loaded, outs, strides, rgb, True, dev)
    rows = []
    for n, smp in enumerate(samples):
        lab = np.zeros((len(smp.labels), 6), np.float32)
        lab[:, 1:] = smp.labels
        lab[:, 0] = n
        rows.append(lab)
    targets = torch.from_numpy(np.concatenate(rows, 0)).to(dev)
    return imgs, targets
