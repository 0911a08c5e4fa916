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

__all__ = ["load_image", "load_mosaic", "train_batch", "rect_batches", "val_batch", "xywhn2xyxy", "xyxy2xywhn",
           "HYP_SCRATCH"]

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


def letterbox_arith(shape, new_shape=(640, 640), auto=True, scale_fill=False, scaleup=True, stride=32):
    """letterbox's arithmetic (yolort/v5/utils/augmentations.py:99-137) for an image of shape (h, w), the reference's
    expressions in its order: ((nh, nw), ratio, (dw, dh), (top, bottom, left, right))."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:  # only scale down, do not scale up (for better val mAP)
        r = min(r, 1.0)
    ratio = r, r  # width, height ratios
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]  # wh padding
    if auto:  # minimum rectangle
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)  # wh padding
    elif scale_fill:  # stretch
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]  # width, height ratios
    dw /= 2  # divide padding into 2 sides
    dh /= 2
    pads = int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1))
    return (new_unpad[1], new_unpad[0]), ratio, (dw, dh), pads


def rect_batches(shapes, img_size: int = 640, batch_size: int = 32, stride: int = 32, pad: float = 0.5):
    """The rect block of upstream v6.0's LoadImagesAndLabels.__init__ for images of `shapes` [(h, w)]: (irect, bi,
    batch_shapes).  The images sorted by aspect ratio h / w (numpy's default argsort) are irect; sorted image j goes
    to batch bi[j] = j // batch_size, whose canvas is batch_shapes[bi[j]] = (H, W), multiples of `stride` (the
    model's largest: 64 for the P6 models)."""
    s = np.array([(w, h) for h, w in shapes], dtype=np.float64)  # wh
    n = len(s)
    if n == 0:
        raise ValueError("rect_batches: no images")
    bi = np.floor(np.arange(n) / batch_size).astype(int)  # batch index
    nb = bi[-1] + 1  # number of batches
    ar = s[:, 1] / s[:, 0]  # aspect ratio
    irect = ar.argsort()
    ar = ar[irect]
    batch_shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            batch_shapes[i] = [maxi, 1]
        elif mini > 1:
            batch_shapes[i] = [1, 1 / mini]
    return irect, bi, np.ceil(np.array(batch_shapes) * img_size / stride + pad).astype(int) * stride


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
        self.area = set()           # loads resized with INTER_AREA (load_image with augment=False, r < 1)

    def load(self, index: int, augment: bool = True) -> Tuple[int, int]:
        h0, w0 = self.shapes[index]
        hw = load_shape(h0, w0, self.s)
        if hw != (h0, w0):
            self.loads[index] = (None, hw)
            if not augment and self.s < max(h0, w0):
                self.area.add(index)
        return hw

    def val_sample(self, index: int, shape: Tuple[int, int]):
        """__getitem__'s augment=False branch into the batch canvas `shape` (H, W): load_image(augment=False), then
        letterbox(auto=False, scaleup=False).  Returns (Sample, shapes)."""
        h0, w0 = self.shapes[index]
        h, w = self.load(index, augment=False)
        (nh, nw), ratio, pad, (top, bottom, left, right) = letterbox_arith((h, w), shape, auto=False, scaleup=False)
        key = index
        if (nh, nw) != (h, w):
            key = ("letterbox", index)
            self.loads[key] = (index, (nh, nw))
        cv = Canvas(nh + top + bottom, nw + left + right)
        cv.places.append((key, top, left, top + nh, left + nw, top, left))
        labels = self.labels[index].copy()
        if labels.size:  # normalized xywh to pixel xyxy format
            labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
        if len(labels):
            labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=cv.w, h=cv.h, clip=True, eps=1E-3)
        smp = Sample(cv.h, cv.w)
        smp.canvases, smp.labels = [cv], labels
        return smp, ((h0, w0), ((h / h0, w / w0), pad))

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
    # INTER_AREA loads take a launch of their own
    levels = [[k for k in levels[0] if k not in planner.area], [k for k in levels[0] if k in planner.area], levels[1]]
    for level, keys in enumerate(levels):
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
        _C.v5_resize(jobs, srcs, dev, area=level == 1)
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
def load_image(im, img_size: int, augment: bool = True):
    """load_image (v6.0): `im` resized by r = img_size / max(h0, w0) to (int(h0 * r), int(w0 * r)) when r != 1, else
    `im` itself; returns (im, (h0, w0), (h, w)).  The resize is cv2.resize(INTER_AREA) when r < 1 and not `augment`
    (the validation loader's), else cv2.resize(INTER_LINEAR).  A side that resizes to 0 raises ValueError."""
    _aug._check_image(im, "load_image")
    h0, w0 = int(im.shape[0]), int(im.shape[1])
    planner = Planner([(h0, w0)], [None], img_size, HYP_SCRATCH)
    h, w = planner.load(0, augment=bool(augment))
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


class ValPlan:
    """val_batch's host plan of one rect batch, and its two launches: `resize()` (the INTER_AREA shrinks, then the
    INTER_LINEAR resizes) and `compose(imgs)` (every canvas, CHW RGB, into a contiguous uint8 [N, 3, H, W]).
    `shapes` and `targets()` are collate_fn's; `targets()` copies from pinned memory without waiting for the device."""

    def __init__(self, images: Sequence[Tensor], labels, indices: Sequence[int], batch_shape, img_size: int = 640,
                 channel_order: str = "bgr"):
        if channel_order not in ("bgr", "rgb"):
            raise ValueError(f"channel_order must be 'bgr' or 'rgb', got {channel_order!r}")
        self.images = list(images)
        self.dev, labels = _check_inputs(self.images, list(labels), None, HYP_SCRATCH, "val_batch")
        indices = [int(i) for i in indices]
        if not indices:
            raise ValueError("val_batch: no indices")
        if any(i < 0 or i >= len(self.images) for i in indices):
            raise IndexError(f"val_batch: an index outside 0..{len(self.images) - 1}")
        H, W = (int(v) for v in batch_shape)
        self.H, self.W = H, W
        if H < 1 or W < 1:
            raise ValueError(f"val_batch: batch_shape {tuple(batch_shape)}")
        self.rgb = channel_order == "rgb"
        self.planner = Planner([(int(im.shape[0]), int(im.shape[1])) for im in self.images], labels, img_size,
                               HYP_SCRATCH)
        self.samples, self.shapes = [], []
        for i in indices:
            smp, shp = self.planner.val_sample(i, (H, W))
            if (smp.out_h, smp.out_w) != (H, W):
                raise ValueError(f"val_batch: image {i} letterboxes to {smp.out_h}x{smp.out_w}, not the canvas {H}x{W}")
            self.samples.append(smp)
            self.shapes.append(shp)
        self.loaded = None

    def resize(self) -> None:
        self.loaded = _run_loads(self.planner, self.images, self.dev)

    def compose(self, imgs: Tensor) -> None:
        n, H, W = len(self.samples), self.H, self.W
        if tuple(imgs.shape) != (n, 3, H, W) or imgs.dtype != torch.uint8 or not imgs.is_contiguous():
            raise ValueError(f"val_batch: the output must be a contiguous uint8 [{n}, 3, {H}, {W}] tensor")
        plane = H * W
        # channel k of the sample lands in plane k (RGB) or 2 - k (BGR)
        outs = [imgs[k] if self.rgb else imgs[k, 2] for k in range(n)]
        strides = [(W, 1, plane if self.rgb else -plane)] * n
        _compose(self.samples, self.images, self.loaded, outs, strides, self.rgb, False, self.dev)

    def targets(self) -> Tensor:
        rows = []
        for k, smp in enumerate(self.samples):
            lab = np.zeros((len(smp.labels), 6), np.float32)
            lab[:, 1:] = smp.labels
            lab[:, 0] = k
            rows.append(lab)
        return torch.from_numpy(np.concatenate(rows, 0)).pin_memory().to(self.dev, non_blocking=True)


def val_batch(images: Sequence[Tensor], labels, indices: Sequence[int], batch_shape, img_size: int = 640,
              channel_order: str = "bgr"):
    """`collate_fn([dataset[i] for i in indices])` [0], [1] and [3] of upstream v6.0's LoadImagesAndLabels(augment=False,
    rect=True): per index load_image(augment=False) (cv2.resize INTER_AREA when it shrinks) and letterbox(auto=False,
    scaleup=False) centred in the batch canvas `batch_shape` (H, W) (rect_batches' batch_shapes).  Returns
    (imgs uint8 [N, 3, H, W] RGB, targets float32 [T, 6] (image, cls, x, y, w, h normalised to the canvas), shapes
    [((h0, w0), ((h / h0, w / w0), (dw, dh)))]), the images and targets on the images' device; nothing waits for the
    device.  `labels` are train_batch's; channel_order "rgb" takes RGB images (decode_jpeg's) as they are."""
    plan = ValPlan(images, labels, indices, batch_shape, img_size, channel_order)
    plan.resize()
    imgs = torch.empty((len(plan.samples), 3, plan.H, plan.W), dtype=torch.uint8, device=plan.dev)
    plan.compose(imgs)
    return imgs, plan.targets(), plan.shapes


def letterbox_image(im, new_shape=(640, 640), color=(114, 114, 114), auto=True, scale_fill=False, scaleup=True,
                    stride=32):
    """augmentations.letterbox: the resize (cv2 INTER_LINEAR, when the size changes) and the constant border, one
    compose launch; HWC in the image's channel order."""
    _aug._check_image(im, "letterbox")
    color = tuple(int(c) for c in color)
    if len(color) != 3 or any(c < 0 or c > 255 for c in color):
        raise ValueError(f"letterbox: color must be three values in 0..255, got {color}")
    h, w = int(im.shape[0]), int(im.shape[1])
    (nh, nw), ratio, pad, (top, bottom, left, right) = letterbox_arith((h, w), new_shape, auto, scale_fill, scaleup,
                                                                       stride)
    if nh < 1 or nw < 1:
        raise ValueError(f"letterbox: a {h}x{w} image resizes to {nh}x{nw}")
    planner = Planner([(h, w)], [None], max(h, w), HYP_SCRATCH)
    key = 0
    if (nh, nw) != (h, w):
        key = ("letterbox", 0)
        planner.loads[key] = (0, (nh, nw))
    oh, ow = nh + top + bottom, nw + left + right
    out = torch.empty((oh, ow, 3), dtype=torch.uint8, device=im.device)
    if color == (114, 114, 114):    # the compose kernel's border value: one launch writes the whole canvas
        dst, smp = out, Sample(oh, ow)
        cv = Canvas(oh, ow)
        cv.places.append((key, top, left, top + nh, left + nw, top, left))
    else:
        out[...] = torch.tensor(color, dtype=torch.uint8).to(im.device)
        dst, smp = out[top:top + nh, left:left + nw], Sample(nh, nw)
        cv = Canvas(nh, nw)
        cv.places.append((key, 0, 0, nh, nw, 0, 0))
    smp.canvases = [cv]
    loaded = _run_loads(planner, [im], im.device)
    _compose([smp], [im], loaded, [dst], [tuple(int(v) for v in dst.stride())], False, False, im.device)
    return out, ratio, pad
