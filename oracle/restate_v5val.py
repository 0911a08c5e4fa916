"""Numpy restatement of YOLOv5's validation batches and rescale (upstream v6.0's LoadImagesAndLabels(augment=False,
rect=True, pad=0.5), collate_fn and val.py), and of the csrc/v5_augment.cu launches that compute them
(v5_resize_area_kernel, v5_resize_kernel, v5_compose_kernel, v5_rescale_kernel), written from the arithmetic alone
(no cv2 import).  Images are uint8 [H, W, 3] arrays.

    resize_area    cv2.resize(INTER_AREA) for 8-bit images, both axes shrinking: the integer-factor path and
                   computeResizeAreaTab + ResizeArea_Invoker's float accumulation
    load_image     load_image(augment=False): INTER_AREA when r < 1, INTER_LINEAR when r > 1
    letterbox      letterbox(im, new_shape, auto, scale_fill, scaleup, stride): geometry and pixels
    rect_plan      the rect block of LoadImagesAndLabels.__init__: irect, bi and batch_shapes
    getitem        __getitem__'s augment=False branch: image CHW RGB, labels_out [n, 6], shapes
    scale_coords   val.py's scale_coords / clip_coords, and targets_native its target rescale, in float32 as torch
                   computes them (python scalars rounded to float32)
"""
import math

import numpy as np

from oracle.restate_v5mosaic import resize_linear

F32 = np.float32
F64 = np.float64
DBL_EPSILON = np.finfo(np.float64).eps


def _cvround(x):
    """cvRound of float values: round half to even."""
    return np.rint(x).astype(np.int64)


def area_taps(ssz, dsz, scale):
    """computeResizeAreaTab of one axis: per output index a list of (source index, float32 weight) in table order."""
    taps = []
    for d in range(dsz):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, ssz - f1)
        s2 = min(math.floor(f2), ssz - 1)
        s1 = min(math.ceil(f1), s2)
        row = []
        if s1 - f1 > 1e-3:
            row.append((s1 - 1, F32((s1 - f1) / cell)))
        for s in range(s1, s2):
            row.append((s, F32(1.0 / cell)))
        if f2 - s2 > 1e-3:
            row.append((s2, F32(min(min(f2 - s2, 1.0), cell) / cell)))
        taps.append(row)
    return taps


def area_mode(h, w, dh, dw):
    """Which path cv2.resize(INTER_AREA) takes: "2x2", "int" (other integer factors) or "general"."""
    sx, sy = 1.0 / (dw / w), 1.0 / (dh / h)
    ix, iy = int(np.rint(sx)), int(np.rint(sy))
    if abs(sx - ix) < DBL_EPSILON and abs(sy - iy) < DBL_EPSILON:
        return "2x2" if ix == 2 and iy == 2 else "int"
    return "general"


def resize_area(im, dh, dw):
    """cv2.resize(im, (dw, dh), interpolation=INTER_AREA) of a uint8 [h, w, 3] image with dh <= h and dw <= w."""
    h, w = im.shape[:2]
    assert dh <= h and dw <= w
    sx, sy = 1.0 / (dw / w), 1.0 / (dh / h)
    mode = area_mode(h, w, dh, dw)
    if mode != "general":
        ix, iy = int(np.rint(sx)), int(np.rint(sy))
        a = im[:dh * iy, :dw * ix].astype(np.int64).reshape(dh, iy, dw, ix, 3).sum(axis=(1, 3))
        if mode == "2x2":
            return ((a + 2) >> 2).astype(np.uint8)
        return np.clip(_cvround(a.astype(F32) * (F32(1) / F32(ix * iy))), 0, 255).astype(np.uint8)
    xt, yt = area_taps(w, dw, sx), area_taps(h, dh, sy)
    src = im.astype(F32)
    # buf rows: the column taps of every source row, accumulated in tap order (buf starts at 0 and 0 + x == x)
    ncol = max(len(r) for r in xt)
    bufs = np.zeros((h, dw, 3), F32)
    for k in range(ncol):
        idx = np.array([r[k][0] if k < len(r) else 0 for r in xt])
        alpha = np.array([r[k][1] if k < len(r) else 0 for r in xt], F32)
        live = np.array([k < len(r) for r in xt])
        term = (src[:, idx] * alpha[None, :, None]).astype(F32)
        bufs = np.where(live[None, :, None], (bufs + term).astype(F32), bufs)
    out = np.zeros((dh, dw, 3), F32)
    for dy, row in enumerate(yt):
        s = None
        for sy_, beta in row:
            t = (beta * bufs[sy_]).astype(F32)
            s = t if s is None else (s + t).astype(F32)
        out[dy] = s
    return np.clip(_cvround(out), 0, 255).astype(np.uint8)


def load_image(im, s, augment=False):
    """load_image (v6.0): r = s / max(h0, w0); when r != 1, cv2.resize to (int(h0 * r), int(w0 * r)) with INTER_AREA if
    r < 1 and not augment, else INTER_LINEAR.  Returns (im, (h0, w0), (h, w))."""
    h0, w0 = im.shape[:2]
    r = s / max(h0, w0)
    if r != 1:
        h, w = int(h0 * r), int(w0 * r)
        if h < 1 or w < 1:
            raise ValueError("resize to an empty image")
        im = resize_area(im, h, w) if r < 1 and not augment else resize_linear(im, h, w)
    return im, (h0, w0), im.shape[:2]


def letterbox_geometry(shape, new_shape=(640, 640), auto=True, scale_fill=False, scaleup=True, stride=32):
    """letterbox's arithmetic for an image of shape (h, w): (new_unpad (w, h), ratio, (dw, dh), (top, bottom, left,
    right)), the reference's expressions in its order."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scale_fill:
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    pads = int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, ratio, (dw, dh), pads


def letterbox(im, new_shape=(640, 640), color=(114, 114, 114), auto=True, scale_fill=False, scaleup=True, stride=32):
    """letterbox: (im, ratio, (dw, dh)); the resize is cv2's INTER_LINEAR, the border copyMakeBorder's constant."""
    new_unpad, ratio, pad, (top, bottom, left, right) = letterbox_geometry(im.shape[:2], new_shape, auto, scale_fill,
                                                                          scaleup, stride)
    if im.shape[1::-1] != new_unpad:
        im = resize_linear(im, new_unpad[1], new_unpad[0])
    out = np.empty((new_unpad[1] + top + bottom, new_unpad[0] + left + right, 3), np.uint8)
    out[...] = np.asarray(color, np.uint8)
    out[top:top + new_unpad[1], left:left + new_unpad[0]] = im
    return out, ratio, pad


def rect_plan(shapes_hw, img_size=640, batch_size=32, stride=32, pad=0.5):
    """The rect block of LoadImagesAndLabels.__init__ (v6.0) for images of (h, w): (irect, bi, batch_shapes [nb, 2]
    (h, w)); batch k holds the images irect[bi == k]."""
    s = np.array([(w, h) for h, w in shapes_hw], dtype=np.float64)  # wh
    n = len(s)
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    ar = s[:, 1] / s[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    batch_shapes = np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
    return irect, bi, batch_shapes


def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
    y = np.copy(x)
    y[:, 0] = w * (x[:, 0] - x[:, 2] / 2) + padw
    y[:, 1] = h * (x[:, 1] - x[:, 3] / 2) + padh
    y[:, 2] = w * (x[:, 0] + x[:, 2] / 2) + padw
    y[:, 3] = h * (x[:, 1] + x[:, 3] / 2) + padh
    return y


def xyxy2xywhn(x, w=640, h=640, clip=False, eps=0.0):
    if clip:
        x[:, [0, 2]] = x[:, [0, 2]].clip(0, w - eps)
        x[:, [1, 3]] = x[:, [1, 3]].clip(0, h - eps)
    y = np.copy(x)
    y[:, 0] = ((x[:, 0] + x[:, 2]) / 2) / w
    y[:, 1] = ((x[:, 1] + x[:, 3]) / 2) / h
    y[:, 2] = (x[:, 2] - x[:, 0]) / w
    y[:, 3] = (x[:, 3] - x[:, 1]) / h
    return y


def getitem(im, labels, shape, img_size=640):
    """__getitem__ (v6.0), augment=False, of a BGR image with float32 labels [n, 5] (cls, xywhn) into the batch canvas
    `shape` (h, w): (CHW RGB image, labels_out float32 [n, 6] with column 0 zero, shapes)."""
    img, (h0, w0), (h, w) = load_image(im, img_size, augment=False)
    img, ratio, pad = letterbox(img, tuple(int(v) for v in shape), auto=False, scaleup=False)
    shapes = (h0, w0), ((h / h0, w / w0), pad)
    labels = np.array(labels, np.float32).reshape(-1, 5).copy()
    if labels.size:
        labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    nl = len(labels)
    if nl:
        labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=img.shape[1], h=img.shape[0], clip=True, eps=1E-3)
    labels_out = np.zeros((nl, 6), np.float32)
    if nl:
        labels_out[:, 1:] = labels
    return np.ascontiguousarray(img.transpose((2, 0, 1))[::-1]), labels_out, shapes


def collate(items):
    """collate_fn's [0], [1], [3] of getitem outputs: (imgs [N, 3, H, W], targets [T, 6], shapes)."""
    targets = []
    for i, (_, lab, _) in enumerate(items):
        lab = lab.copy()
        lab[:, 0] = i
        targets.append(lab)
    return np.stack([it[0] for it in items]), np.concatenate(targets, 0), [it[2] for it in items]


# -- val.py's rescale, float32 as torch computes it ----------------------------------------------------------------
def clip_coords(boxes, shape):
    """clip_coords of float32 boxes [n, 4] to shape (h, w), in place (torch.clamp_: NaN stays NaN)."""
    for c, hi in ((0, shape[1]), (1, shape[0]), (2, shape[1]), (3, shape[0])):
        v = boxes[:, c]
        v = np.where(v < 0, F32(0), v)
        boxes[:, c] = np.where(v > hi, F32(hi), v)
    return boxes


def scale_coords(img1_shape, coords, img0_shape, ratio_pad=None):
    """scale_coords of float32 coords [n, >= 4], in place."""
    if ratio_pad is None:
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    else:
        gain = ratio_pad[0][0]
        pad = ratio_pad[1]
    coords[:, [0, 2]] = (coords[:, [0, 2]] - F32(pad[0])).astype(F32)
    coords[:, [1, 3]] = (coords[:, [1, 3]] - F32(pad[1])).astype(F32)
    coords[:, :4] = (coords[:, :4] / F32(gain)).astype(F32)
    clip_coords(coords, img0_shape)
    return coords


def xywh2xyxy(x):
    """xywh2xyxy of float32 [n, 4] (w / 2 exactly as w * 0.5)."""
    y = np.copy(x)
    y[:, 0] = x[:, 0] - x[:, 2] / F32(2)
    y[:, 1] = x[:, 1] - x[:, 3] / F32(2)
    y[:, 2] = x[:, 0] + x[:, 2] / F32(2)
    y[:, 3] = x[:, 1] + x[:, 3] / F32(2)
    return y


def targets_native(targets, canvas_hw, shapes):
    """val.py's labels of one batch in native pixels: targets[:, 2:] *= [W, H, W, H], then per image xywh2xyxy and
    scale_coords(img[si].shape[1:], tbox, shapes[si][0], shapes[si][1]).  Returns [T, 6] (image, cls, xyxy)."""
    H, W = canvas_hw
    t = np.array(targets, np.float32).copy()
    t[:, 2:] = (t[:, 2:] * np.array([W, H, W, H], np.float32)).astype(F32)
    out = t.copy()
    for si in range(len(shapes)):
        m = t[:, 0] == si
        tbox = xywh2xyxy(t[m, 2:6])
        out[m, 2:6] = scale_coords((H, W), tbox, shapes[si][0], shapes[si][1])
    return out


def boxes_native(boxes, counts, canvas_hw, shapes):
    """val.py's predn of padded detections [n, D, 4] (slots below counts), per image; other slots unchanged."""
    out = np.array(boxes, np.float32).copy()
    for si in range(len(shapes)):
        c = int(counts[si])
        out[si, :c] = scale_coords(canvas_hw, out[si, :c].copy(), shapes[si][0], shapes[si][1])
    return out
