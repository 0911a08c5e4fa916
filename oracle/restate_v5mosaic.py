"""Numpy restatement of csrc/v5_augment.cu's mosaic loader launches (v5_resize_kernel, v5_compose_kernel): YOLOv5's
mosaic training samples as upstream v6.0's LoadImagesAndLabels(augment=True, rect=False) computes them with OpenCV 4.x
(cv2.resize INTER_LINEAR, the mosaic canvas, letterbox), written from the arithmetic alone (no cv2 import).  The warp,
mixup and HSV steps are oracle/restate_v5aug.py's.  Images are uint8 [H, W, 3] arrays.

    resize_linear  cv2.resize(INTER_LINEAR) for 8-bit images: 11-bit coefficients, horizontal pass in int, then the
                   (S >> 4) * b >> 16 vertical pass; an exact 2x downscale is INTER_AREA's (2 x 2 sum + 2) >> 2
    mosaic_rects   load_mosaic's placement arithmetic
    letterbox_pad  letterbox(auto=False, scaleup=True)'s size and padding
    sample_pixels  one training sample from its host plan: canvases, warps, mixup, HSV, flips, CHW RGB

Upstream's loader is not part of the reference tree; its steps are restated from v6.0's datasets.py: load_image
resizes by r = s / max(h0, w0) to (int(h0 * r), int(w0 * r)) with INTER_LINEAR when r != 1; load_mosaic places four
load_image outputs around a centre drawn as int(uniform(s // 2, 2s - s // 2)) (y first), after
random.choices(range(n), k=3) and random.shuffle; the letterbox branch is letterbox(s, auto=False, scaleup=True).
"""
import numpy as np

from oracle.restate_v5aug import BORDER, F32, _cvround, mixup_pixels, pipeline, warp

RESIZE_BITS = 11                   # INTER_RESIZE_COEF_BITS


def _resize_axis(ssz, dsz, clamp):
    """cv::resize's source index and 11-bit weights along one axis: fx = float((d + 0.5) * scale - 0.5),
    s = floor(fx), weights saturate_cast<short>((1 - f) * 2048), (f * 2048).  The horizontal axis (`clamp`) moves a
    position outside [0, ssz - 1) to the edge pixel with weights (2048, 0); the vertical axis keeps its weights."""
    scale = 1.0 / (dsz / ssz)
    f = ((np.arange(dsz, dtype=np.float64) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    if clamp:
        edge = (s < 0) | (s >= ssz - 1)
        f = np.where(edge, F32(0), f).astype(F32)
        s = np.where(s < 0, 0, np.where(s >= ssz - 1, ssz - 1, s))
    one = F32(1 << RESIZE_BITS)
    return s, _cvround((F32(1) - f) * one), _cvround(f * one)


def resize_linear(im, dh, dw):
    """cv2.resize(im, (dw, dh), interpolation=INTER_LINEAR) of a uint8 [h, w, 3] image, OpenCV 4.x's arithmetic: an
    exact 2x downscale is INTER_AREA ((2 x 2 sum + 2) >> 2); otherwise the horizontal pass S = src[sx] * a0 +
    src[sx + 1] * a1 in int, then VResizeLinear's 8-bit vertical pass ((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16)
    + 2 >> 2 over rows clamp(sy) and clamp(sy + 1) (its vector and scalar code compute the same)."""
    h, w = im.shape[:2]
    a = im.astype(np.int64)
    if 2 * dh == h and 2 * dw == w:
        return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    sx, a0, a1 = _resize_axis(w, dw, True)
    sy, b0, b1 = _resize_axis(h, dh, False)
    hor = a[:, sx] * a0[None, :, None] + a[:, np.minimum(sx + 1, w - 1)] * a1[None, :, None]
    S0, S1 = hor[np.clip(sy, 0, h - 1)], hor[np.clip(sy + 1, 0, h - 1)]
    out = ((((S0 >> 4) * b0[:, None, None]) >> 16) + (((S1 >> 4) * b1[:, None, None]) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def load_image(im, s):
    """load_image (augment=True): (im, (h0, w0), (h, w))."""
    h0, w0 = im.shape[:2]
    r = s / max(h0, w0)
    if r != 1:
        im = resize_linear(im, int(h0 * r), int(w0 * r))
    return im, (h0, w0), im.shape[:2]


def mosaic_rects(i, s, xc, yc, h, w):
    """load_mosaic's rectangles of quadrant i: canvas (x1a, y1a, x2a, y2a) and image (x1b, y1b, x2b, y2b)."""
    if i == 0:
        a = (max(xc - w, 0), max(yc - h, 0), xc, yc)
        b = (w - (a[2] - a[0]), h - (a[3] - a[1]), w, h)
    elif i == 1:
        a = (xc, max(yc - h, 0), min(xc + w, 2 * s), yc)
        b = (0, h - (a[3] - a[1]), min(w, a[2] - a[0]), h)
    elif i == 2:
        a = (max(xc - w, 0), yc, xc, min(2 * s, yc + h))
        b = (w - (a[2] - a[0]), 0, w, min(a[3] - a[1], h))
    else:
        a = (xc, yc, min(xc + w, 2 * s), min(2 * s, yc + h))
        b = (0, 0, min(w, a[2] - a[0]), min(a[3] - a[1], h))
    return a, b


def mosaic_canvas(loaded, s, xc, yc):
    """The 2s x 2s canvas of 114 with the four load_image outputs `loaded` placed (in shuffled order)."""
    img4 = np.full((2 * s, 2 * s, 3), BORDER, np.uint8)
    for i, im in enumerate(loaded):
        (x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b) = mosaic_rects(i, s, xc, yc, *im.shape[:2])
        img4[y1a:y2a, x1a:x2a] = im[y1b:y2b, x1b:x2b]
    return img4


def letterbox_pad(h, w, s):
    """letterbox(auto=False, scaleup=True) to s x s: ((nh, nw), (top, bottom, left, right))."""
    r = min(s / h, s / w)
    nw, nh = int(round(w * r)), int(round(h * r))
    dw, dh = (s - nw) / 2, (s - nh) / 2
    return (nh, nw), (int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1)))


def letterbox_canvas(im, s):
    """letterbox(im, s, auto=False, scaleup=True)'s image: the resize (when the size changes) padded with 114."""
    (nh, nw), (top, bottom, left, right) = letterbox_pad(*im.shape[:2], s)
    if (nh, nw) != im.shape[:2]:
        im = resize_linear(im, nh, nw)
    out = np.full((nh + top + bottom, nw + left + right, 3), BORDER, np.uint8)
    out[top:top + nh, left:left + nw] = im
    return out


def sample_pixels(sample, images, s, rgb=False):
    """One training sample of the compose kernel, restated on whole arrays from the host plan `sample`
    (yolort_b200.v5.utils.datasets.Sample; its canvases' placement keys name dataset images, or ("letterbox", i)):
    each canvas assembled in numpy, warped, mixed up, through the HSV steps and the flips; returns CHW RGB uint8."""
    outs = []
    for cv in sample.canvases:
        canvas = np.full((cv.h, cv.w, 3), BORDER, np.uint8)
        for key, y0, x0, y1, x1, oy, ox in cv.places:
            if isinstance(key, tuple):
                im = letterbox_canvas(load_image(images[key[1]], s)[0], s)[oy:, ox:]
            else:
                im = load_image(images[key], s)[0]
            canvas[y0:y1, x0:x1] = im[y0 - oy:y1 - oy, x0 - ox:x1 - ox]
        oh, ow = sample.out_h, sample.out_w
        outs.append(canvas if cv.inv is None else warp(canvas, cv.inv, oh, ow, cv.perspective))
    im = outs[0] if len(outs) == 1 else mixup_pixels(outs[0], outs[1], sample.r)
    im = pipeline(im, im.shape[0], im.shape[1], lut=sample.lut, flip_ud=sample.flip_ud, flip_lr=sample.flip_lr,
                  rgb=rgb)
    return np.ascontiguousarray(im.transpose(2, 0, 1) if rgb else im.transpose(2, 0, 1)[::-1])
