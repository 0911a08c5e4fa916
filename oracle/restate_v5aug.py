"""Numpy restatement of csrc/v5_augment.cu: YOLOv5's augment_hsv / random_perspective / cutout / mixup pixels as
OpenCV 4.x computes them (cv2.warpAffine, cv2.warpPerspective, cv2.cvtColor BGR<->HSV, cv2.LUT), written from the
arithmetic alone (no cv2 import).  Images are uint8 [H, W, 3] arrays.

    warp      OpenCV's fixed-point remap: inverse map; affine coordinates in AB_BITS = 10 fixed point with a
              round delta of 16, perspective coordinates as cvRound(X * (32 / W)) in double; INTER_BITS = 5 sub-pixel
              bits; 15-bit bilinear weights, (sum + 2^14) >> 15; every tap outside the image reads the border value
    to_hsv    RGB2HSV_b: hsv_shift = 12 with sdiv_table / hdiv_table180 (exact integers)
    lut       the per-channel 256-entry tables
    from_hsv  HSV2RGB_b, fp32: each row's first floor(w / 32) * 32 pixels take the vector path (fused
              v * fma(-s, h, 1), truncation), the rest the scalar path (fmod / floor sector, the same fused products,
              round half to even).  32 = 4 vectors of 8 lanes: the split of OpenCV's x86 AVX2 build.
"""
import numpy as np

F32 = np.float32
BORDER = 114
HSV_SHIFT = 12
HSV_VEC = 32                       # pixels per vector step of HSV2RGB_b (4 x v_float32 of 8 lanes)
SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def _cvround(x):
    return np.rint(x).astype(np.int64)          # cvRound: round half to even


# -- geometry ----------------------------------------------------------------------------------------------------
def invert_affine(M):
    """warpAffine's inverse of a 2x3 map (imgwarp.cpp: invertAffineTransform, in place on a copy)."""
    M = [float(v) for v in np.asarray(M, np.float64).reshape(-1)[:6]]
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0], M[1], M[3], M[4] = A11, M[1] * -D, M[3] * -D, A22
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return np.array(M, np.float64)


def invert_perspective(M):
    """cv::invert(DECOMP_LU) of a 3x3 double matrix: the closed form OpenCV takes for n == 3."""
    S = np.asarray(M, np.float64).reshape(3, 3)
    s = lambda i, j: float(S[i, j])  # noqa: E731
    d = (s(0, 0) * (s(1, 1) * s(2, 2) - s(1, 2) * s(2, 1)) - s(0, 1) * (s(1, 0) * s(2, 2) - s(1, 2) * s(2, 0)) +
         s(0, 2) * (s(1, 0) * s(2, 1) - s(1, 1) * s(2, 0)))
    if d == 0.0:
        return np.zeros(9, np.float64)
    d = 1.0 / d
    t = [(s(1, 1) * s(2, 2) - s(1, 2) * s(2, 1)) * d, (s(0, 2) * s(2, 1) - s(0, 1) * s(2, 2)) * d,
         (s(0, 1) * s(1, 2) - s(0, 2) * s(1, 1)) * d, (s(1, 2) * s(2, 0) - s(1, 0) * s(2, 2)) * d,
         (s(0, 0) * s(2, 2) - s(0, 2) * s(2, 0)) * d, (s(0, 2) * s(1, 0) - s(0, 0) * s(1, 2)) * d,
         (s(1, 0) * s(2, 1) - s(1, 1) * s(2, 0)) * d, (s(0, 1) * s(2, 0) - s(0, 0) * s(2, 1)) * d,
         (s(0, 0) * s(1, 1) - s(0, 1) * s(1, 0)) * d]
    return np.array(t, np.float64)


def perspective_block_w(h, w):
    """The width of WarpPerspectiveInvoker's pixel blocks (BLOCK_SZ = 32): coordinates are summed from each block's
    first column."""
    bh0 = min(16, h)
    return min(1024 // bh0, w)


def source_coords(inv, out_h, out_w, perspective):
    """Fixed-point source coordinates of every output pixel: integer (sy, sx) of the top-left tap and the 5-bit
    fractions (ay, ax)."""
    y = np.arange(out_h, dtype=np.float64)[:, None]
    x = np.arange(out_w, dtype=np.float64)[None, :]
    m = inv
    if perspective:
        bw = perspective_block_w(out_h, out_w)
        xb = np.floor(x / bw) * bw
        x1 = x - xb
        X0 = m[0] * xb + m[1] * y + m[2]
        Y0 = m[3] * xb + m[4] * y + m[5]
        W0 = m[6] * xb + m[7] * y + m[8]
        W = W0 + m[6] * x1
        with np.errstate(divide="ignore"):
            W = np.where(W != 0, 32.0 / np.where(W != 0, W, 1.0), 0.0)
        lo, hi = float(np.iinfo(np.int32).min), float(np.iinfo(np.int32).max)
        fX = np.maximum(lo, np.minimum(hi, (X0 + m[0] * x1) * W))
        fY = np.maximum(lo, np.minimum(hi, (Y0 + m[3] * x1) * W))
        X, Y = _cvround(fX), _cvround(fY)
    else:
        adelta = _cvround(m[0] * x * 1024)
        bdelta = _cvround(m[3] * x * 1024)
        X0 = _cvround((m[1] * y + m[2]) * 1024) + 16
        Y0 = _cvround((m[4] * y + m[5]) * 1024) + 16
        X = (X0 + adelta) >> 5
        Y = (Y0 + bdelta) >> 5
    sx = np.clip(X >> 5, -32768, 32767)
    sy = np.clip(Y >> 5, -32768, 32767)
    return sy, sx, Y & 31, X & 31


def warp(im, inv, out_h, out_w, perspective, border=BORDER):
    """cv2.warpAffine / cv2.warpPerspective(INTER_LINEAR, BORDER_CONSTANT) given the inverse map `inv`."""
    h, w = im.shape[:2]
    sy, sx, ay, ax = source_coords(inv, out_h, out_w, perspective)
    acc = np.zeros((out_h, out_w, 3), np.int64)
    for dy, wy in ((0, 32 - ay), (1, ay)):
        for dx, wx in ((0, 32 - ax), (1, ax)):
            ty, tx = sy + dy, sx + dx
            inside = (ty >= 0) & (ty < h) & (tx >= 0) & (tx < w)
            v = im[np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)].astype(np.int64)
            v[~inside] = border
            acc += v * ((wy * wx) << 5)[..., None]
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


# -- colour ------------------------------------------------------------------------------------------------------
def hsv_tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, _cvround((255 << HSV_SHIFT) / np.maximum(i, 1)), 0)
        hdiv = np.where(i > 0, _cvround((180 << HSV_SHIFT) / (6.0 * np.maximum(i, 1))), 0)
    return sdiv, hdiv


def to_hsv(im, rgb=False):
    """cv2.cvtColor(im, COLOR_BGR2HSV) (COLOR_RGB2HSV with rgb=True)."""
    sdiv, hdiv = hsv_tables()
    a = im.astype(np.int64)
    b, g, r = (a[..., 2], a[..., 1], a[..., 0]) if rgb else (a[..., 0], a[..., 1], a[..., 2])
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * sdiv[v] + (1 << (HSV_SHIFT - 1))) >> HSV_SHIFT
    hh = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    hh = (hh * hdiv[diff] + (1 << (HSV_SHIFT - 1))) >> HSV_SHIFT
    hh = np.where(hh < 0, hh + 180, hh)
    return np.stack([hh, s, v], -1).astype(np.uint8)


def _fma_f32(a, b, c):
    """fp32 fma(a, b, c): the product of two fp32 values is exact in double, so one rounding of a*b + c to fp32
    is a double sum rounded once (the double sum itself is exact here: |a*b| <= 1 and c == 1)."""
    return (a.astype(np.float64) * b.astype(np.float64) + np.float64(c)).astype(F32)


def from_hsv(hsv, rgb=False, row_x=None, row_w=None):
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) (COLOR_HSV2RGB with rgb=True) of a [H, W, 3] array whose rows OpenCV converts
    one by one.  `row_x` / `row_w` give each pixel's column and the row length when they differ from the array's own
    (the kernel converts pixels that a flip moved)."""
    H, W = hsv.shape[:2]
    if row_x is None:
        row_x = np.broadcast_to(np.arange(W)[None, :], (H, W))
        row_w = W
    vec = row_x < (row_w // HSV_VEC) * HSV_VEC
    h = hsv[..., 0].astype(F32) * (F32(6.0) / F32(180))
    s = hsv[..., 1].astype(F32) * F32(1.0 / 255.0)
    v = hsv[..., 2].astype(F32) * F32(1.0 / 255.0)
    one = F32(1)
    # vector path: sector from trunc, no fmod (h < 180 keeps it below 6)
    pre = np.trunc(h).astype(F32)
    sec_v = (pre - np.trunc(pre * F32(1.0 / 6.0)).astype(F32) * F32(6)).astype(np.int64)
    # scalar path
    hs = np.fmod(h, F32(6)).astype(F32)
    sec_s = np.floor(hs).astype(np.int64)
    bad = (sec_s < 0) | (sec_s >= 6)
    frac_s = np.where(bad, F32(0), hs - sec_s.astype(F32)).astype(F32)
    sec_s = np.where(bad, 0, sec_s)
    sec = np.where(vec, sec_v, sec_s)
    frac = np.where(vec, (h - pre).astype(F32), frac_s).astype(F32)
    tab = np.stack([v, v * (one - s), v * _fma_f32(-s, frac, 1.0), v * _fma_f32(-s, (one - frac).astype(F32), 1.0)],
                   -1)
    out = np.take_along_axis(tab, SECTOR[sec], -1)           # (b, g, r)
    out = np.where((~vec & (hsv[..., 1] == 0))[..., None], v[..., None], out).astype(F32) * F32(255)
    q = np.where(vec[..., None], np.trunc(out), np.rint(out))
    q = np.clip(q, 0, 255).astype(np.uint8)
    return q[..., ::-1].copy() if rgb else q


def hsv_gains_lut(r):
    """augment_hsv's tables for gains r (float64 [3]), the reference's expressions."""
    x = np.arange(0, 256, dtype=r.dtype)
    lut_hue = ((x * r[0]) % 180).astype(np.uint8)
    lut_sat = np.clip(x * r[1], 0, 255).astype(np.uint8)
    lut_val = np.clip(x * r[2], 0, 255).astype(np.uint8)
    return np.stack([lut_hue, lut_sat, lut_val])


# -- the kernel's pipeline -----------------------------------------------------------------------------------------
def pipeline(src, out_h, out_w, inv=None, perspective=False, lut=None, to_hsv_op=None, from_hsv_op=None,
             flip_ud=False, flip_lr=False, rects=(), rgb=False):
    """One image of v5_augment_kernel: output pixel (y, x) maps back through the flips, then through the inverse
    warp (or reads src at the same place), then runs to_hsv -> lut -> from_hsv (each when present), then the last
    cutout rectangle (y0, x0, y1, x1, (c0, c1, c2)) that holds (y, x) sets it.  With `lut` the three colour steps
    default to on."""
    to_hsv_op = lut is not None if to_hsv_op is None else to_hsv_op
    from_hsv_op = lut is not None if from_hsv_op is None else from_hsv_op
    if inv is not None:
        im = warp(src, inv, out_h, out_w, perspective)
    else:
        assert src.shape[:2] == (out_h, out_w)
        im = src.copy()
    if to_hsv_op:
        im = to_hsv(im, rgb)
    if lut is not None:
        im = np.stack([lut[c][im[..., c]] for c in range(3)], -1)
    if from_hsv_op:
        im = from_hsv(im, rgb)
    if flip_ud:
        im = im[::-1]
    if flip_lr:
        im = im[:, ::-1]
    im = np.ascontiguousarray(im)
    for y0, x0, y1, x1, c in rects:
        im[y0:y1, x0:x1] = c
    return im


def mixup_pixels(im, im2, r):
    """mixup's (im * r + im2 * (1 - r)).astype(uint8) in float64."""
    return (im * r + im2 * (1 - r)).astype(np.uint8)


def all_bgr_image():
    """Every 24-bit triple once, as a 4096 x 4096 image: pixel k holds (k & 255, (k >> 8) & 255, k >> 16)."""
    k = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([k & 255, (k >> 8) & 255, k >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)


def all_hsv_image(width=256):
    """Every valid (h < 180, s, v) triple once, h-major then s then v, as rows of `width` pixels."""
    k = np.arange(180 * 256 * 256, dtype=np.uint32)
    return np.stack([k >> 16, (k >> 8) & 255, k & 255], -1).astype(np.uint8).reshape(-1, width, 3)
