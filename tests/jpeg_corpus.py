"""Seeded JPEG corpus for the decoder tests: files are generated at test time with PIL (and cv2 where present), so
only the two camera files under tests/golden/jpeg are committed."""
import hashlib
import io
import os

import numpy as np
import torch

GOLDEN_JPEG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
ASSETS = ("bus.jpg", "zidane.jpg")

SMALL_SIZES = ((1, 1), (7, 9), (61, 117))
LARGE_SIZES = ((480, 640), (1536, 2048))
QUALITIES = (50, 75, 90, 100)


def photo(h: int, w: int, seed: int) -> np.ndarray:
    """[h, w, 3] uint8: smooth structure plus noise and a few hard edges, so every quality keeps AC energy."""
    from PIL import Image

    r = np.random.default_rng(seed)
    base = r.integers(0, 256, (max(1, h // 8 + 1), max(1, w // 8 + 1), 3)).astype(np.uint8)
    a = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR)).astype(np.int32)
    a = a + r.integers(-24, 25, (h, w, 3))
    if h > 4 and w > 4:
        a[h // 3: h // 2, w // 4: w // 2] = 255          # saturated block edges: the IDCT's range limit is exercised
        a[h // 2: 2 * h // 3, w // 2:] = 0
    return np.clip(a, 0, 255).astype(np.uint8)


def pil_jpeg(a: np.ndarray, gray=False, **kw) -> bytes:
    from PIL import Image

    im = Image.fromarray(a)
    if gray:
        im = im.convert("L")
        kw.pop("subsampling", None)
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def corpus(sizes=SMALL_SIZES):
    """(name, bytes, expected) for every size x quality x subsampling, plus gray, optimised-table and restart-marker
    variants; `expected` holds the geometry the parser must report."""
    out = []
    for (h, w) in sizes:
        a = photo(h, w, 1000 * h + w)
        for q in QUALITIES:
            for ss in (0, 1, 2):
                samp = {0: [(1, 1)] * 3, 1: [(2, 1), (1, 1), (1, 1)], 2: [(2, 2), (1, 1), (1, 1)]}[ss]
                out.append((f"{h}x{w}_q{q}_ss{ss}", pil_jpeg(a, quality=q, subsampling=ss),
                            dict(width=w, height=h, components=3, sampling=samp, restart_interval=0)))
            out.append((f"{h}x{w}_q{q}_gray", pil_jpeg(a, gray=True, quality=q),
                        dict(width=w, height=h, components=1, sampling=[(1, 1)], restart_interval=0)))
        out.append((f"{h}x{w}_opt", pil_jpeg(a, quality=85, subsampling=2, optimize=True),
                    dict(width=w, height=h, components=3, sampling=[(2, 2), (1, 1), (1, 1)], restart_interval=0)))
        out.append((f"{h}x{w}_rst3", pil_jpeg(a, quality=90, subsampling=2, restart_marker_blocks=3),
                    dict(width=w, height=h, components=3, sampling=[(2, 2), (1, 1), (1, 1)], restart_interval=3)))
        out.append((f"{h}x{w}_rst1_gray", pil_jpeg(a, gray=True, quality=95, restart_marker_blocks=1),
                    dict(width=w, height=h, components=1, sampling=[(1, 1)], restart_interval=1)))
        out.append((f"{h}x{w}_rstrow_opt", pil_jpeg(a, quality=75, subsampling=1, optimize=True, restart_marker_rows=1),
                    dict(width=w, height=h, components=3, sampling=[(2, 1), (1, 1), (1, 1)], restart_interval=None)))
    return out


def cv2_corpus(sizes=SMALL_SIZES):
    """cv2 (libjpeg-turbo) files with DRI, in the three samplings; empty without cv2."""
    try:
        import cv2
    except ImportError:
        return []
    out = []
    for (h, w) in sizes:
        a = photo(h, w, 7 * h + w)
        for rst in (1, 4):
            for name, ss, samp in (("444", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, [(1, 1)] * 3),
                                   ("422", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422, [(2, 1), (1, 1), (1, 1)]),
                                   ("420", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, [(2, 2), (1, 1), (1, 1)])):
                ok, enc = cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_QUALITY, 92, cv2.IMWRITE_JPEG_RST_INTERVAL, rst,
                                                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR, ss])
                assert ok
                out.append((f"cv2_{h}x{w}_rst{rst}_{name}", enc.tobytes(),
                            dict(width=w, height=h, components=3, sampling=samp, restart_interval=rst)))
    return out


def assets():
    out = []
    for name in ASSETS:
        with open(os.path.join(GOLDEN_JPEG, name), "rb") as f:
            out.append((name, f.read()))
    return out


def progressive(seed=3) -> bytes:
    return pil_jpeg(photo(40, 56, seed), quality=80, progressive=True)


def cmyk(seed=4) -> bytes:
    from PIL import Image

    b = io.BytesIO()
    Image.fromarray(photo(24, 32, seed)).convert("CMYK").save(b, "JPEG", quality=80)
    return b.getvalue()


def cpu_decode(data: bytes) -> torch.Tensor:
    from torchvision.io import ImageReadMode, decode_jpeg

    return decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), mode=ImageReadMode.RGB)


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def scan_segment(data: bytes):
    """(begin, end) of the entropy-coded segment: after the SOS header, up to the EOI marker."""
    i = data.index(b"\xff\xda")
    begin = i + 2 + (data[i + 2] << 8 | data[i + 3])
    return begin, data.rindex(b"\xff\xd9")
