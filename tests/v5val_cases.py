"""Seeded cases of YOLOv5's rect validation batches (yolort_b200.v5.utils.datasets.val_batch, rect_batches,
augmentations.letterbox, general.scale_coords_padded) and the paths each one reaches (host logic, no GPU needed)."""
import numpy as np

from oracle import restate_v5val as R

# name: (image sizes (h, w), img_size, batch_size, stride, seed, pad)
DATASETS = {
    "mixed": ([(480, 640), (640, 480), (750, 1000), (1280, 960), (1440, 1920), (300, 200), (640, 640), (123, 457),
               (457, 123), (1000, 999), (97, 1300), (640, 427)], 640, 4, 32, 1, 0.5),
    "landscape": ([(480, 640), (375, 500), (333, 500), (960, 1280), (427, 640), (200, 201)], 320, 3, 32, 2, 0.5),
    "portrait": ([(640, 480), (500, 375), (500, 333), (1280, 960), (801, 600)], 320, 2, 32, 3, 0.5),
    "p6": ([(720, 1280), (1080, 1920), (640, 480), (1300, 97), (512, 512), (999, 1000), (1200, 900)], 1280, 3, 64, 4, 0.5),
    "no pad": ([(480, 640), (960, 1280), (640, 480), (512, 512)], 640, 2, 32, 5, 0.0),
}

# letterbox(im, new_shape, auto, scale_fill, scaleup, stride) cases on images of (h, w)
LETTERBOX = [
    ("auto shrink", (480, 640), dict(new_shape=(320, 320), auto=True)),
    ("auto grow", (97, 130), dict(new_shape=640, auto=True)),
    ("square shrink", (750, 1000), dict(new_shape=(640, 640), auto=False)),
    ("square grow", (100, 75), dict(new_shape=(256, 256), auto=False)),
    ("no scaleup", (100, 75), dict(new_shape=(256, 256), auto=False, scaleup=False)),
    ("scale_fill", (300, 500), dict(new_shape=(256, 320), auto=False, scale_fill=True)),
    ("auto stride 64", (500, 333), dict(new_shape=(640, 640), auto=True, stride=64)),
    ("exact 2x", (512, 640), dict(new_shape=(320, 320), auto=True)),
    ("odd pads", (101, 200), dict(new_shape=(203, 203), auto=False)),
    ("colour", (60, 90), dict(new_shape=(96, 96), auto=False, color=(0, 10, 255))),
]


def image(h, w, seed):
    """A seeded BGR uint8 [h, w, 3] image with smooth structure and noise (area averages of it are not constant)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = (np.sin(x / 7.0 + seed)[..., None] * 60 + np.cos(y / 5.0)[..., None] * 50 + 128)
    return np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)


def labels_for(n_img, seed):
    rng = np.random.default_rng(1000 + seed)
    out = []
    for _ in range(n_img):
        k = int(rng.integers(0, 5))
        xy = rng.uniform(0.05, 0.95, (k, 2))
        wh = rng.uniform(0.02, 0.6, (k, 2))
        out.append(np.concatenate([rng.integers(0, 80, (k, 1)), xy, wh], 1).astype(np.float32))
    return out


def dataset(name):
    sizes, img_size, bs, stride, seed, _ = DATASETS[name]
    return [image(h, w, seed * 100 + i) for i, (h, w) in enumerate(sizes)], labels_for(len(sizes), seed)


def batches(name):
    """[(indices into the dataset, (H, W))] in upstream's order."""
    sizes, img_size, bs, stride, _, pad = DATASETS[name]
    irect, bi, shapes = R.rect_plan(sizes, img_size, bs, stride, pad)
    return [([int(i) for i in irect[bi == k]], tuple(int(v) for v in shapes[k])) for k in range(len(shapes))]


def load_path(h0, w0, s):
    r = s / max(h0, w0)
    if r == 1:
        return "no resize"
    h, w = int(h0 * r), int(w0 * r)
    if r > 1:
        return "linear up-scale"
    return {"2x2": "area 2x2", "int": "area other integer", "general": "area general"}[R.area_mode(h0, w0, h, w)]


def _pad_paths(pads):
    out = set()
    for side, p in zip(("top", "bottom", "left", "right"), pads):
        out.add(f"{'zero' if p == 0 else 'odd' if p % 2 else 'even'} pad {side}")
    return out


def paths():
    """Every path the case tables reach."""
    out = set()
    for name, (sizes, s, bs, stride, _, pad) in DATASETS.items():
        if stride == 64:
            out.add("stride 64")
        if len(sizes) % bs:
            out.add("partial last batch")
        for h0, w0 in sizes:
            out.add(load_path(h0, w0, s))
        irect, _, shapes = R.rect_plan(sizes, s, bs, stride, pad)
        ar = np.array([h / w for h, w in sizes])[irect]
        for k in range(len(shapes)):
            a = ar[k * bs:(k + 1) * bs]
            out.add("landscape batch" if a.max() < 1 else "portrait batch" if a.min() > 1 else "mixed batch")
        for idx, (H, W) in batches(name):
            for i in idx:
                h0, w0 = sizes[i]
                r = s / max(h0, w0)
                h, w = (int(h0 * r), int(w0 * r)) if r != 1 else (h0, w0)
                _, _, _, pads = R.letterbox_geometry((h, w), (H, W), auto=False, scaleup=False)
                out |= _pad_paths(pads)
    for _, (h, w), kw in LETTERBOX:
        kw = dict(kw)
        kw.pop("color", None)
        new_unpad, _, _, pads = R.letterbox_geometry((h, w), **kw)
        if new_unpad != (w, h):
            out.add("letterbox resize, " + ("scale_fill" if kw.get("scale_fill") else "auto" if kw.get("auto", True)
                                            else "fixed"))
        out |= {"letterbox " + p for p in _pad_paths(pads)}
    return out
