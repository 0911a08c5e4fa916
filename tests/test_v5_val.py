"""The numpy restatement of YOLOv5's rect validation batches and rescale (oracle/restate_v5val.py) against cv2 4.x,
against the reference's outputs and upstream's loader (tests/golden/v5val.npz), and the package's host-side planner
against upstream's rect block (no GPU needed)."""
import hashlib
import os

import numpy as np
import pytest

import v5val_cases as C
from oracle import restate_v5val as R
from yolort_b200.v5.utils import datasets as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v5val.npz")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _triples():
    """>= 300 seeded (h0, w0, img_size) triples: random sizes, exact 2x / other integer factors, 1-pixel outputs,
    long thin images, and COCO-like sizes at img_size 320 / 640 / 1280."""
    rng = np.random.default_rng(11)
    out = [(int(rng.integers(2, 160)), int(rng.integers(2, 160)), int(rng.integers(1, 150))) for _ in range(200)]
    out += [(4, 4, 2), (8, 6, 4), (9, 9, 3), (16, 12, 4), (640, 480, 320), (960, 1280, 640), (1920, 1440, 640),
            (2560, 1920, 1280), (300, 3, 100), (3, 300, 1), (1, 200, 50), (500, 2, 100), (2, 2, 1), (1000, 750, 640)]
    for s in (320, 640, 1280):
        for _ in range(30):
            long = int(rng.integers(s + 1, 2 * s + 300))
            short = int(rng.integers(max(2, long // 8), long + 1))
            out.append((long, short, s) if rng.random() < 0.5 else (short, long, s))
    return out


def test_resize_area_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    triples = _triples()
    assert len(triples) >= 300
    modes = set()
    for k, (h0, w0, s) in enumerate(triples):
        r = s / max(h0, w0)
        h, w = int(h0 * r), int(w0 * r)
        if h < 1 or w < 1 or r >= 1:
            continue
        im = C.image(h0, w0, k)
        modes.add(R.area_mode(h0, w0, h, w))
        got = R.resize_area(im, h, w)
        want = cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA)
        assert np.array_equal(got, want), (h0, w0, s)
    assert modes == {"general", "2x2", "int"}


def test_read_image_equals_cv2_imdecode():
    """The pixel contract: torchvision's read_image(RGB) is cv2.imdecode(IMREAD_COLOR)[..., ::-1] on the corpus."""
    cv2 = pytest.importorskip("cv2")
    import jpeg_corpus as J

    sizes = tuple(J.SMALL_SIZES) + ((480, 640),)
    files = [(n, d) for n, d, _ in J.corpus(sizes) + J.cv2_corpus(sizes)] + J.assets()
    assert len(files) >= 100
    for name, data in files:
        want = J.cpu_decode(data).permute(1, 2, 0).numpy()
        got = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]
        assert np.array_equal(want, got), name


def test_letterbox_equals_reference(gold):
    for k, (name, (h, w), kw) in enumerate(C.LETTERBOX):
        im, ratio, pad = R.letterbox(C.image(h, w, 500 + k), **kw)
        assert _sha(im) == gold[f"lb/{k}/sha256"], name
        assert np.array_equal(np.array(im.shape), gold[f"lb/{k}/shape"]), name
        assert np.array_equal(np.array(ratio, np.float64), gold[f"lb/{k}/ratio"]), name
        assert np.array_equal(np.array(pad, np.float64), gold[f"lb/{k}/pad"]), name


def test_scale_coords_equals_reference(gold):
    c = gold["sc/coords"]
    rp = gold["sc/ratio_pad"]
    ratio_pad = ((rp[0], rp[0]), (rp[1], rp[2]))
    s1, s0 = tuple(gold["sc/shape1"]), tuple(gold["sc/shape0"])
    got = R.scale_coords(s1, c.copy(), s0, ratio_pad)
    assert np.array_equal(got, gold["sc/out"], equal_nan=True)
    got = R.scale_coords(s1, c.copy(), s0, None)
    assert np.array_equal(got, gold["sc/out_auto"], equal_nan=True)
    assert np.array_equal(R.clip_coords(c.copy(), (300, 400)), gold["sc/clip"], equal_nan=True)
    assert np.array_equal(R.xywh2xyxy(gold["sc/xywh"]), gold["sc/xyxy"])


@pytest.mark.parametrize("name", sorted(C.DATASETS))
def test_rect_batches_equal_upstream(gold, name):
    sizes, s, bs, stride, _, pad = C.DATASETS[name]
    for irect, _, shapes in (R.rect_plan(sizes, s, bs, stride, pad), D.rect_batches(sizes, s, bs, stride, pad)):
        assert np.array_equal(irect, gold[f"ds/{name}/irect"])
        assert np.array_equal(shapes, gold[f"ds/{name}/batch_shapes"])


def test_rect_batches_ties_keep_numpy_order():
    sizes = [(480, 640)] * 5 + [(640, 480)] * 3 + [(480, 640)] * 4
    irect, bi, _ = D.rect_batches(sizes, 640, 4)
    s = np.array([(w, h) for h, w in sizes], np.float64)
    assert np.array_equal(irect, (s[:, 1] / s[:, 0]).argsort())
    assert list(bi) == [0] * 4 + [1] * 4 + [2] * 4


@pytest.mark.parametrize("name", sorted(C.DATASETS))
def test_getitem_equals_upstream(gold, name):
    sizes, s, _, _, _, _ = C.DATASETS[name]
    images, labels = C.dataset(name)
    for b, (idx, shape) in enumerate(C.batches(name)):
        imgs, targets, shapes = R.collate([R.getitem(images[i], labels[i], shape, s) for i in idx])
        assert [_sha(im) for im in imgs] == list(gold[f"ds/{name}/{b}/sha256"])
        assert np.array_equal(targets, gold[f"ds/{name}/{b}/targets"])
        flat = np.array([[*hw0, *g, *p] for hw0, (g, p) in shapes], np.float64)
        assert np.array_equal(flat, gold[f"ds/{name}/{b}/shapes"])


def test_load_shape_zero_side_raises():
    with pytest.raises(ValueError):
        D.load_shape(1, 2000, 640)
    with pytest.raises(ValueError):
        R.load_image(np.zeros((1, 2000, 3), np.uint8), 640)


def test_letterbox_arith_is_the_restatement():
    for _, (h, w), kw in C.LETTERBOX:
        kw = dict(kw)
        kw.pop("color", None)
        (nh, nw), ratio, pad, pads = D.letterbox_arith((h, w), **kw)
        new_unpad, ratio2, pad2, pads2 = R.letterbox_geometry((h, w), **kw)
        assert (nw, nh) == new_unpad and ratio == ratio2 and pad == pad2 and pads == pads2
