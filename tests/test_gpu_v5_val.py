"""YOLOv5's rect validation batches and val.run on the GPU, bit for bit against the restatement
(oracle/restate_v5val.py), the fixtures (tests/golden/v5val.npz) and the host composition of val.py."""
import hashlib
import os

import numpy as np
import pytest
import torch

import v5val_cases as C
from oracle import restate_v5metrics as RM
from oracle import restate_v5val as R
from yolort_b200 import _C
from yolort_b200.v5 import val as V
from yolort_b200.v5.utils import augmentations as A
from yolort_b200.v5.utils import datasets as D
from yolort_b200.v5.utils import general as G

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v5val.npz")
KEYS = ("mp", "mr", "map50", "map", "maps", "p", "r", "ap50", "ap", "f1", "ap_class", "nt", "fitness")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _strided(im):
    """The image as a strided CUDA view: a window of a padded buffer with 4 bytes per pixel (row and pixel padding)."""
    h, w = im.shape[:2]
    big = torch.zeros((h + 3, w + 5, 4), dtype=torch.uint8, device=DEV)
    big[1:h + 1, 2:w + 2, :3] = torch.from_numpy(im).to(DEV)
    view = big[1:h + 1, 2:w + 2, :3]
    assert not view.is_contiguous() and view.stride() == ((w + 5) * 4, 4, 1)
    return view


def _planar(im):
    """The image as the HWC view of planar CHW memory (channel stride h * w), as decode_jpeg returns it."""
    view = torch.from_numpy(np.ascontiguousarray(im.transpose(2, 0, 1))).to(DEV).permute(1, 2, 0)
    assert view.stride(2) == im.shape[0] * im.shape[1]
    return view


def _sources(im):
    return (torch.from_numpy(im).to(DEV), _strided(im), _planar(im))


def test_load_image_area_equals_restatement():
    rng = np.random.default_rng(5)
    cases = [(750, 1000, 640), (960, 1280, 640), (1440, 1920, 640), (1300, 97, 640), (999, 1000, 320),
             (300, 200, 640), (640, 480, 640), (2560, 1920, 1280), (200, 7, 64), (5, 300, 60)]
    cases += [(int(rng.integers(20, 500)), int(rng.integers(20, 500)), int(rng.integers(16, 300))) for _ in range(40)]
    for k, (h0, w0, s) in enumerate(cases):
        im = C.image(h0, w0, k)
        want, _, hw = R.load_image(im, s, augment=False)
        for src in _sources(im):
            got, hw0, got_hw = D.load_image(src, s, augment=False)
            assert got_hw == hw and hw0 == (h0, w0)
            assert np.array_equal(got.cpu().numpy(), want), (h0, w0, s)
        # augment=True keeps INTER_LINEAR
        got, _, _ = D.load_image(torch.from_numpy(im).to(DEV), s)
        assert np.array_equal(got.cpu().numpy(), R.load_image(im, s, augment=True)[0])


def test_load_image_area_on_decoded_jpeg():
    from yolort_b200.io import decode_jpeg

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")
    for name in ("bus.jpg", "zidane.jpg"):
        with open(os.path.join(root, name), "rb") as f:
            data = f.read()
        t = decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), device=DEV)
        hwc = t.permute(1, 2, 0) if t.shape[0] == 3 else t
        im = hwc.cpu().numpy()
        for s in (320, 640):
            got = D.load_image(hwc, s, augment=False)[0]
            assert np.array_equal(got.cpu().numpy(), R.load_image(im, s, augment=False)[0]), (name, s)


def test_zero_side_raises():
    with pytest.raises(ValueError):
        D.load_image(torch.zeros((1, 2000, 3), dtype=torch.uint8, device=DEV), 640, augment=False)


def test_letterbox_equals_reference():
    z = np.load(GOLDEN)
    for k, (name, (h, w), kw) in enumerate(C.LETTERBOX):
        im = C.image(h, w, 500 + k)
        for src in _sources(im):
            out, ratio, pad = A.letterbox(src, **kw)
            assert _sha(out.cpu().numpy()) == z[f"lb/{k}/sha256"], name
            assert np.array_equal(np.array(ratio, np.float64), z[f"lb/{k}/ratio"]), name
            assert np.array_equal(np.array(pad, np.float64), z[f"lb/{k}/pad"]), name


@pytest.mark.parametrize("name", sorted(C.DATASETS))
@pytest.mark.parametrize("order", ["bgr", "rgb"])
def test_val_batch_equals_fixture(name, order):
    z = np.load(GOLDEN)
    sizes, s, _, _, _, _ = C.DATASETS[name]
    images, labels = C.dataset(name)
    dev_images = [_strided(im) if order == "bgr" else _planar(np.ascontiguousarray(im[..., ::-1])) for im in images]
    for b, (idx, shape) in enumerate(C.batches(name)):
        imgs, targets, shapes = D.val_batch(dev_images, labels, idx, shape, s, channel_order=order)
        got = imgs.cpu().numpy()
        assert [_sha(im) for im in got] == list(z[f"ds/{name}/{b}/sha256"]), (name, b)
        assert np.array_equal(targets.cpu().numpy(), z[f"ds/{name}/{b}/targets"])
        flat = np.array([[*hw0, *g, *p] for hw0, (g, p) in shapes], np.float64)
        assert np.array_equal(flat, z[f"ds/{name}/{b}/shapes"])


def _guarded(n):
    """n bytes inside a buffer of 0xA5 sentinels: (buffer, view)."""
    buf = torch.full((n + 256,), 0xA5, dtype=torch.uint8, device=DEV)
    return buf, buf[128:128 + n]


def _sentinels_intact(buf):
    return bool((buf[:128] == 0xA5).all()) and bool((buf[-128:] == 0xA5).all())


def test_outputs_leave_sentinels_untouched():
    # the area kernel: every job's destination between sentinels
    cases = [(750, 1000, 480, 640), (960, 1280, 480, 640), (1440, 1920, 480, 640), (301, 97, 63, 20)]
    jobs = (_C.V5ResizeJob * len(cases))()
    keep, want = [], []
    for k, (j, (h0, w0, h, w)) in enumerate(zip(jobs, cases)):
        im = C.image(h0, w0, 40 + k)
        src = _strided(im)
        buf, dst = _guarded(h * w * 3)
        j.src, j.dst = src.data_ptr(), dst.data_ptr()
        j.src_stride_y, j.src_stride_x, j.src_stride_c = (int(v) for v in src.stride())
        j.src_h, j.src_w, j.dst_h, j.dst_w = h0, w0, h, w
        keep += [src, buf, dst]
        want.append((buf, dst, R.resize_area(im, h, w)))
    _C.v5_resize(jobs, keep, DEV, area=True)
    for buf, dst, ref in want:
        assert np.array_equal(dst.view(ref.shape).cpu().numpy(), ref)
        assert _sentinels_intact(buf)
    # the compose launch of val_batch: the batch output between sentinels
    name = "mixed"
    z = np.load(GOLDEN)
    sizes, s, _, _, _, _ = C.DATASETS[name]
    images, labels = C.dataset(name)
    dev_images = [torch.from_numpy(im).to(DEV) for im in images]
    for b, (idx, (H, W)) in enumerate(C.batches(name)):
        plan = D.ValPlan(dev_images, labels, idx, (H, W), s)
        plan.resize()
        buf, flat = _guarded(len(idx) * 3 * H * W)
        plan.compose(flat.view(len(idx), 3, H, W))
        got = flat.view(len(idx), 3, H, W).cpu().numpy()
        assert [_sha(im) for im in got] == list(z[f"ds/{name}/{b}/sha256"])
        assert _sentinels_intact(buf)
    # the rescale writes counts[i] boxes of image i and nothing past them
    n, d = 3, 8
    boxes = torch.full((n, d, 4), -7.0, device=DEV)
    fresh = torch.rand((n, 2, 4), device=DEV) * 600
    boxes[:, :2] = fresh
    counts = torch.tensor([2, 0, 1], dtype=torch.int32, device=DEV)
    params = torch.tensor([[0.5, 3.0, 4.0, 480.0, 640.0]] * n, device=DEV)
    G.scale_coords_padded(boxes, counts, params)
    b = boxes.cpu()
    assert bool((b[0, 2:] == -7).all()) and bool((b[1, 2:] == -7).all()) and bool((b[1, :2] == fresh[1].cpu()).all())
    assert bool((b[2, 1] == fresh[2, 1].cpu()).all()) and bool((b[2, 2:] == -7).all())


def test_scale_coords_padded_equals_restatement_and_torch():
    rng = np.random.default_rng(3)
    n, d = 5, 40
    boxes = rng.uniform(-30, 700, (n, d, 4)).astype(np.float32)
    boxes[1, 3, 2] = np.nan
    counts = np.array([40, 0, 17, 1, 33], np.int32)
    shapes = [((int(rng.integers(100, 1500)), int(rng.integers(100, 1500))),
               ((float(rng.uniform(0.2, 1)), 0.0), (float(rng.uniform(0, 40)), float(rng.uniform(0, 40)))))
              for _ in range(n)]
    shapes = [(hw, ((g, g), p)) for hw, ((g, _), p) in shapes]
    H, W = 480, 672
    tg = [np.concatenate([np.full((k, 1), i, np.float32), rng.integers(0, 80, (k, 1)),
                          rng.uniform(0, 1, (k, 4))], 1).astype(np.float32) for i, k in enumerate((3, 0, 5, 1, 2))]
    targets = np.concatenate(tg)
    tb = torch.from_numpy(boxes).to(DEV)
    native = G.scale_coords_padded(tb, torch.from_numpy(counts), G.rescale_params(shapes, DEV),
                                   torch.from_numpy(targets).to(DEV), (H, W))
    want = R.boxes_native(boxes, counts, (H, W), shapes)
    assert np.array_equal(tb.cpu().numpy(), want, equal_nan=True)
    assert np.array_equal(native.cpu().numpy(), R.targets_native(targets, (H, W), shapes))
    # the single-image helpers run torch's own ops on the device, whose division by a python scalar may differ from
    # the correctly rounded quotient in the last place
    def close(a, b):
        a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
        both = np.isnan(a) & np.isnan(b)
        return bool(np.all(both | (np.abs(a - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b))))))

    for i in range(n):
        c = torch.from_numpy(boxes[i, :counts[i]].copy()).to(DEV)
        G.scale_coords((H, W), c, shapes[i][0], shapes[i][1])
        assert close(c.cpu().numpy(), want[i, :counts[i]])
    t = torch.from_numpy(targets).to(DEV)
    t[:, 2:] *= torch.tensor([W, H, W, H], dtype=torch.float32, device=DEV)
    for i in range(n):
        m = t[:, 0] == i
        tbox = G.xywh2xyxy(t[m, 2:6])
        G.scale_coords((H, W), tbox, shapes[i][0], shapes[i][1])
        assert close(tbox.cpu().numpy(), native[m, 2:6].cpu().numpy())


# -- val.run ---------------------------------------------------------------------------------------------------------
def _model(size):
    import parity_util as util
    from yolort_b200.models import yolov5n, yolov5n6

    ctor = {"n": yolov5n, "n6": yolov5n6}[size]
    sd = util.synth_state_dict(util.layouts()[size], knob_obj=7.0, knob_cls=4.5, seed=0,
                               gain=util.GAIN_N6 if size == "n6" else 2.0)
    m = ctor(score_thresh=0.25, nms_thresh=0.45, detections_per_img=100).eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def _set(n_img, seed, nc=80):
    rng = np.random.default_rng(seed)
    sizes = []
    for _ in range(n_img):
        long = int(rng.integers(200, 900))
        short = int(long * rng.uniform(0.4, 1.0))
        sizes.append((long, short) if rng.random() < 0.4 else (short, long))
    images = [C.image(h, w, seed * 1000 + i) for i, (h, w) in enumerate(sizes)]
    labels = C.labels_for(n_img, seed)
    for lab in labels:
        lab[:, 0] = np.mod(lab[:, 0], nc)
    return images, labels


def _host_composition(yolo, images, labels, batch_size, img_size, conf, iou, max_det, pad=0.5):
    """val.py composed on the host: the same model's detections per rect batch (plan + decode_nms on its stored
    logits), the restated rescale, the restated metrics."""
    stride = int(max(yolo.anchor_generator.strides))
    irect, bi, shapes_b = R.rect_plan([im.shape[:2] for im in images], img_size, batch_size, stride, pad)
    pc = yolo.post_config()
    per_image = []
    for k in range(len(shapes_b)):
        idx = [int(i) for i in irect[bi == k]]
        H, W = (int(v) for v in shapes_b[k])
        imgs, targets, shapes = R.collate([R.getitem(images[i], labels[i], (H, W), img_size) for i in idx])
        plan = yolo.engine().plan(len(idx), H, W)
        yolo._write_samples(plan, torch.from_numpy(imgs).to(DEV))
        plan.run()
        dets = _C.decode_nms(plan.heads, "nhwc", pc["strides"], pc["anchors_px"], conf, iou, max_det,
                             pc["semantics"], num_classes=yolo.num_classes)
        tn = R.targets_native(targets, (H, W), shapes)
        for si, dt in enumerate(dets):
            c = int(dt["scores"].shape[0])
            b = R.boxes_native(dt["boxes"].cpu().numpy()[None], [c], (H, W), [shapes[si]])[0]
            det = np.concatenate([b, dt["scores"].cpu().numpy()[:, None],
                                  dt["labels"].cpu().numpy()[:, None].astype(np.float32)], 1).astype(np.float32)
            per_image.append((det, tn[tn[:, 0] == si, 1:]))
    return RM.val_metrics(per_image, yolo.num_classes)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("size,img_size,n_img", [("n", 320, 100), ("n6", 512, 24)])
def test_run_equals_host_composition(size, img_size, n_img):
    m = _model(size)
    pp = m.model.post_process
    images, labels = _set(n_img, 7 if size == "n" else 8)
    before = (pp.score_thresh, pp.nms_thresh, pp.detections_per_img)
    got = V.run(m, [torch.from_numpy(im).to(DEV) for im in images], labels, batch_size=16, img_size=img_size,
                conf_thres=0.001, iou_thres=0.6, max_det=300)
    want = _host_composition(m.model, images, labels, 16, img_size, 0.001, 0.6, 300)
    for k in KEYS:
        assert _same(got[k], want[k]), k
    assert (pp.score_thresh, pp.nms_thresh, pp.detections_per_img) == before
    # a bare YOLO runs the same loop
    got2 = V.run(m.model, [torch.from_numpy(im).to(DEV) for im in images], labels, batch_size=16,
                 img_size=img_size)
    for k in KEYS:
        assert _same(got2[k], got[k]), k


def test_run_on_paths_equals_run_on_decoded(tmp_path):
    cv2 = pytest.importorskip("cv2")

    m = _model("n")
    images, labels = _set(12, 9)
    paths = []
    for i, im in enumerate(images):
        p = str(tmp_path / (f"{i}.jpg" if i % 3 else f"{i}.png"))
        cv2.imwrite(p, im)
        paths.append(p)
    decoded = m._ingest_files(paths, DEV)
    tensors = [t.permute(1, 2, 0) for t in decoded]
    a = V.run(m, paths, labels, batch_size=5, img_size=320)
    b = V.run(m, tensors, labels, batch_size=5, img_size=320, channel_order="rgb")
    for k in KEYS:
        assert _same(a[k], b[k]), k


def test_run_arena_overflow_gives_the_same_result():
    m = _model("n")
    images, labels = _set(20, 10)
    ims = [torch.from_numpy(im).to(DEV) for im in images]
    roomy = V.run(m, ims, labels, batch_size=8, img_size=320)
    arena = _C._arenas.setdefault(DEV, _C._NmsArena())
    arena.cap_per_image, arena.ws = 64, None
    small = V.run(m, ims, labels, batch_size=8, img_size=320)
    assert arena.cap_per_image > 64
    for k in KEYS:
        assert _same(roomy[k], small[k]), k
