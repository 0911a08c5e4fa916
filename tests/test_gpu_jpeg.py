"""Device JPEG decode (csrc/jpeg_decode.cu): bit-identical to torchvision's CPU decoder, bounded writes, per-image
status, and predict(paths) / predict_stream(paths) unchanged by it."""
import os

import pytest
import torch

import jpeg_corpus as J
import parity_util as util
from yolort_b200 import _C
from yolort_b200.io import decode_jpeg
from yolort_b200.models import yolov5n

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _blob(data: bytes) -> torch.Tensor:
    return torch.frombuffer(bytearray(data), dtype=torch.uint8)


def _files(large=True):
    files = [(n, d) for n, d, _ in J.corpus(J.SMALL_SIZES + (J.LARGE_SIZES if large else ()))]
    files += [(n, d) for n, d, _ in J.cv2_corpus()]
    return files + J.assets()


def _assert_same(name, got, want):
    assert got.shape == want.shape, name
    if not torch.equal(got.cpu(), want):
        diff = (got.cpu().int() - want.int()).abs()
        pytest.fail(f"{name}: {int((diff > 0).sum())} bytes differ, max {int(diff.max())}")


def test_decode_one_at_a_time_is_bit_identical():
    for name, data in _files():
        got = decode_jpeg(_blob(data), DEV)
        assert got.is_cuda and got.stride() == (1, 3 * got.shape[2], 3), name
        _assert_same(name, got, J.cpu_decode(data))


def test_decode_mixed_batch_is_bit_identical():
    files = _files(large=False) + [(n, d) for n, d, _ in J.corpus(((480, 640),))[::5]]
    got = decode_jpeg([_blob(d) for _, d in files], DEV)
    for (name, data), g in zip(files, got):
        _assert_same(name, g, J.cpu_decode(data))
    again = decode_jpeg([_blob(d) for _, d in reversed(files)], DEV)     # replays are bit-identical
    for g, a in zip(got, reversed(again)):
        assert torch.equal(g, a)


def test_writes_stay_inside_each_image():
    files = [(n, d) for n, d, _ in J.corpus(((7, 9), (61, 117)))][::3] + J.assets()
    infos = [_C.jpeg_parse(d) for _, d in files]
    pad = 4096
    sizes = [int(i.height) * int(i.width) * 3 for i in infos]
    buf = torch.full((sum(sizes) + pad * (len(files) + 1),), 0xA5, dtype=torch.uint8, device=DEV)
    dst, off = [], pad
    for i, sz in zip(infos, sizes):
        dst.append(buf[off:off + sz].view(int(i.height), int(i.width), 3))
        off += sz + pad
    images, status = _C.jpeg_decode([_blob(d) for _, d in files], infos, torch.device(DEV), dst=dst)
    assert status.cpu().tolist() == [0] * len(files)
    mask = torch.ones_like(buf, dtype=torch.bool)
    off = pad
    for sz in sizes:
        mask[off:off + sz] = False
        off += sz + pad
    assert bool((buf[mask] == 0xA5).all())
    for (name, data), g in zip(files, images):
        _assert_same(name, g, J.cpu_decode(data))


def _truncated(data: bytes) -> bytes:
    b, e = J.scan_segment(data)
    return data[:b + (e - b) // 2] + b"\xff\xd9"


def _swapped_restart(data: bytes) -> bytes:
    b, e = J.scan_segment(data)
    seg = bytearray(data[b:e])
    k = seg.index(b"\xff\xd1")
    seg[k + 1] = 0xD2
    return data[:b] + bytes(seg) + data[e:]


def test_corrupt_entropy_data_is_flagged_and_isolated():
    clean = [d for _, d in J.assets()] + [d for _, d, _ in J.corpus(((61, 117),))[:6]]
    bus = clean[0]
    bad = {1: _truncated(clean[1]), 3: _swapped_restart(bus), 5: _truncated(bus)}
    batch = list(clean)
    for k, v in bad.items():
        batch.insert(k, v)
    infos = [_C.jpeg_parse(d) for d in batch]
    assert all(i.supported for i in infos)
    images, status = _C.jpeg_decode([_blob(d) for d in batch], infos, torch.device(DEV))
    st = status.cpu().tolist()
    for k, d in enumerate(batch):
        if k in bad:
            assert st[k] != 0, k
        else:
            assert st[k] == 0, (k, st[k])
            _assert_same(str(k), images[k], J.cpu_decode(d))
    assert st[1] & _C.YB_JPEG_ST_TRUNCATED and st[3] & _C.YB_JPEG_ST_RESTART
    with pytest.raises(RuntimeError, match="image 1"):
        decode_jpeg([_blob(clean[0]), _blob(bad[1])], DEV)


def test_unsupported_files_raise_value_error():
    with pytest.raises(ValueError, match="progressive"):
        decode_jpeg(_blob(J.progressive()), DEV)
    with pytest.raises(ValueError, match="4 components"):
        decode_jpeg([_blob(J.assets()[0][1]), _blob(J.cmyk())], DEV)


# -- predict(paths) -----------------------------------------------------------------------------------------------
def _model():
    sd = util.synth_state_dict(util.layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0)
    m = yolov5n(size=(256, 256), score_thresh=0.15).eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def _write_mixed(tmp_path):
    from torchvision.io import write_png

    paths = []
    for name, data in J.assets():
        paths.append(str(tmp_path / name))
        open(paths[-1], "wb").write(data)
    for k, (name, data, _) in enumerate(J.corpus(((61, 117), (480, 640)))[::7]):
        paths.append(str(tmp_path / f"c{k}.jpg"))
        open(paths[-1], "wb").write(data)
    paths.append(str(tmp_path / "prog.jpg"))
    open(paths[-1], "wb").write(J.progressive())
    png = torch.from_numpy(J.photo(90, 128, 5)).permute(2, 0, 1).contiguous()
    paths.append(str(tmp_path / "p.png"))
    write_png(png, paths[-1])
    return paths


def _same_dets(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a["labels"].cpu(), b["labels"].cpu()) and torch.equal(a["scores"].cpu(), b["scores"].cpu())
        assert torch.equal(a["boxes"].cpu(), b["boxes"].cpu())


def _with_env(value, fn):
    old = os.environ.get("YB_JPEG_DECODE")
    os.environ["YB_JPEG_DECODE"] = value
    try:
        return fn()
    finally:
        if old is None:
            del os.environ["YB_JPEG_DECODE"]
        else:
            os.environ["YB_JPEG_DECODE"] = old


def test_predict_paths_is_bit_identical_to_cpu_decode(tmp_path):
    from torchvision.io import ImageReadMode, read_image

    paths = _write_mixed(tmp_path)
    m = _model()
    decoded = [read_image(p, mode=ImageReadMode.RGB) for p in paths]
    want = m.predict([d.contiguous() for d in decoded])
    assert sum(len(w["scores"]) for w in want) > 0
    _same_dets(m.predict(paths), want)
    _same_dets(_with_env("cpu", lambda: m.predict(paths)), want)
    half = len(paths) // 2          # each batch letterboxes to its own canvas: compare batch by batch
    batches = [paths[:half], paths[half:], paths]
    streamed = [d for batch in m.predict_stream(batches) for d in batch]
    planar = [d.contiguous() for d in decoded]
    _same_dets(streamed, m.predict(planar[:half]) + m.predict(planar[half:]) + want)
    cpu_streamed = _with_env("cpu", lambda: [d for batch in m.predict_stream(batches) for d in batch])
    _same_dets(streamed, cpu_streamed)


def test_corrupt_jpeg_in_predict_behaves_as_cpu_path(tmp_path):
    paths = _write_mixed(tmp_path)[:4]
    with open(paths[1], "rb") as f:
        data = f.read()
    with open(paths[1], "wb") as f:
        f.write(_truncated(data))
    m = _model()

    def run():
        try:
            return ("ok", m.predict(paths))
        except Exception as e:        # whatever the CPU decoder does with the file, both paths must do it
            return ("raised", type(e), str(e))

    gpu, cpu = run(), _with_env("cpu", run)
    assert gpu[0] == cpu[0]
    if gpu[0] == "ok":
        _same_dets(gpu[1], cpu[1])
    else:
        assert gpu[1:] == cpu[1:]
