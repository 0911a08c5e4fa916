"""Every case of tests/letterbox_cases.py on the H100, bit for bit against oracle.restate.letterbox.

The restatement is ATen's upsample_bilinear2d in numpy fp32 with the kernels' unfused operations in their order, the
same ratio float(h) / float(nh) and the same `uint8 / 255.0` values; the kernels differ from it only in ways that
change no value after the cast to the destination dtype (taps of weight zero are skipped, which can flip only the
sign of a zero; the copy paths compute byte * (1/255), which rounds to the fp16 / bf16 of byte / 255.0 for every byte,
tests/test_host_logic.py).  So every path is compared with torch.equal (+0 == -0), without a tolerance.
"""
import time

import pytest
import torch

from letterbox_cases import CASES, DTYPES, byte_offsets, geometry, letterbox_paths, make_images, pixel_path
from oracle import restate as R
from yolort_b200 import _C

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _first_mismatch(case, geoms, Hb, Wb, got, want):
    bad = (got != want) | torch.isnan(got)
    n, c, y, x = (int(v) for v in bad.nonzero()[0])
    return (f"{int(bad.sum())} of {bad.numel()} values differ; first at image {n} channel {c} pixel (y={y}, x={x}): "
            f"got {got[n, c, y, x].item()!r} want {want[n, c, y, x].item()!r} "
            f"[{pixel_path(case, geoms, Hb, Wb, n, y, x)}]")


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_letterbox_case_is_bit_exact(case):
    t0 = time.perf_counter()
    geoms, (Hb, Wb) = geometry(case)
    paths = letterbox_paths(case, geoms, Hb, Wb)
    ims, ref_ims = make_images(case, DEV)
    # the host mirror's alignment model (letterbox_cases.byte_offsets) is the real one
    assert [im.data_ptr() % 16 for im in ims] == [o % 16 for o in byte_offsets(case)]
    n = len(ims)
    dt = DTYPES[case.dtype]
    shape = (n + 1, 3, Hb, Wb) if case.layout == "nchw" else (n + 1, Hb // 2, Wb // 2, 16)
    out = torch.full(shape, float("nan"), dtype=dt, device=DEV)   # one slot past the batch must stay untouched
    fill = case.fill_color / 255
    if any(p.startswith("reject") for p in paths):
        with pytest.raises(_C.NativeLibraryError):
            _C.letterbox(ims, geoms, Hb, Wb, fill, out, case.layout_code)
        torch.cuda.synchronize()
        assert torch.isnan(out).all()
        return
    _C.letterbox(ims, geoms, Hb, Wb, fill, out, case.layout_code)
    got = out.cpu()
    assert torch.isnan(got[n]).all(), "the launch wrote past the batch"
    got = got[:n]
    if case.layout == "s2d":
        # s2d[n, Y, X, (dy*2+dx)*4 + c] == nchw[n, c, 2Y+dy, 2X+dx]; channel 3 of every quad is zero
        v = got.view(n, Hb // 2, Wb // 2, 2, 2, 4)
        pad = v[..., 3]
        if not torch.all(pad == 0):
            i, Y, X, dy, dx = (int(a) for a in (pad != 0).nonzero()[0])
            pytest.fail(f"channel 3 of image {i} pixel (y={2 * Y + dy}, x={2 * X + dx}) is {pad[i, Y, X, dy, dx].item()!r} "
                        f"[{pixel_path(case, geoms, Hb, Wb, i, 2 * Y + dy, 2 * X + dx)}]")
        got = v[..., :3].permute(0, 5, 1, 3, 2, 4).reshape(n, 3, Hb, Wb)
    ref, _, geo = R.letterbox(ref_ims, case.min_size, case.max_size, case.size_divisible, case.fixed_shape,
                              case.fill_color)
    assert geo == [(g.new_h, g.new_w, g.top, g.left) for g in geoms]
    want = ref.to(dt)
    assert torch.equal(got, want), _first_mismatch(case, geoms, Hb, Wb, got, want)
    print(f"{case.name}: {n} images, canvas {Hb}x{Wb}, {time.perf_counter() - t0:.2f} s; {sorted(paths)}")
