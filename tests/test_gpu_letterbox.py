"""Letterbox kernel vs the reference fixtures / oracle (H100)."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200 import _C
from yolort_b200.models.transform import YOLOTransform

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_pixels_vs_reference_fixture_uint8():
    z = util.load_npz("letterbox_pixels.npz")
    ims = [torch.from_numpy(z[f"img{i}"]).to(DEV) for i in range(4)]
    tr = YOLOTransform(96, 96)
    nt, _ = tr(ims)
    got = nt.tensors.cpu().numpy()
    assert got.shape == z["batch"].shape and got.dtype == np.float32
    assert [tuple(s) for s in nt.image_sizes] == [tuple(s) for s in z["sizes"]]
    err = np.abs(got - z["batch"]).max()
    print("letterbox max abs err vs reference:", err)
    assert err <= 5e-5          # tolerance of SURVEY.md appendix A.3 (fp32 source-coordinate rounding)
    assert np.array_equal(got[2], z["batch"][2])   # identity resize: exact copy


def test_float_inputs_and_s2d_layout_agree_with_nchw():
    g = torch.Generator().manual_seed(5)
    ims = [torch.rand(3, 70, 101, generator=g), torch.rand(3, 128, 128, generator=g), torch.rand(3, 55, 40, generator=g)]
    tr = YOLOTransform(128, 128)
    ref, sizes, _ = R.letterbox(ims, 128.0, 128.0)
    dims = [im.to(DEV) for im in ims]
    nt, _ = tr(dims)
    assert np.abs(nt.tensors.cpu().numpy() - ref.numpy()).max() <= 5e-5
    geoms, (Hb, Wb) = tr.geometry(dims)
    for dt in (torch.float16, torch.bfloat16):
        s2d = torch.empty((3, Hb // 2, Wb // 2, 16), dtype=dt, device=DEV)
        tr.letterbox_into(dims, geoms, Hb, Wb, s2d, _C.YB_LAYOUT_S2D16)
        nchw = torch.empty((3, 3, Hb, Wb), dtype=dt, device=DEV)
        tr.letterbox_into(dims, geoms, Hb, Wb, nchw, _C.YB_LAYOUT_NCHW)
        # s2d[n, Y, X, (dy*2+dx)*4 + c] == nchw[n, c, 2Y+dy, 2X+dx]; channel 3 of every quad is zero
        v = s2d.view(3, Hb // 2, Wb // 2, 2, 2, 4)
        assert torch.all(v[..., 3] == 0)
        back = v[..., :3].permute(0, 5, 1, 3, 2, 4).reshape(3, 3, Hb, Wb)
        assert torch.equal(back, nchw)
        assert (nchw.float().cpu() - ref).abs().max() <= (2e-3 if dt == torch.float16 else 8e-3)


@pytest.mark.parametrize("hw", [(640, 640), (128, 192), (64, 72)])
def test_identity_full_canvas_uint8_fast_kernel(hw):
    """uint8 images that already have the canvas size (identity resize, no padding) take the dedicated copy kernel:
    s2d[n, Y, X, (dy*2+dx)*4 + c] == half(byte / 255.0) bit for bit, the fourth channel of every quad zero; and a mixed
    batch (one image smaller -> generic tile kernel) writes the same bits for the identity image."""
    h, w = hw
    g = torch.Generator().manual_seed(h + w)
    ims = [torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g).to(DEV) for _ in range(3)]
    tr = YOLOTransform(min(h, w), max(h, w), size_divisible=8)
    geoms, (Hb, Wb) = tr.geometry(ims)
    if (Hb, Wb) != (h, w):
        pytest.skip("transform rounds this canvas up")
    for dt in (torch.float16, torch.bfloat16):
        s2d = torch.full((3, Hb // 2, Wb // 2, 16), 9.0, dtype=dt, device=DEV)
        tr.letterbox_into(ims, geoms, Hb, Wb, s2d, _C.YB_LAYOUT_S2D16)
        v = s2d.view(3, Hb // 2, Wb // 2, 2, 2, 4)
        assert torch.all(v[..., 3] == 0)
        back = v[..., :3].permute(0, 5, 1, 3, 2, 4).reshape(3, 3, Hb, Wb)
        want = torch.stack([(im.float() / 255.0).to(dt) for im in ims])
        assert torch.equal(back, want)
        # same image next to a smaller one: the batch goes through the generic tile kernel
        small = torch.randint(0, 256, (3, h - 8, w - 16), dtype=torch.uint8, generator=g).to(DEV)
        mixed = [ims[0], small]
        geoms2, (Hb2, Wb2) = tr.geometry(mixed)
        if (Hb2, Wb2) == (Hb, Wb):
            s2 = torch.full((2, Hb // 2, Wb // 2, 16), 9.0, dtype=dt, device=DEV)
            tr.letterbox_into(mixed, geoms2, Hb, Wb, s2, _C.YB_LAYOUT_S2D16)
            assert torch.equal(s2[0], s2d[0])


def test_mixed_batch_geometry_639_trap():
    # sizes whose long side resizes to 639 (SURVEY.md appendix A.2) in one batch with a 640 one
    ims = [torch.randint(0, 256, (3, 800, 600), dtype=torch.uint8), torch.randint(0, 256, (3, 480, 640), dtype=torch.uint8)]
    ref, sizes, geo = R.letterbox(ims)
    nt, _ = YOLOTransform(640, 640)([im.to(DEV) for im in ims])
    assert nt.image_sizes == [tuple(s) for s in sizes] and nt.image_sizes[0] == (639, 479)
    assert np.abs(nt.tensors.cpu().numpy() - ref.numpy()).max() <= 5e-5


def test_rejects_bad_inputs():
    tr = YOLOTransform(64, 64)
    with pytest.raises(ValueError):
        tr([torch.rand(1, 3, 8, 8, device=DEV)])
    with pytest.raises(_C.NativeLibraryError):
        tr([torch.rand(3, 8, 8)])   # CPU tensor: no fallback


def test_interleaved_hwc_sources_equal_planar():
    """Decoded image files are HWC in memory (a [3,H,W] view with strides (1, 3W, 3)); the kernel reads them in
    place (yb_letterbox_strided) and must produce the bits of the planar path."""
    g = torch.Generator().manual_seed(11)
    for make in (lambda h, w: torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8),
                 lambda h, w: torch.rand(h, w, 3, generator=g)):
        hwc = [make(70, 101).to(DEV), make(128, 128).to(DEV), make(55, 40).to(DEV), make(300, 211).to(DEV)]
        views = [t.permute(2, 0, 1) for t in hwc]
        assert all(_C._is_hwc_view(v) for v in views)
        planar = [v.contiguous() for v in views]
        tr = YOLOTransform(128, 128)
        geoms, (Hb, Wb) = tr.geometry(views)
        for layout, shape in ((_C.YB_LAYOUT_NCHW, (4, 3, Hb, Wb)), (_C.YB_LAYOUT_S2D16, (4, Hb // 2, Wb // 2, 16))):
            a = torch.empty(shape, dtype=torch.float16, device=DEV)
            b = torch.empty(shape, dtype=torch.float16, device=DEV)
            tr.letterbox_into(views, geoms, Hb, Wb, a, layout)
            tr.letterbox_into(planar, geoms, Hb, Wb, b, layout)
            assert torch.equal(a, b)
        # a mixed list (one planar image) falls back to the planar path for the whole batch
        mixed = [views[0], planar[1], views[2], views[3]]
        c = torch.empty((4, 3, Hb, Wb), dtype=torch.float16, device=DEV)
        tr.letterbox_into(mixed, geoms, Hb, Wb, c, _C.YB_LAYOUT_NCHW)
        tr.letterbox_into(planar, geoms, Hb, Wb, b := torch.empty_like(c), _C.YB_LAYOUT_NCHW)
        assert torch.equal(c, b)
