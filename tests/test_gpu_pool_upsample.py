"""SPP max-pool cascade and nearest 2x upsample kernels vs PyTorch reference ops (H100)."""
import pytest
import torch
import torch.nn.functional as F

from yolort_b200 import _C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _desc(kind, x_full, in_off, C, out_full, out_off, Cout, N, H, W, Ho, Wo, dtype):
    d = _C.OpDesc()
    d.kind, d.dtype = kind, _C.dtype_code(dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride = N, H, W, C, x_full.shape[-1]
    d.in_ = x_full.data_ptr() + in_off * 2
    d.Ho, d.Wo, d.Cout, d.out_cstride = Ho, Wo, Cout, out_full.shape[-1]
    d.out = out_full.data_ptr() + out_off * 2
    return d


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("hw", [(20, 20), (13, 20), (40, 40), (7, 5)])
def test_spp_pool_matches_max_pool2d(hw, dtype):
    N, C = 3, 64
    H, W = hw
    g = torch.Generator().manual_seed(1)
    cat = torch.randn(N, H, W, 4 * C, generator=g).to(dtype).to(DEV)   # the SPP concat buffer
    ref_in = cat[..., :C].float().permute(0, 3, 1, 2)
    d = _desc(_C.YB_OP_SPP_POOL, cat, 0, C, cat, C, 3 * C, N, H, W, H, W, dtype)
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    for i, k in enumerate((5, 9, 13)):
        ref = F.max_pool2d(ref_in, k, 1, k // 2)     # yolort/v5/models/common.py:183
        got = cat[..., (i + 1) * C:(i + 2) * C].float().permute(0, 3, 1, 2)
        assert torch.equal(got, ref), (k, hw)
    assert torch.equal(cat[..., :C].float().permute(0, 3, 1, 2), ref_in)   # input window untouched


def test_upsample2x_into_channel_window():
    N, H, W, C = 2, 10, 6, 32
    g = torch.Generator().manual_seed(2)
    src = torch.randn(N, H, W, 2 * C, generator=g).half().to(DEV)
    dst = torch.full((N, 2 * H, 2 * W, 3 * C), 5.0, dtype=torch.float16, device=DEV)
    d = _desc(_C.YB_OP_UPSAMPLE2X, src, C, C, dst, C, C, N, H, W, 2 * H, 2 * W, torch.float16)
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    ref = F.interpolate(src[..., C:].float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    assert torch.equal(dst[..., C:2 * C].float().permute(0, 3, 1, 2), ref)
    assert torch.all(dst[..., :C] == 5.0) and torch.all(dst[..., 2 * C:] == 5.0)
