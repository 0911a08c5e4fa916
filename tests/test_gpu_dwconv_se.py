"""The MobileNetV3 ops in isolation (H100): YB_OP_DWCONV against fp32 F.conv2d(groups=C) and YB_OP_SE against fp32
squeeze-excitation, both on the op's own rounded input and weights, over channel counts, kernel sizes, strides, map
shapes, batch sizes, dtypes and activations, on strided views with sentinels in the channel gaps."""
import pytest
import torch
import torch.nn.functional as F

from stagewise import TOL, act_ref
from yolort_b200 import _C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CHANNELS = [8, 16, 40, 72, 88, 120, 144, 288, 576]
SENTINEL = 7.0
ACTS = [_C.YB_ACT_NONE, _C.YB_ACT_RELU, _C.YB_ACT_HARDSWISH]


def _strided(N, H, W, C, lead, tail, dtype, g):
    """[N,H,W,lead+C+tail] filled with SENTINEL, the window [lead, lead+C) random; returns (buffer, window)."""
    buf = torch.full((N, H, W, lead + C + tail), SENTINEL, dtype=dtype, device=DEV)
    buf[..., lead:lead + C] = torch.randn(N, H, W, C, generator=g, device=DEV).mul_(2.0).to(dtype)
    return buf, buf[..., lead:lead + C]


def _desc(kind, dtype, src_buf, lead_in, dst_buf, lead_out, N, H, W, Ho, Wo, C):
    d = _C.OpDesc()
    d.kind, d.dtype = kind, _C.dtype_code(dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride = N, H, W, C, src_buf.shape[-1]
    d.in_ = src_buf.data_ptr() + lead_in * 2
    d.Ho, d.Wo, d.Cout, d.out_cstride = Ho, Wo, C, dst_buf.shape[-1]
    d.out = dst_buf.data_ptr() + lead_out * 2
    return d


def _maps(C):
    maps = [(1, 1, 1), (2, 7, 9), (3, 8, 6), (32, 10, 12)]
    if C <= 144:
        maps.append((4, 40, 40))
    return maps


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("k", [1, 3, 5])
@pytest.mark.parametrize("C", CHANNELS)
def test_dwconv_matches_fp32_conv2d(C, k, s, dtype):
    g = torch.Generator(device=DEV).manual_seed(C * 100 + k * 10 + s)
    p = k // 2
    tol = TOL[dtype]
    for mi, (N, H, W) in enumerate(_maps(C)):
        act = ACTS[(mi + k + s) % 3]
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        src_buf, x = _strided(N, H, W, C, 8, 16, dtype, g)
        dst_buf = torch.full((N, Ho, Wo, C + 24), SENTINEL, dtype=dtype, device=DEV)
        w = (torch.randn(C, 1, k, k, generator=g, device=DEV) / k).to(dtype)
        b = torch.randn(C, generator=g, device=DEV) * 0.5
        wp = w.reshape(C, k * k).t().contiguous()
        d = _desc(_C.YB_OP_DWCONV, dtype, src_buf, 8, dst_buf, 16, N, H, W, Ho, Wo, C)
        d.ksize, d.stride, d.pad, d.act = k, s, p, act
        d.weight, d.bias = wp.data_ptr(), b.data_ptr()
        _C.Plan([d], DEV).run()
        torch.cuda.synchronize()
        ref = act_ref(F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, s, p, 1, C), act)
        got = dst_buf[..., 16:16 + C].float().permute(0, 3, 1, 2)
        err = (got - ref).abs()
        bad = int((err > tol * (1.0 + ref.abs())).sum())
        assert bad == 0, (C, k, s, (N, H, W), act, bad, float(err.max()))
        assert bool((dst_buf[..., :16] == SENTINEL).all()) and bool((dst_buf[..., 16 + C:] == SENTINEL).all())
        assert bool((src_buf[..., :8] == SENTINEL).all()) and bool((src_buf[..., 8 + C:] == SENTINEL).all())


def test_dwconv_unit_weights_stride2_is_the_max_pool_subsample():
    """max_pool2d(k=1, s=2) of the FPN's LastLevelMaxPool: ksize 1, stride 2, unit weights, zero bias -- exact."""
    N, H, W, C = 4, 10, 14, 256
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(N, H, W, C, generator=g, device=DEV).mul_(30.0).half()
    out = torch.empty(N, H // 2, W // 2, C, dtype=torch.float16, device=DEV)
    w = torch.ones(1, C, dtype=torch.float16, device=DEV)
    b = torch.zeros(C, device=DEV)
    d = _desc(_C.YB_OP_DWCONV, torch.float16, x, 0, out, 0, N, H, W, H // 2, W // 2, C)
    d.ksize, d.stride, d.pad = 1, 2, 0
    d.weight, d.bias = w.data_ptr(), b.data_ptr()
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 1, 2, 0).permute(0, 2, 3, 1).half()
    assert torch.equal(out, ref)


def _se_ref(x, w1, b1, w2, b2):
    """x [N,H,W,C] rounded input -> fp32 x * hardsigmoid(W2 relu(W1 mean + b1) + b2)."""
    xf = x.float()
    m = xf.mean((1, 2))
    h = F.relu(m @ w1.t() + b1)
    gate = F.hardsigmoid(h @ w2.t() + b2)
    return xf * gate[:, None, None, :], gate


def _se_weights(C, S, g):
    w1 = torch.randn(S, C, generator=g, device=DEV) * (2.0 / C) ** 0.5
    b1 = torch.randn(S, generator=g, device=DEV) * 0.5
    w2 = torch.randn(C, S, generator=g, device=DEV) * (6.0 / S) ** 0.5
    b2 = torch.randn(C, generator=g, device=DEV)
    wt = torch.cat([w1.t().reshape(-1), w2.t().reshape(-1)]).contiguous()
    bt = torch.cat([b1, b2]).contiguous()
    return w1, b1, w2, b2, wt, bt


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("C", CHANNELS)
def test_se_matches_fp32(C, dtype):
    S = max(8, (C // 4 + 7) // 8 * 8)
    g = torch.Generator(device=DEV).manual_seed(C + 3)
    tol = TOL[dtype]
    maps = [(1, 1, 1), (3, 3, 5), (32, 20, 20), (2, 80, 80)]
    if C <= 144:
        maps.append((1, 160, 160))
    w1, b1, w2, b2, wt, bt = _se_weights(C, S, g)
    for N, H, W in maps:
        buf, x = _strided(N, H, W, C, 8, 8, dtype, g)
        x0 = x.clone()
        d = _desc(_C.YB_OP_SE, dtype, buf, 8, buf, 8, N, H, W, H, W, C)
        d.ksize = S
        d.weight, d.bias = wt.data_ptr(), bt.data_ptr()
        plan = _C.Plan([d], DEV)
        plan.run()
        torch.cuda.synchronize()
        ref, gate = _se_ref(x0, w1, b1, w2, b2)
        err = (x.float() - ref).abs()
        bad = int((err > tol * (1.0 + ref.abs())).sum())
        assert bad == 0, (C, (N, H, W), bad, float(err.max()))
        assert bool((buf[..., :8] == SENTINEL).all()) and bool((buf[..., 8 + C:] == SENTINEL).all())
        # the same input gives the same bits (fixed-order reduction, no atomics)
        first = x.clone()
        x.copy_(x0)
        plan.run()
        torch.cuda.synchronize()
        assert torch.equal(x, first)
