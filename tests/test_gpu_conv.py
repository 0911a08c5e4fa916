"""wgmma implicit-GEMM convolution vs a plain fp32 PyTorch conv on the same fp16/bf16-rounded operands (H100)."""
import pytest
import torch
import torch.nn.functional as F

from yolort_b200 import _C
from yolort_b200.engine import pack_bias, pack_weight

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def run_conv(N, H, W, Cin, Cout, k, s, p, dtype=torch.float16, act=True, residual=False, in_pad=0, out_pad=0, seed=0,
             bias_scale=0.5, force_im2col=False, force_planes=False):
    torch.backends.cudnn.allow_tf32 = False      # the fp32 reference must not run on TF32 tensor cores
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    in_cs, out_cs = Cin + in_pad, Cout + out_pad
    x_full = (torch.randn(N, H, W, in_cs, generator=g)).to(dtype).to(DEV)
    in_off = in_pad // 2 // 8 * 8
    out_off = out_pad // 2 // 8 * 8
    w = (torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).to(dtype)
    b = torch.randn(Cout, generator=g) * bias_scale
    wp, ci_pad, co_pad = pack_weight(w.double(), dtype, DEV)
    bp = pack_bias(b.double(), co_pad, DEV)
    out_full = torch.full((N, Ho, Wo, out_cs), 7.0, dtype=dtype, device=DEV)
    res = (torch.randn(N, Ho, Wo, Cout, generator=g)).to(dtype).to(DEV) if residual else None
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_CONV, _C.dtype_code(dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride = N, H, W, Cin, in_cs
    d.in_ = x_full.data_ptr() + in_off * 2
    d.Ho, d.Wo, d.Cout, d.out_cstride = Ho, Wo, Cout, out_cs
    d.out = out_full.data_ptr() + out_off * 2
    act_code = {True: _C.YB_ACT_SILU, False: _C.YB_ACT_NONE, "hardswish": _C.YB_ACT_HARDSWISH,
                "leaky": _C.YB_ACT_LEAKY01}[act]
    d.ksize, d.stride, d.pad, d.act = k, s, p, act_code
    d.weight, d.Cin_pad, d.Cout_pad, d.bias = wp.data_ptr(), ci_pad, co_pad, bp.data_ptr()
    if residual:
        d.residual, d.res_cstride = res.data_ptr(), Cout
    d.reserved = (1 if force_im2col else 0) | (4 if force_planes else 0)
    plan = _C.Plan([d], DEV)
    plan.run()
    torch.cuda.synchronize()
    x = x_full[..., in_off:in_off + Cin].float().permute(0, 3, 1, 2)
    ref = F.conv2d(x, w.float().to(DEV), b.to(DEV), s, p)
    if act == "hardswish":
        ref = F.hardswish(ref)
    elif act == "leaky":
        ref = F.leaky_relu(ref, 0.1)
    elif act:
        ref = F.silu(ref)
    if residual:
        ref = ref + res.float().permute(0, 3, 1, 2)
    got = out_full[..., out_off:out_off + Cout].float().permute(0, 3, 1, 2)
    # channels outside the destination window must be untouched
    if out_pad:
        mask = torch.ones(out_cs, dtype=torch.bool)
        mask[out_off:out_off + Cout] = False
        assert torch.all(out_full[..., mask.to(DEV)] == 7.0)
    err = (got - ref).abs()
    tol = (2.0 ** -9 if dtype == torch.float16 else 2.0 ** -6)   # SURVEY.md section 8c stage-wise bound
    bound = tol * (1.0 + ref.abs())
    bad = (err > bound).sum().item()
    print(f"conv N{N} {H}x{W} {Cin}->{Cout} k{k}s{s} {dtype}: max_abs_err={err.max().item():.3e} "
          f"ref_absmax={ref.abs().max().item():.2f} violations={bad}/{err.numel()}")
    if bad:
        idx = (err > bound).nonzero()[:8]
        print("first violations (n,c,y,x):", idx.tolist())
        print("got", got[tuple(idx[0])].item(), "ref", ref[tuple(idx[0])].item())
    assert bad == 0


@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 64), (32, 32), (16, 32), (256, 256), (512, 256), (48, 96), (80, 160)])
def test_conv1x1(cin, cout):
    run_conv(2, 20, 20, cin, cout, 1, 1, 0)


def test_conv1x1_ragged_m_and_channel_windows():
    run_conv(3, 13, 11, 64, 64, 1, 1, 0, in_pad=64, out_pad=32)       # M = 429, not a tile multiple; sliced views


@pytest.mark.parametrize("cin,cout,s", [(64, 64, 1), (32, 64, 2), (16, 32, 1), (128, 128, 2), (256, 256, 1), (48, 48, 1)])
def test_conv3x3(cin, cout, s):
    run_conv(2, 24, 40, cin, cout, 3, s, 1)


def test_conv3x3_crosses_image_boundaries():
    run_conv(5, 6, 10, 64, 64, 3, 1, 1)      # 60 pixels/image: every 128-pixel tile spans 2-3 images
    run_conv(4, 10, 6, 32, 64, 3, 2, 1)      # stride 2, Wo=3


def test_bottleneck_residual_and_inplace_window():
    run_conv(2, 20, 20, 64, 64, 3, 1, 1, residual=True, out_pad=64)


def test_head_conv_bias_no_activation():
    run_conv(2, 20, 20, 128, 256, 1, 1, 0, act=False)


def test_wide_output_splits_into_n_tiles():
    run_conv(1, 16, 16, 64, 320, 1, 1, 0)    # block_n = 160 x 2 tiles
    run_conv(1, 16, 16, 128, 512, 3, 1, 1)   # block_n = 256 x 2 tiles


def test_bf16():
    run_conv(2, 20, 20, 64, 128, 1, 1, 0, dtype=torch.bfloat16)
    run_conv(2, 20, 20, 64, 64, 3, 2, 1, dtype=torch.bfloat16)


def test_large_m_many_tiles():
    run_conv(8, 80, 80, 64, 64, 3, 1, 1)     # 51 200 pixels -> 400 CTAs


def test_silu_strongly_negative_preactivations():
    """Pre-activations below -8, where SiLU is a few 1e-3 and an approximation through tanh in fp16 would cancel: the
    epilogue evaluates v / (1 + e^-v) in fp32 and must stay within the stage-wise bound there.  Large biases put ~10 %
    of the outputs in that range."""
    run_conv(2, 20, 20, 64, 64, 1, 1, 0, bias_scale=6.0, seed=21)
    run_conv(2, 24, 24, 64, 64, 3, 1, 1, bias_scale=6.0, seed=22, residual=True)
    run_conv(2, 20, 20, 64, 128, 1, 1, 0, bias_scale=6.0, seed=23, dtype=torch.bfloat16)
    run_conv(2, 24, 40, 32, 64, 3, 2, 1, bias_scale=6.0, seed=24)


def test_rejects_unsupported():
    d = _C.OpDesc()
    d.kind = 99
    with pytest.raises(_C.NativeLibraryError):
        _C.Plan([d], DEV)


# ---- halo-patch 3x3 kernel (conv3x3_patch_sm90.cu)  -------------------------------------------------------
@pytest.mark.parametrize("cin,cout", [(64, 64), (16, 32), (32, 32), (128, 128), (256, 256), (48, 48), (80, 80), (96, 192)])
def test_patch_conv_channel_widths(cin, cout):
    """Halo-patch kernel over the channel widths of the zoo, incl. widths that do not fill a 64-channel chunk
    (48 / 80 / 96: the last chunk runs 3 / 1 / 2 K-steps over TMA-zero-filled rows)."""
    run_conv(2, 32, 40, cin, cout, 3, 1, 1, seed=3)


def test_patch_conv_ragged_edges_residual_and_windows():
    run_conv(3, 40, 44, 64, 64, 3, 1, 1, residual=True, in_pad=32, out_pad=64)   # W=44: last column tile half empty
    run_conv(1, 48, 24, 128, 128, 3, 1, 1, dtype=torch.bfloat16)


@pytest.mark.parametrize("shape", [
    (1, 40, 40, 128, 128, False),    # weights streamed: 15 tiles -> 7 pair tasks + one single (odd count)
    (3, 40, 40, 128, 256, True),     # Cout 256 splits into two 128-column N tiles under pairing; residual
    (2, 48, 24, 192, 192, False),    # three chunks, block_n 96 x 2
    (2, 20, 20, 256, 256, True),     # wrap tiling (5 x 24 tiles on a 20-wide map) + pairs + residual
    (3, 20, 20, 128, 128, False),    # wrap tiling, resident or streamed weights
    (2, 17, 19, 64, 64, True),       # wrap tiling, ragged height/width, resident weights
    (1, 13, 22, 96, 160, False),     # wrap tiling at its widest map (22), partial last chunk
    (5, 10, 20, 256, 128, False),    # wrap tiling, H = 2 tiles exactly, odd tile count
])
def test_patch_conv_pairs_and_wrap_tiles(shape):
    """Two M tiles per weight pass (weights that do not fit in shared memory) and the 5 x 24 wrap tiling of narrow
    maps, against the fp32 convolution."""
    n, h, w, ci, co, res = shape
    run_conv(n, h, w, ci, co, 3, 1, 1, residual=res, seed=5)
    run_conv(n, h, w, ci, co, 3, 1, 1, residual=res, seed=6, dtype=torch.bfloat16, out_pad=64 if co <= 128 else 0)


@pytest.mark.parametrize("shape", [
    (2, 64, 64, 32, 64, 0, 0),       # body.1-like: 32 channels = half-filled 128-byte rows, resident weights
    (2, 64, 64, 64, 128, 0, 64),     # body.3-like: weights streamed, output into a channel window
    (1, 96, 80, 128, 256, 128, 0),   # body.5-like: input is the right half of a concat buffer (cstride 256), N split 2 x 128
    (3, 32, 48, 48, 96, 0, 0),       # partial last chunk (48 channels: 3 K-steps)
    (1, 160, 160, 16, 32, 0, 0),     # yolov5n body.1: 16 channels, 32-byte K rows
    (2, 80, 88, 256, 256, 0, 0),     # four chunks; Wo = 44: last column tile half empty; Ho = 40
])
def test_patch_conv_stride2_parity_planes(shape):
    """3x3 / stride 2 on the halo-patch kernel (two column-parity planes per chunk) vs the fp32 convolution, and vs
    the generic im2col kernel on the same operands."""
    n, h, w, ci, co, in_pad, out_pad = shape
    run_conv(n, h, w, ci, co, 3, 2, 1, in_pad=in_pad, out_pad=out_pad, seed=7, force_planes=True)
    run_conv(n, h, w, ci, co, 3, 2, 1, in_pad=in_pad, out_pad=out_pad, seed=7, force_im2col=True)
    run_conv(n, h, w, ci, co, 3, 2, 1, in_pad=in_pad, out_pad=out_pad, seed=8, dtype=torch.bfloat16, force_planes=True)
    run_conv(n, h, w, ci, co, 3, 2, 1, in_pad=in_pad, out_pad=out_pad, seed=9)      # the plan's own choice


def test_patch_conv_matches_im2col_kernel():
    """Same layer through both kernels (reserved bit 0 forces the generic im2col path)."""
    run_conv(2, 32, 32, 64, 64, 3, 1, 1, seed=11, force_im2col=True)
    run_conv(2, 32, 32, 64, 64, 3, 1, 1, seed=11)


@pytest.mark.parametrize("shape", [
    (32, 160, 160, 64, 64, 1, 1, 0, False),     # body.2.cv3 of yolov5s batch 32: M = 819 200 rows, 6 400 tiles
    (32, 320, 320, 32, 64, 3, 2, 1, False),     # body.1: stride 2 on the 320^2 map
    (32, 160, 160, 32, 32, 3, 1, 1, True),      # body.2.m.0.cv2: 64-byte rows + residual
    (32, 20, 20, 256, 256, 3, 1, 1, True),      # body.8.m.0.cv2: deep 3x3, weight ring
    (32, 40, 40, 256, 512, 3, 2, 1, False),     # body.7
    (32, 20, 20, 1024, 512, 1, 1, 0, False),    # SPP cv2: K = 1024
])
def test_conv_at_bench_layer_shapes(shape):
    """The layer shapes of the yolov5s batch-32 640x640 benchmark (dozens of tiles and mbarrier phase wraps per
    persistent CTA), against the fp32 convolution of the same operands."""
    n, h, w, ci, co, k, s, p, res = shape
    run_conv(n, h, w, ci, co, k, s, p, residual=res)


@pytest.mark.parametrize("act", ["hardswish", "leaky"])
def test_r31_activations(act):
    """Hardswish (r3.1 Conv) and LeakyReLU(0.1) (BottleneckCSP) epilogues, on both kernels (1x1 generic, 3x3 patch)."""
    run_conv(2, 24, 40, 64, 64, 1, 1, 0, act=act, bias_scale=2.0)
    run_conv(2, 32, 32, 32, 64, 3, 1, 1, act=act, residual=(act == "hardswish"), bias_scale=2.0)
    run_conv(1, 20, 28, 48, 96, 3, 2, 1, act=act, dtype=torch.bfloat16)


# ---- chained pointwise tails (yb_conv_chain: conv -> 1x1 conv inside one launch) ---------------------------
def run_chain(N, H, W, Cin, C1, k, c_own, C2, extra=False, residual=False, dtype=torch.float16, seed=0, store_first=True,
              act2=True):
    """First convolution (k x k, stride 1, C1 outputs, optional shortcut) with a chained 1x1 tail over
    [first_out[:c_own] | extra(c_own channels)] -> C2 channels.  Checks: the library accepts the fusion; the first
    output (when stored) against fp32 on the rounded inputs; the tail against fp32 applied to the STORED first output
    (= exactly the fp16 tile the tail consumed on chip); and, with store_first=False, bit equality of the tail with
    the store_first=True run (the flag only gates the TMA store)."""
    import ctypes

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(seed)
    p = k // 2
    x = torch.randn(N, H, W, Cin, generator=g).to(dtype).to(DEV)
    w1 = (torch.randn(C1, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).to(dtype)
    b1 = torch.randn(C1, generator=g) * 0.5
    K2 = c_own * (2 if extra else 1)
    w2 = (torch.randn(C2, K2, 1, 1, generator=g) * (2.0 / K2) ** 0.5).to(dtype)
    b2 = torch.randn(C2, generator=g) * 0.5
    wp1, ci_pad, co_pad = pack_weight(w1.double(), dtype, DEV)
    bp1 = pack_bias(b1.double(), co_pad, DEV)
    wp2, k2_pad, co2_pad = pack_weight(w2.double(), dtype, DEV)
    bp2 = pack_bias(b2.double(), co2_pad, DEV)
    # the first output lives in the left window of a concat buffer whose right window is the extra operand (C3 layout)
    cat_cs = C1 + (c_own if extra else 0)
    cat = torch.randn(N, H, W, cat_cs, generator=g).to(dtype).to(DEV)
    cat0 = cat.clone()
    res = torch.randn(N, H, W, C1, generator=g).to(dtype).to(DEV) if residual else None
    out2 = torch.full((N, H, W, C2 + 16), 7.0, dtype=dtype, device=DEV)      # tail output into a channel window too

    def launch(store):
        cat.copy_(cat0)
        out2.fill_(7.0)
        d = _C.OpDesc()
        d.kind, d.dtype = _C.YB_OP_CONV, _C.dtype_code(dtype)
        d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, H, W, Cin, Cin, x.data_ptr()
        d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = H, W, C1, cat_cs, cat.data_ptr()
        d.ksize, d.stride, d.pad, d.act = k, 1, p, _C.YB_ACT_SILU
        d.weight, d.Cin_pad, d.Cout_pad, d.bias = wp1.data_ptr(), ci_pad, co_pad, bp1.data_ptr()
        if residual:
            d.residual, d.res_cstride = res.data_ptr(), C1
        c = _C.ConvChain()
        c.weight, c.bias, c.Cout, c.Cout_pad, c.K_pad = wp2.data_ptr(), bp2.data_ptr(), C2, co2_pad, k2_pad
        c.act = _C.YB_ACT_SILU if act2 else _C.YB_ACT_NONE
        c.out, c.out_cstride, c.own_C = out2.data_ptr(), C2 + 16, c_own
        if extra:
            c.extra, c.extra_C, c.extra_cstride = cat.data_ptr() + C1 * 2, c_own, cat_cs
        c.store_first = 1 if store else 0
        d.chain = ctypes.addressof(c)
        assert _C.conv_chain_supported(d), _C.lib().yb_last_error().decode()
        plan = _C.Plan([d], DEV)
        plan.run()
        torch.cuda.synchronize()
        return out2[..., :C2].clone()

    tol = 2.0 ** -9 if dtype == torch.float16 else 2.0 ** -6
    got2 = launch(True)
    ref1 = F.silu(F.conv2d(x.float().permute(0, 3, 1, 2), w1.float().to(DEV), b1.to(DEV), 1, p))
    if residual:
        ref1 = ref1 + res.float().permute(0, 3, 1, 2)
    got1 = cat[..., :C1].float().permute(0, 3, 1, 2)
    e1 = (got1 - ref1).abs()
    bad1 = int((e1 > tol * (1 + ref1.abs())).sum())
    if extra:
        assert torch.equal(cat[..., C1:], cat0[..., C1:])                    # the extra window is only read
    a2 = torch.cat([cat[..., :c_own], cat[..., C1:C1 + c_own]], -1) if extra else cat[..., :c_own]
    ref2 = F.conv2d(a2.float().permute(0, 3, 1, 2), w2.float().to(DEV), b2.to(DEV))
    if act2:
        ref2 = F.silu(ref2)
    e2 = (got2.float().permute(0, 3, 1, 2) - ref2).abs()
    bad2 = int((e2 > tol * (1 + ref2.abs())).sum())
    print(f"chain N{N} {H}x{W} {Cin}->{C1} k{k} -> [{c_own}{'+' + str(c_own) if extra else ''}]->{C2} {dtype}: "
          f"first max_err {e1.max().item():.3e} viol {bad1}; tail max_err {e2.max().item():.3e} viol {bad2}")
    if bad2:
        idx = (e2 > tol * (1 + ref2.abs())).nonzero()[:8]
        print("tail violations (n,c,y,x):", idx.tolist(), "got/ref/err:",
              [(round(float(got2.float().permute(0, 3, 1, 2)[tuple(i)]), 5), round(float(ref2[tuple(i)]), 5), round(float(e2[tuple(i)]), 5))
               for i in idx])
    if bad1:
        idx = (e1 > tol * (1 + ref1.abs())).nonzero()[:8]
        print("first-output violations (n,c,y,x):", idx.tolist(), "got/ref:", [(float(got1[tuple(i)]), float(ref1[tuple(i)])) for i in idx])
    assert torch.all(out2[..., C2:] == 7.0)
    assert bad1 == 0 and bad2 == 0
    got2c = launch(True)
    nd = (got2c != got2)
    if nd.any():
        print("NONDETERMINISTIC tail (two store_first=1 launches):", int(nd.sum()), "elements, first", nd.nonzero()[:6].tolist())
    assert torch.equal(got2c, got2)              # same launch twice: bit-identical
    if not store_first:
        got2b = launch(False)
        df = (got2b != got2)
        if df.any():
            idx = df.nonzero()
            print("store_first=0 differs in", int(df.sum()), "elements; first", idx[:8].tolist(), "rows(n,y,x) distinct:",
                  len({tuple(i[:3].tolist()) for i in idx}), "max diff", float((got2b.float() - got2.float()).abs().max()))
        assert torch.equal(got2b, got2)
        assert torch.equal(cat, cat0)            # nothing of the first output was written


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_chain_1x1_into_bottleneck_cv1(dtype):
    """C3: cv1||cv2 (one 1x1 GEMM, 2c outputs) -> m.0.cv1 over its first c channels (common.py:168-172)."""
    run_chain(2, 40, 44, 64, 64, 1, 32, 32, dtype=dtype, seed=1)        # c = 32: half a 64-column box feeds the tail
    run_chain(3, 24, 40, 128, 128, 1, 64, 64, dtype=dtype, seed=2)      # c = 64: box 0 of two
    run_chain(1, 17, 19, 256, 128, 1, 64, 64, dtype=dtype, seed=3)      # ragged M (323 pixels), 256 input channels
    run_chain(2, 16, 16, 64, 64, 1, 32, 32, dtype=dtype, seed=4, act2=False)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_chain_3x3_into_next_cv1_and_cv3(dtype):
    """Bottleneck 3x3 (+ shortcut) -> the next bottleneck's cv1 (common.py:111-116), and the last bottleneck -> cv3
    over cat(m_out, cv2(x)) with the cv2 half fetched per tile (common.py:173); first output stored / not stored."""
    run_chain(2, 40, 44, 64, 64, 3, 64, 64, residual=True, dtype=dtype, seed=5)                       # m.i.cv2 -> m.(i+1).cv1
    run_chain(2, 40, 44, 64, 64, 3, 64, 128, extra=True, residual=True, dtype=dtype, seed=6, store_first=False)
    run_chain(2, 48, 40, 32, 32, 3, 32, 64, extra=True, residual=True, dtype=dtype, seed=7, store_first=False)
    run_chain(1, 20, 20, 64, 64, 3, 64, 128, extra=True, residual=False, dtype=dtype, seed=8, store_first=False)   # wrap tiles


def test_chain_many_tiles_per_cta():
    """Bench-like extents: tens of tiles per persistent CTA (mbarrier phases of the tail hand-off wrap many times)."""
    run_chain(8, 160, 160, 64, 64, 1, 32, 32, seed=9)
    run_chain(8, 160, 160, 32, 32, 3, 32, 64, extra=True, residual=True, seed=10, store_first=False)
    run_chain(16, 80, 80, 64, 64, 3, 64, 128, extra=True, residual=True, seed=11, store_first=False)
