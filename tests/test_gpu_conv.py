"""wgmma implicit-GEMM convolution vs a plain fp64 PyTorch conv on the same fp16/bf16-rounded operands (H100)."""
import pytest
import torch

import conv_cases as C
import stagewise as S
from yolort_b200 import _C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def run_conv(N, H, W, Cin, Cout, k, s, p, dtype=torch.float16, act=True, residual=False, in_pad=0, out_pad=0, seed=0,
             bias_scale=0.5, force_im2col=False, force_planes=False, **kw):
    """One convolution through tests/conv_cases.py: the fp64 reference bound, the channel sentinels and the guard image,
    bit-identical relaunches (one-CTA launch of a two-CTA plan included), and the stage-wise bound of SURVEY.md
    section 8c, tol * (1 + |ref|).  Further keyword arguments are Case fields (residual / input / output windows,
    reserved bits...)."""
    assert p == k // 2
    act_code = {True: C.SILU, False: C.NONE, "hardswish": C.HSWISH, "leaky": C.LEAKY, "relu": C.RELU}[act]
    case = C.Case(f"conv N{N} {H}x{W} {Cin}->{Cout} k{k}s{s}", N, H, W, Cin, Cout, k=k, s=s, dtype=dtype, act=act_code,
                  residual=residual, in_cstride=Cin + in_pad, in_off=in_pad // 2 // 8 * 8, out_cstride=Cout + out_pad,
                  out_off=out_pad // 2 // 8 * 8, seed=seed, bias_scale=bias_scale,
                  reserved=((_C.YB_CONV_FORCE_IM2COL if force_im2col else 0) |
                            (_C.YB_CONV_FORCE_PLANES if force_planes else 0)), **kw)
    return C.check_case(case, DEV, legacy_tol=S.TOL[dtype])


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
    maps, against the fp64 convolution."""
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
    """3x3 / stride 2 on the halo-patch kernel (two column-parity planes per chunk) vs the fp64 convolution, and vs
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
    persistent CTA), against the fp64 convolution of the same operands."""
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
    [first_out[:c_own] | extra(c_own channels)] -> C2 channels, through tests/conv_cases.py.  Checks: the library
    accepts the fusion; the first output against fp64 on the rounded inputs; the tail against fp64 applied to the STORED
    first output (= exactly the fp16 tile the tail consumed on chip); the extra window is only read; and, with
    store_first=False, bit equality of the tail with the store_first=True run (the flag only gates the TMA store) and
    nothing of the first output written."""
    chain = C.Chain(c_own, C2, extra=extra, store_first=store_first, act2=C.SILU if act2 else C.NONE)
    case = C.Case(f"chain N{N} {H}x{W} {Cin}->{C1} k{k} -> [{c_own}{'+' + str(c_own) if extra else ''}]->{C2}",
                  N, H, W, Cin, C1, k=k, dtype=dtype, residual=residual, seed=seed, chain=chain)
    return C.check_case(case, DEV, legacy_tol=S.TOL[dtype])


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
