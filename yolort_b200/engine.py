"""Lowering of the YOLOv5 r6.0 graph (backbone + PAN + head) to a native launch plan.

The reference executes ~60-126 `conv2d -> batch_norm -> silu` triples plus `cat`/`Upsample`/
`max_pool2d` as separate PyTorch ops (yolort/models/backbone_utils.py:54-57,
path_aggregation_network.py:199-239, box_head.py:68-82).  Here the module tree is walked ONCE per
(batch, canvas) shape and turned into a flat list of `yb_op_desc` for libyolort_b200.so:

  * BatchNorm (eps = module.eps = 1e-3) is folded into the conv weights in fp64, then rounded to the
    compute dtype; the folded shift becomes the fp32 epilogue bias.
  * activations live in NHWC buffers of one arena; every `torch.cat` of the reference disappears
    because producers write straight into channel windows of the concat buffer.
  * C3's sibling 1x1 convs cv1 and cv2 (common.py:168-169) read the same input, so they run as one
    GEMM with concatenated output channels.
  * the 6x6/s2 stem (darknetv6.py:82) runs as a 3x3/s1 conv over the space-to-depth input the
    letterbox kernel emits (exact rewrite: tap kh = 2a+dy, kw = 2b+dx).

Host code only prepares descriptors; all arithmetic happens in csrc/*.cu.
"""
import ctypes
import math
import os
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _C
from .models.common import C3, C3TR, BottleneckCSP, Conv, Focus, SPP, TransformerBlock


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


GLOBAL = 0           # _Buf.div of a buffer with one pixel per image whatever the canvas (pooled vectors)


@dataclass
class _Buf:
    name: str
    div: int          # spatial divisor w.r.t. the canvas, or GLOBAL
    C: int            # total channels (pixel stride)
    offset: int = 0   # byte offset in the arena
    esz: int = 2      # bytes per element: 2 (fp16 / bf16), 1 (e4m3 buffers of an FP8 plan)

    def hw(self, H: int, W: int) -> Tuple[int, int]:
        """Spatial extent of this buffer on an H x W canvas."""
        return (1, 1) if self.div == GLOBAL else (H // self.div, W // self.div)


@dataclass
class _View:
    buf: _Buf
    ch0: int
    C: int


@dataclass(kw_only=True)
class _Op:
    kind: int
    src: _View
    dst: _View
    ksize: int = 1
    stride: int = 1
    pad: int = 0
    act: int = _C.YB_ACT_NONE
    weight: Optional[torch.Tensor] = None  # packed [Cout_pad, taps, Cin_pad] compute dtype
    bias: Optional[torch.Tensor] = None    # fp32 [Cout_pad]
    residual: Optional[_View] = None
    name: str = ""
    flops_per_pixel: int = 0               # 2*MACs per output pixel of the REFERENCE conv (algorithmic work)
    pack: int = 1                          # horizontally adjacent pixels treated as ONE pixel with pack x channels
    force_im2col: bool = False             # keep this 3x3/s1 conv on the generic im2col kernel
    band: bool = False                     # weight is the banded super-pixel stem matrix (stem_band), Cin_pad 64
    # The NEXT op of the list is a 1x1 convolution over this op's output (channels [0, chain_own) of it, followed by the
    # channels of `chain_extra` if set) and may run as this op's chained tail in the same launch (yb_conv_chain);
    # `chain_store`: this op's output is still read by somebody else and has to be written to memory.
    chain_own: int = 0
    chain_extra: Optional[_View] = None
    chain_store: bool = True
    # FP8 plans (lower_fp8): element type code of the op when it differs from the plan's compute dtype (e4m3 ops; the
    # QUANTIZE op carries its source type), and the option bits of an e4m3 convolution (16-bit head outputs)
    dtype: Optional[int] = None
    reserved: int = 0


# ---------------------------------------------------------------------------------------------------
# parameter preparation
# ---------------------------------------------------------------------------------------------------
def bn_scale_shift(bn: nn.BatchNorm2d) -> Tuple[torch.Tensor, torch.Tensor]:
    """gamma/sqrt(var+eps) and beta - mean*gamma/sqrt(var+eps) in fp64 (on the parameters' device: IEEE fp64
    mul/div/sqrt give the same bits on the host and on the GPU)."""
    scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    shift = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
    return scale, shift


def fold_conv_bn(m: Conv) -> Tuple[torch.Tensor, torch.Tensor]:
    """w' = w * gamma/sqrt(var+eps), b' = beta - mean*gamma/sqrt(var+eps), in fp64.
    (Equivalent to conv -> BatchNorm2d.eval(), yolort/v5/models/common.py:60-70.)"""
    scale, shift = bn_scale_shift(m.bn)
    return m.conv.weight.detach().double() * scale.view(-1, 1, 1, 1), shift


def act_code(act: nn.Module) -> int:
    if isinstance(act, nn.SiLU):
        return _C.YB_ACT_SILU
    if isinstance(act, nn.Hardswish):
        return _C.YB_ACT_HARDSWISH
    if isinstance(act, nn.ReLU):
        return _C.YB_ACT_RELU
    if isinstance(act, nn.Identity):
        return _C.YB_ACT_NONE
    raise NotImplementedError(f"no epilogue for activation {type(act).__name__}")


def focus_to_s2d(w: torch.Tensor) -> torch.Tensor:
    """Focus conv weight [Co,12,3,3] -> [Co,16,3,3] over the plan's space-to-depth input.  focus_transform
    (common.py:237-240) orders the four parities as (row,col) = (0,0), (1,0), (0,1), (1,1); the plan's input channel
    is (dy*2+dx)*4 + c with c == 3 a zero channel, so this is a pure channel permutation (stride 1, pad 1 kept)."""
    co, ci, kh, kw = w.shape
    assert ci == 12 and (kh, kw) == (3, 3)
    out = torch.zeros((co, 16, 3, 3), dtype=w.dtype, device=w.device)
    for g, (dy, dx) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        q = (dy * 2 + dx) * 4
        out[:, q:q + 3] = w[:, 3 * g:3 * g + 3]
    return out


def stem_to_s2d(w: torch.Tensor) -> torch.Tensor:
    """[Co,3,6,6] stride-2 pad-2 kernel -> [Co,16,3,3] stride-1 pad-1 kernel over the space-to-depth
    input whose channel is (dy*2+dx)*4 + c (c == 3 is a zero channel)."""
    co = w.shape[0]
    out = torch.zeros((co, 16, 3, 3), dtype=w.dtype, device=w.device)
    for a in range(3):
        for b in range(3):
            for dy in range(2):
                for dx in range(2):
                    q = (dy * 2 + dx) * 4
                    out[:, q:q + 3, a, b] = w[:, :, 2 * a + dy, 2 * b + dx]
    return out


def stem_s2_to_s2d(w: torch.Tensor) -> torch.Tensor:
    """[Co,3,3,3] stride-2 pad-1 kernel -> [Co,16,3,3] stride-1 pad-1 kernel over the space-to-depth input whose channel
    is (dy*2+dx)*4 + c (c == 3 is a zero channel).  Output pixel y reads input rows 2y-1+ky = 2(y-1+a)+dy, so the taps map
    as ky=0 -> (a=0, dy=1), ky=1 -> (a=1, dy=0), ky=2 -> (a=1, dy=1), the same in x; the a=2 / b=2 taps stay zero."""
    co = w.shape[0]
    assert tuple(w.shape[1:]) == (3, 3, 3)
    out = torch.zeros((co, 16, 3, 3), dtype=w.dtype, device=w.device)
    tap = ((0, 1), (1, 0), (1, 1))
    for ky, (a, dy) in enumerate(tap):
        for kx, (b, dx) in enumerate(tap):
            q = (dy * 2 + dx) * 4
            out[:, q:q + 3, a, b] = w[:, :, ky, kx]
    return out


def stem_superpixel(w: torch.Tensor, b: torch.Tensor, pack: int = 4) -> Tuple[torch.Tensor, torch.Tensor]:
    """Rewrite a 3x3/s1/p1 conv over C-channel pixels as a 3x3/s1/p1 conv over "super-pixels" of `pack`
    horizontally adjacent pixels (pack*C input channels, pack*Co output channels, width / pack).

    Exact: output pixel x = pack*X + po reads input pixels x + b - 1 = pack*(X + S - 1) + pi, i.e. column tap
    b = pack*(S-1) + pi - po + 1 when that lies in {0,1,2}; all other entries of the expanded kernel are zero.
    The memory layouts do not change (NHWC rows are contiguous), only the GEMM's shape does: the 16-channel
    space-to-depth stem input would otherwise be fetched by the TMA unit in 32-byte rows; as 128-byte super-pixels the stem runs like an ordinary 64->128 3x3 layer."""
    co, ci, kh, kw = w.shape
    assert (kh, kw) == (3, 3)
    out = torch.zeros((pack * co, pack * ci, 3, 3), dtype=w.dtype, device=w.device)
    for po in range(pack):
        for pi in range(pack):
            for S in range(3):
                bcol = pack * (S - 1) + pi - po + 1
                if 0 <= bcol <= 2:
                    out[po * co:(po + 1) * co, pi * ci:(pi + 1) * ci, :, S] = w[:, :, :, bcol]
    return out, b.repeat(pack)


def stem_band(w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Banded form of `stem_superpixel(w, b, pack=4)` for a 16-channel 3x3/s1/p1 conv (the space-to-depth stem).

    A group of 4 output pixels (one super-pixel X) reads, per filter row, the 6 input pixels 4X-1 .. 4X+4; in the
    patch kernel's shared-memory patch those 6 x 16 channels are 192 contiguous bytes.  Row `po*Co + co` of the result
    holds, per filter row ky, the 96 weights over (r, c) with r = po + kx the position inside that span; everything
    else of the 4Co x (3*3*64) super-pixel matrix is structurally zero and is not stored.  Layout
    [4*Co, 3, 128]: 96 real K-columns per filter row padded to two 64-column blocks (the kernel multiplies 6 K=16
    steps per row and never touches the padding)."""
    co, ci, kh, kw = w.shape
    assert (ci, kh, kw) == (16, 3, 3)
    out = torch.zeros((4 * co, 3, 128), dtype=w.dtype, device=w.device)
    for po in range(4):
        for kx in range(3):
            r = po + kx
            out[po * co:(po + 1) * co, :, r * 16:(r + 1) * 16] = w[:, :, :, kx].permute(0, 2, 1)   # [co, ky, c]
    return out, b.repeat(4)


def pack_weight(w: torch.Tensor, dtype: torch.dtype, device: torch.device) -> Tuple[torch.Tensor, int, int]:
    """[Co,Ci,k,k] -> K-major [Co_pad, k*k, Ci_pad], zero padded.  Ci_pad is a multiple of 64 once Ci > 32, so that the
    kernels always fetch 128-byte (SWIZZLE_128B) operand rows: 48-, 80- or 96-channel layers (yolov5m / x) would
    otherwise fall to 32- or 64-byte TMA rows, which the TMA unit moves at a fraction of the rate.  The padding costs no
    tensor work: the kernels issue only ceil(Ci/16) K-steps of the last chunk (`kk_last`)."""
    co, ci, kh, kw = w.shape
    ci_pad, co_pad = (_round_up(ci, 64) if ci > 32 else _round_up(ci, 16)), _round_up(co, 16)
    p = torch.zeros((co_pad, kh * kw, ci_pad), dtype=torch.float64, device=w.device)
    p[:co, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return p.to(dtype).to(device).contiguous(), ci_pad, co_pad


def pack_bias(b: torch.Tensor, co_pad: int, device: torch.device) -> torch.Tensor:
    out = torch.zeros((co_pad,), dtype=torch.float64, device=b.device)
    out[: b.numel()] = b
    return out.to(torch.float32).to(device).contiguous()


# ---------------------------------------------------------------------------------------------------
# graph lowering
# ---------------------------------------------------------------------------------------------------
class _Lowering:
    def __init__(self, dtype: torch.dtype, device: torch.device):
        self.bufs: List[_Buf] = []
        self.ops: List[_Op] = []
        self.dtype = dtype
        self.device = device

    def buf(self, name: str, div: int, C: int) -> _Buf:
        b = _Buf(name, div, C)
        self.bufs.append(b)
        return b

    def conv(self, name, w, b, src: _View, dst: _View, k, s, p, act, residual=None, ref_flops_per_pixel=None, pack=1, force_im2col=False):
        assert w.shape[1] == src.C * pack and w.shape[0] <= dst.C * pack, (name, tuple(w.shape), src.C, dst.C)
        if pack > 1:
            assert src.ch0 == 0 and src.C == src.buf.C and dst.ch0 == 0 and dst.C == dst.buf.C and residual is None
        wp, bp = self.pack(w, b)
        if ref_flops_per_pixel is None:
            ref_flops_per_pixel = 2 * w.shape[0] * w.shape[1] * k * k
        self.ops.append(_Op(kind=_C.YB_OP_CONV, src=src, dst=dst, ksize=k, stride=s, pad=p, act=act, weight=wp, bias=bp,
                            residual=residual, name=name, flops_per_pixel=ref_flops_per_pixel, pack=pack,
                            force_im2col=force_im2col))

    def pack(self, w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Packed weight and fp32 bias of a convolution from its fp64 folded weight and bias."""
        wp, _, co_pad = pack_weight(w, self.dtype, self.device)
        return wp, pack_bias(b, co_pad, self.device)

    def conv_band(self, name, w_band, b, src: _View, dst: _View, act, ref_flops_per_pixel):
        """Stem on the banded super-pixel weights (stem_band): pack 4, 3x3/s1/p1, handled by the patch kernel's
        kBand variant."""
        co4 = w_band.shape[0]
        assert src.C == 16 and src.ch0 == 0 and src.C == src.buf.C and dst.ch0 == 0 and dst.C == dst.buf.C and 4 * dst.C == co4
        assert co4 % 64 == 0 and co4 <= 256, "banded stem needs 64 | 4*Cout <= 256"
        wp = w_band.to(self.dtype).to(self.device).contiguous()
        bp = pack_bias(b, co4, self.device)
        self.ops.append(_Op(kind=_C.YB_OP_CONV, src=src, dst=dst, ksize=3, stride=1, pad=1, act=act, weight=wp, bias=bp,
                            name=name, flops_per_pixel=ref_flops_per_pixel, pack=4, band=True))

    def conv_module(self, name, m: Conv, src: _View, dst: _View, residual=None):
        w, b = fold_conv_bn(m)
        k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
        self.conv(name, w, b, src, dst, k, s, p, act_code(m.act), residual)

    def block(self, name, m, src: _View, dst: _View):
        """C3 (r4.0 / r6.0 graphs), C3TR (yolov5ts) or BottleneckCSP (r3.1)."""
        if isinstance(m, C3TR):      # a C3 subclass: tested first
            self.c3tr(name, m, src, dst)
        elif isinstance(m, C3):
            self.c3(name, m, src, dst)
        elif isinstance(m, BottleneckCSP):
            self.csp(name, m, src, dst)
        else:
            raise NotImplementedError(f"{name}: no lowering for {type(m).__name__}")

    def csp(self, name, m: BottleneckCSP, src: _View, dst: _View):
        """common.py:144-146: cv4(LeakyReLU(BN(cat(cv3(m(cv1(x))), cv2(x))))).  The BatchNorm over the concat is
        per channel, so its two halves fold into the bare convolutions cv3 and cv2 (fp64), each followed by the
        LeakyReLU in its own epilogue; the concat is the channel window the two GEMMs write."""
        div = src.buf.div
        c_ = m.cv1.conv.out_channels
        cat = self.buf(f"{name}.cat", div, 2 * c_)
        scale, shift = bn_scale_shift(m.bn)
        y = _View(self.buf(f"{name}.y", div, c_), 0, c_)
        self.conv_module(f"{name}.cv1", m.cv1, src, y)
        w2 = m.cv2.weight.detach().double() * scale[c_:].view(-1, 1, 1, 1)
        self.conv(f"{name}.cv2+bn", w2, shift[c_:], src, _View(cat, c_, c_), 1, 1, 0, _C.YB_ACT_LEAKY01)
        for i, blk in enumerate(m.m):
            t = _View(self.buf(f"{name}.m{i}.t", div, c_), 0, c_)
            self.conv_module(f"{name}.m.{i}.cv1", blk.cv1, y, t)
            out = _View(self.buf(f"{name}.m{i}.y", div, c_), 0, c_)
            self.conv_module(f"{name}.m.{i}.cv2", blk.cv2, t, out, residual=y if blk.add else None)
            y = out
        w3 = m.cv3.weight.detach().double() * scale[:c_].view(-1, 1, 1, 1)
        self.conv(f"{name}.cv3+bn", w3, shift[:c_], y, _View(cat, 0, c_), 1, 1, 0, _C.YB_ACT_LEAKY01)
        self.conv_module(f"{name}.cv4", m.cv4, _View(cat, 0, 2 * c_), dst)

    def c3(self, name, m: C3, src: _View, dst: _View):
        div = src.buf.div
        c_ = m.cv1.conv.out_channels
        cat = self.buf(f"{name}.cat", div, 2 * c_)
        w1, b1 = fold_conv_bn(m.cv1)
        w2, b2 = fold_conv_bn(m.cv2)
        # cv1 || cv2 as one GEMM: channels [0,c_) = cv1(x), [c_,2c_) = cv2(x)  (common.py:173 cat order)
        self.conv(f"{name}.cv1+cv2", torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), src,
                  _View(cat, 0, 2 * c_), 1, 1, 0, _C.YB_ACT_SILU)
        y = _View(cat, 0, c_)
        n = len(m.m)
        # Pointwise chains (common.py:94-116,149-173): every 1x1 convolution of the block consumes the tile its
        # predecessor has just produced -- cv1||cv2 -> m.0.cv1, m.i.cv2 -> m.(i+1).cv1, m.last.cv2 -> cv3 (whose other
        # half, cv2(x), is fetched per tile).  Marked here, fused per shape where the kernels support it
        # (PlanInstance); the last bottleneck's output is then never written (only cv3 reads it).
        if n > 0:
            self.ops[-1].chain_own = c_
        for i, blk in enumerate(m.m):
            t = self.buf(f"{name}.m{i}.t", div, c_)
            self.conv_module(f"{name}.m.{i}.cv1", blk.cv1, y, _View(t, 0, c_))
            out = _View(cat, 0, c_) if i == n - 1 else _View(self.buf(f"{name}.m{i}.y", div, c_), 0, c_)
            self.conv_module(f"{name}.m.{i}.cv2", blk.cv2, _View(t, 0, c_), out, residual=y if blk.add else None)
            self.ops[-1].chain_own = c_
            if i == n - 1:
                self.ops[-1].chain_extra = _View(cat, c_, c_)
                self.ops[-1].chain_store = False
            y = out
        self.conv_module(f"{name}.cv3", m.cv3, _View(cat, 0, 2 * c_), dst)

    def c3tr(self, name, m: C3TR, src: _View, dst: _View):
        """common.py:360-367: cv3(cat(m(cv1(x)), cv2(x))) with m a TransformerBlock; cv1 || cv2 and cv3 as in c3()."""
        div = src.buf.div
        c_ = m.cv1.conv.out_channels
        cat = self.buf(f"{name}.cat", div, 2 * c_)
        w1, b1 = fold_conv_bn(m.cv1)
        w2, b2 = fold_conv_bn(m.cv2)
        self.conv(f"{name}.cv1+cv2", torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), src,
                  _View(cat, 0, 2 * c_), 1, 1, 0, _C.YB_ACT_SILU)
        self.transformer(f"{name}.m", m.m, _View(cat, 0, c_), _View(cat, 0, c_))
        self.conv_module(f"{name}.cv3", m.cv3, _View(cat, 0, 2 * c_), dst)

    def transformer(self, name, m: TransformerBlock, src: _View, dst: _View):
        """TransformerBlock over the H*W tokens of each image (common.py:334-357, TransformerLayer :308-331) as 1x1
        convolutions (act NONE) around one attention op per layer.  Every linear map in front of the attention folds
        into its neighbour in fp64 and is rounded once:
            pos   p' = (I + W_linear) p + b_linear
            qkv   [W_in,q W_q ; W_in,k W_k ; W_in,v W_v] p' + in_proj_bias          (E -> 3E)
            attn  softmax(Q_h K_h^T / sqrt(d)) V_h per head                          (YB_OP_ATTENTION)
            out   x1 = W_out a + b_out + p'
            fc    x2 = (W_fc2 W_fc1) x1 + x1
        The 1/sqrt(d) scale stays in the attention op.  flops_per_pixel counts the reference's work (q, k, v and
        in_proj are four E x E products; fc1 and fc2 two)."""
        if m.conv is not None:
            raise NotImplementedError(f"{name}: transformer block with an input Conv (c1 != c2)")
        if len(m.tr) == 0:
            raise NotImplementedError(f"{name}: transformer block without layers")
        div = src.buf.div
        E = m.c2
        lin = m.linear
        W = lin.weight.detach().double()
        eye = torch.eye(E, dtype=torch.float64, device=W.device)

        def w4(t):       # [Cout, E] linear map -> 1x1 convolution weight
            return t.reshape(t.shape[0], E, 1, 1)

        x = _View(self.buf(f"{name}.p", div, E), 0, E)
        self.conv(f"{name}.linear(pos)", w4(eye + W), lin.bias.detach().double(), src, x, 1, 1, 0, _C.YB_ACT_NONE,
                  ref_flops_per_pixel=2 * E * E)
        n = len(m.tr)
        for i, layer in enumerate(m.tr):
            ma = layer.ma
            heads = ma.num_heads
            if E % heads or E // heads != 64 or not getattr(ma, "_qkv_same_embed_dim", True) or ma.in_proj_bias is None:
                raise NotImplementedError(f"{name}.tr.{i}: the attention kernel implements 64-wide heads with a packed "
                                          f"in-projection and bias (E={E}, heads={heads})")
            p = f"{name}.tr.{i}"
            w_in = ma.in_proj_weight.detach().double()
            w_qkv = torch.cat([w_in[:E] @ layer.q.weight.detach().double(),
                               w_in[E:2 * E] @ layer.k.weight.detach().double(),
                               w_in[2 * E:] @ layer.v.weight.detach().double()], 0)
            qkv = _View(self.buf(f"{p}.qkv", div, 3 * E), 0, 3 * E)
            self.conv(f"{p}.q|k|v+in_proj", w4(w_qkv), ma.in_proj_bias.detach().double(), x, qkv, 1, 1, 0,
                      _C.YB_ACT_NONE, ref_flops_per_pixel=12 * E * E)
            att = _View(self.buf(f"{p}.attn", div, E), 0, E)
            self.ops.append(_Op(kind=_C.YB_OP_ATTENTION, src=qkv, dst=att, ksize=heads, name=f"{p}.ma(attention)"))
            x1 = _View(self.buf(f"{p}.x1", div, E), 0, E)
            self.conv(f"{p}.ma.out_proj", w4(ma.out_proj.weight.detach().double()), ma.out_proj.bias.detach().double(),
                      att, x1, 1, 1, 0, _C.YB_ACT_NONE, residual=x, ref_flops_per_pixel=2 * E * E)
            out = dst if i == n - 1 else _View(self.buf(f"{p}.y", div, E), 0, E)
            w_fc = layer.fc2.weight.detach().double() @ layer.fc1.weight.detach().double()
            self.conv(f"{p}.fc2*fc1", w4(w_fc), torch.zeros(E, dtype=torch.float64, device=W.device), x1, out, 1, 1, 0,
                      _C.YB_ACT_NONE, residual=x1, ref_flops_per_pixel=4 * E * E)
            x = out

    def spp(self, name, m: SPP, src: _View, dst: _View):
        if tuple(m.k) != (5, 9, 13):
            raise NotImplementedError("SPP pooling kernel implements k=(5,9,13) (the r6.0 neck)")
        div = src.buf.div
        c_ = m.cv1.conv.out_channels
        cat = self.buf(f"{name}.cat", div, 4 * c_)
        self.conv_module(f"{name}.cv1", m.cv1, src, _View(cat, 0, c_))
        self.ops.append(_Op(kind=_C.YB_OP_SPP_POOL, src=_View(cat, 0, c_), dst=_View(cat, c_, 3 * c_),
                            name=f"{name}.pool"))
        self.conv_module(f"{name}.cv2", m.cv2, _View(cat, 0, 4 * c_), dst)

    def upsample(self, name, src: _View, dst: _View):
        self.ops.append(_Op(kind=_C.YB_OP_UPSAMPLE2X, src=src, dst=dst, name=name))

    def stem(self, prefix: str, stem: nn.Module, stem_variant: str) -> Tuple[_Buf, _View]:
        """The CSPDarknet stem over the plan's space-to-depth canvas: (canvas buffer, stem output view).  A Focus
        (r3.1 / r4.0) is a channel permutation of the s2d input, the r6.0 6x6/s2/p2 convolution an exact 3x3/s1/p1
        convolution over it."""
        if isinstance(stem, Focus):       # r3.1 / r4.0: Focus = 2x2 space-to-depth + 3x3/s1/p1 conv (darknetv4.py:82)
            stem = stem.conv
            if stem.conv.kernel_size != (3, 3) or stem.conv.stride != (1, 1) or stem.conv.padding != (1, 1):
                raise NotImplementedError("Focus stem must be the 3x3/s1/p1 convolution")
            to_s2d = focus_to_s2d
        else:                             # r6.0: 6x6/s2/p2 conv == 3x3/s1/p1 over the same space-to-depth input
            if stem.conv.kernel_size != (6, 6) or stem.conv.stride != (2, 2) or stem.conv.padding != (2, 2):
                raise NotImplementedError("stem must be the r6.0 6x6/s2/p2 convolution")
            to_s2d = stem_to_s2d
        w, b = fold_conv_bn(stem)
        return self.s2d_stem(f"{prefix}.0", w, b, to_s2d, act_code(stem.act), stem_variant)

    def s2d_stem(self, name: str, w: torch.Tensor, b: torch.Tensor, to_s2d, act: int, variant: str,
                 what: str = "3x3") -> Tuple[_Buf, _View]:
        """The first convolution (folded weight `w`, bias `b`), rewritten by `to_s2d` into a 3x3/s1/p1 convolution over
        the plan's space-to-depth canvas: (canvas buffer, output view).  `variant`: "auto" | "band" | "superpixel" |
        "im2col"; `what` names the rewrite in the op name.  flops_per_pixel counts the reference convolution's work
        per super-pixel."""
        x0 = self.buf("input.s2d", 2, 16)
        co = w.shape[0]
        t0 = self.buf(name, 2, co)
        w_s2d = to_s2d(w)
        # The stem runs over "super-pixels" of 4 horizontally adjacent s2d pixels (128-byte TMA rows instead of 32).  Its
        # expanded weight matrix is block-banded, and when the band (6 slabs of 4*Cout x 64) fits in shared memory next
        # to two patches (4*Cout <= 128: yolov5n / s) the banded kernel variant multiplies only the band; wider stems
        # (m / l / x) use the dense super-pixel form.
        spk = 4
        co4 = spk * co
        flops = spk * 2 * w.numel()
        if variant == "band" or (variant == "auto" and co4 % 64 == 0 and co4 <= 128
                                 and act in (_C.YB_ACT_SILU, _C.YB_ACT_NONE)):
            w_b, b_b = stem_band(w_s2d, b)
            self.conv_band(f"{name}(stem: banded {what} over s2d super-pixels)", w_b, b_b, _View(x0, 0, 16),
                           _View(t0, 0, co), act, ref_flops_per_pixel=flops)
        else:
            w_sp, b_sp = stem_superpixel(w_s2d, b, spk)
            self.conv(f"{name}(stem: {what} over s2d super-pixels)", w_sp, b_sp, _View(x0, 0, 16), _View(t0, 0, co),
                      3, 1, 1, act, ref_flops_per_pixel=flops, pack=spk, force_im2col=(variant == "im2col"))
        return x0, _View(t0, 0, co)

    def stages(self, prefix: str, mods: List[nn.Module], cur: _View, tap_dst: Dict[int, _View]) -> _View:
        """Modules 1.. of a CSPDarknet body after the stem: 3x3/s2 Convs, blocks (C3 / BottleneckCSP) and the closing
        SPP of r3.1 / r4.0.  Module i writes into tap_dst[i] when given (a concat window of the neck).  Returns the
        last output."""
        div = cur.buf.div
        for i, m in enumerate(mods, start=1):
            name = f"{prefix}.{i}"
            if isinstance(m, Conv):
                div *= 2
                co = m.conv.out_channels
                t = self.buf(name, div, co)
                self.conv_module(name, m, cur, _View(t, 0, co))
                cur = _View(t, 0, co)
            elif isinstance(m, SPP):      # r3.1 / r4.0 keep the SPP as the last body module (darknetv4.py:97)
                co = m.cv2.conv.out_channels
                dst = _View(self.buf(name, div, co), 0, co)
                self.spp(name, m, cur, dst)
                cur = dst
            else:
                if not isinstance(m, (C3, BottleneckCSP)):
                    raise NotImplementedError(f"{name}: no lowering for {type(m).__name__}")
                co = (m.cv3 if isinstance(m, C3) else m.cv4).conv.out_channels
                dst = tap_dst.get(i) or _View(self.buf(name, div, co), 0, co)
                assert dst.C == co
                self.block(name, m, cur, dst)
                cur = dst
        return cur

    def heads(self, feats: List[_View], convs) -> List[_Buf]:
        """The detection head: one 1x1 convolution `convs[i]` (an nn.Conv2d with bias, no activation) per level over
        feats[i], into buffer "head.{i}" with the output channels padded to 16.  Returns those buffers."""
        head_bufs = []
        for i, (feat, conv) in enumerate(zip(feats, convs)):
            co_buf = _round_up(conv.out_channels, 16)
            hb = self.buf(f"head.{i}", feat.buf.div, co_buf)
            self.conv(f"head.head.{i}", conv.weight.detach().double(), conv.bias.detach().double(), feat,
                      _View(hb, 0, co_buf), 1, 1, 0, _C.YB_ACT_NONE)
            head_bufs.append(hb)
        return head_bufs

    def avgpool(self, name, src: _View, dst: _View):
        self.ops.append(_Op(kind=_C.YB_OP_AVGPOOL, src=src, dst=dst, name=name))

    def dwconv(self, name, w, b, src: _View, dst: _View, k, s, act):
        """Depthwise k x k / s convolution (YB_OP_DWCONV): w [C,1,k,k] (BN folded, fp64) -> [k*k][C] in the compute
        dtype, b -> fp32 [C]."""
        C = src.C
        assert tuple(w.shape) == (C, 1, k, k) and dst.C == C, (name, tuple(w.shape), src.C, dst.C)
        wp = w.reshape(C, k * k).t().contiguous().to(self.dtype).to(self.device)
        bp = b.to(torch.float32).to(self.device).contiguous()
        self.ops.append(_Op(kind=_C.YB_OP_DWCONV, src=src, dst=dst, ksize=k, stride=s, pad=k // 2, act=act, weight=wp,
                            bias=bp, name=name, flops_per_pixel=2 * k * k * C))

    def squeeze_excitation(self, name, m: nn.Module, x: _View):
        """torchvision.ops.SqueezeExcitation (ops/misc.py): x * hardsigmoid(fc2(relu(fc1(mean_hw(x))))) in place
        (YB_OP_SE).  fc1 / fc2 stay fp32 and unrounded, transposed so that the kernel reads them coalesced."""
        if not (isinstance(m.activation, nn.ReLU) and isinstance(m.scale_activation, nn.Hardsigmoid)):
            raise NotImplementedError(f"{name}: SE kernel implements relu / hardsigmoid")
        S, C = m.fc1.out_channels, m.fc1.in_channels
        assert C == x.C and m.fc2.out_channels == C and m.fc2.in_channels == S
        w1t = m.fc1.weight.detach().reshape(S, C).t().float()
        w2t = m.fc2.weight.detach().reshape(C, S).t().float()
        w = torch.cat([w1t.reshape(-1), w2t.reshape(-1)]).to(self.device).contiguous()
        b = torch.cat([m.fc1.bias.detach().float(), m.fc2.bias.detach().float()]).to(self.device).contiguous()
        self.ops.append(_Op(kind=_C.YB_OP_SE, src=x, dst=x, ksize=S, weight=w, bias=b, name=name))

    def conv_norm_act(self, name, m: nn.Sequential, src: _View, dst: _View, residual=None):
        """torchvision Conv2dNormActivation: conv [-> FrozenBatchNorm2d] [-> activation], one group, BN folded in fp64
        (scale = w * rsqrt(rv + eps), shift = b - rm * scale)."""
        conv, bn, act = _split_conv_norm_act(name, m)
        if conv.groups != 1:
            raise NotImplementedError(f"{name}: grouped convolution outside the depthwise case")
        w, b = _fold_conv_norm(conv, bn)
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        self.conv(name, w, b, src, dst, k, s, p, act, residual)

    def inverted_residual(self, name, m: nn.Module, src: _View) -> _View:
        """torchvision InvertedResidual: [1x1 expand] -> depthwise k x k / s -> [SE] -> 1x1 project (no act)
        [+ input when use_res_connect].  Every fact comes from the modules."""
        from torchvision.ops import SqueezeExcitation

        x = src
        mods = list(m.block)
        for j, sub in enumerate(mods):
            sn = f"{name}.block.{j}"
            if isinstance(sub, SqueezeExcitation):
                self.squeeze_excitation(sn, sub, x)
                continue
            conv, bn, act = _split_conv_norm_act(sn, sub)
            if conv.groups > 1:
                if conv.groups != conv.in_channels or conv.out_channels != conv.in_channels:
                    raise NotImplementedError(f"{sn}: grouped convolution that is not depthwise")
                k, s = conv.kernel_size[0], conv.stride[0]
                if conv.kernel_size != (k, k) or conv.stride != (s, s) or conv.padding != (k // 2, k // 2) \
                        or conv.dilation != (1, 1):
                    raise NotImplementedError(f"{sn}: depthwise kernel implements square k x k / s, pad k // 2")
                w, b = _fold_conv_norm(conv, bn)
                dst = _View(self.buf(sn, x.buf.div * s, x.C), 0, x.C)
                self.dwconv(sn, w, b, x, dst, k, s, act)
            else:
                last = j == len(mods) - 1
                co = conv.out_channels
                dst = _View(self.buf(name if last else sn, x.buf.div, co), 0, co)
                self.conv_norm_act(sn, sub, x, dst, residual=src if (last and m.use_res_connect) else None)
            x = dst
        return x


class _Fp8Lowering(_Lowering):
    """The same walk for an FP8 plan (lower_fp8): the stem is packed in the compute dtype and one YB_OP_QUANTIZE
    converts its output to e4m3; every later convolution packs its weight to e4m3 at once, with one scale per output
    channel (`s_w[op index]`, fp64).  The activation scales, hence the epilogue multipliers, come later."""

    def __init__(self, dtype: torch.dtype, device: torch.device):
        super().__init__(dtype, device)
        self.quantized = False
        self.s_w: Dict[int, torch.Tensor] = {}

    def pack(self, w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if not self.quantized:
            return super().pack(w, b)
        s_w = e4m3_scales(w.abs().amax(dim=(1, 2, 3)))
        self.s_w[len(self.ops)] = s_w
        wq = pack_weight_e4m3(w, s_w, self.device)
        return wq, pack_bias(b, wq.shape[0], self.device)

    def stem(self, prefix: str, stem: nn.Module, stem_variant: str) -> Tuple[_Buf, _View]:
        x0, out = super().stem(prefix, stem, stem_variant)
        q = _View(self.buf(f"{prefix}.0(e4m3)", out.buf.div, out.C), 0, out.C)
        self.ops.append(_Op(kind=_C.YB_OP_QUANTIZE, src=out, dst=q, name=f"{prefix}.0(quantize)"))
        self.quantized = True
        return x0, q


def lower_yolo(model: nn.Module, dtype: torch.dtype, device: torch.device, stem_variant: str = "auto",
               fp8: bool = False):
    """Walk YOLO.backbone / YOLO.head and emit (lowering, input_buf, head_bufs, features).
    `stem_variant`: "auto" | "band" | "superpixel" | "im2col" (the last two are kept for parity tests and A/B timing).
    `fp8`: the walk of an FP8 plan (_Fp8Lowering; lower_fp8 quantises it)."""
    L = (_Fp8Lowering if fp8 else _Lowering)(dtype, device)
    bb = model.backbone
    body, pan = bb.body, bb.pan
    ch = list(bb.out_channels)
    nl = len(ch)                                   # detection levels: 3, or 4 with the P6 intermediate block
    has_p6 = getattr(pan, "intermediate_blocks", None) is not None
    if nl not in (3, 4) or len(model.head.head) != nl or has_p6 != (nl == 4):
        raise NotImplementedError("lowering covers the r6.0 topologies: 3 levels, or 4 levels with the P6 block")

    x0, stem_out = L.stem("body", body["0"], stem_variant)

    # Concat buffers of the neck (path_aggregation_network.py:215-237), level l at stride 8 << l:
    #   cat_dn[l] = [up(lateral from level l+1) | body tap of level l]   (descending pass, l < nl-1)
    #   cat_up[l] = [down(result of level l-1) | lateral of level l]     (ascending pass,  l > 0)
    # lateral k (k = 1..nl-1) is the 1x1 conv output at level nl-k; producers write straight into these windows.
    taps = (4, 6, 8)
    cat_dn = {l: L.buf(f"pan.cat{nl - 1 - l}[up(lat{nl - 1 - l})|f{taps[l]}]", 8 << l, 2 * ch[l]) for l in range(nl - 1)}
    cat_up = {l: L.buf(f"pan.cat_p{l + 3}[down(p{l + 2})|lat{nl - l}]", 8 << l, 2 * ch[l - 1]) for l in range(1, nl)}

    tap_dst = {taps[l]: _View(cat_dn[l], ch[l], ch[l]) for l in range(min(nl - 1, 3))}
    top = L.stages("body", [body[str(i)] for i in range(1, 9)], stem_out, tap_dst)
    if has_p6:   # IntermediateLevelP6 (path_aggregation_network.py:34-41): stride-64 level from the last tap
        p6m = pan.intermediate_blocks.p6
        t = _View(L.buf("pan.p6.conv", 64, ch[3]), 0, ch[3])
        L.conv_module("pan.intermediate_blocks.p6.0", p6m[0], top, t)
        top = _View(L.buf("pan.p6.c3", 64, ch[3]), 0, ch[3])     # (the ascending pass's level-6 result is "pan.p6")
        L.block("pan.intermediate_blocks.p6.1", p6m[1], t, top)

    inner, layer = pan.inner_blocks, pan.layer_blocks
    # descending pass (`:215-222`): idx-th iteration works at level nl-1-idx
    last = _View(L.buf("pan.spp", 8 << (nl - 1), ch[-1]), 0, ch[-1])
    if isinstance(inner[0], SPP):
        L.spp("pan.inner_blocks.0", inner[0], top, last)
    else:                             # r3.1 / r4.0: a block without shortcut (path_aggregation_network.py:108-109)
        L.block("pan.inner_blocks.0", inner[0], top, last)
    for idx in range(nl - 1):
        l = nl - 1 - idx
        if idx > 0:
            u = _View(L.buf(f"pan.u{idx}", 8 << l, ch[l]), 0, ch[l])
            L.block(f"pan.inner_blocks.{3 * idx}", inner[3 * idx], _View(cat_dn[l], 0, 2 * ch[l]), u)
            last = u
        lat = _View(cat_up[l], ch[l - 1], ch[l - 1])
        L.conv_module(f"pan.inner_blocks.{3 * idx + 1}", inner[3 * idx + 1], last, lat)
        L.upsample(f"pan.inner_blocks.{3 * idx + 2}", lat, _View(cat_dn[l - 1], 0, ch[l - 1]))
    # ascending pass (`:226-237`)
    results = [_View(L.buf("pan.p3", 8, ch[0]), 0, ch[0])]
    L.block("pan.layer_blocks.0", layer[0], _View(cat_dn[0], 0, 2 * ch[0]), results[0])
    for idx in range(nl - 1):
        l = idx + 1
        L.conv_module(f"pan.layer_blocks.{2 * idx + 1}", layer[2 * idx + 1], results[idx], _View(cat_up[l], 0, ch[idx]))
        r = _View(L.buf(f"pan.p{l + 3}", 8 << l, ch[l]), 0, ch[l])
        L.block(f"pan.layer_blocks.{2 * idx + 2}", layer[2 * idx + 2], _View(cat_up[l], 0, 2 * ch[idx]), r)
        results.append(r)

    return L, x0, L.heads(results, model.head.head), {f"p{l + 3}": r for l, r in enumerate(results)}


# ---------------------------------------------------------------------------------------------------
# FP8 (e4m3) plans
# ---------------------------------------------------------------------------------------------------
E4M3_MAX = 448.0


def e4m3_scale(amax: float) -> float:
    """The smallest power of two s with amax / s <= 448 (1 for an all-zero tensor).  Powers of two make every
    dequantisation and every epilogue multiplier exact."""
    if not amax > 0:
        return 1.0
    s = 2.0 ** math.ceil(math.log2(amax / E4M3_MAX))
    while amax / s > E4M3_MAX:
        s *= 2.0
    while amax / (0.5 * s) <= E4M3_MAX:
        s *= 0.5
    return s


def e4m3_scales(amax: torch.Tensor) -> torch.Tensor:
    """e4m3_scale of every element of `amax`, in fp64 (per-output-channel weight scales)."""
    a = amax.double()
    s = torch.exp2(torch.ceil(torch.log2(a / E4M3_MAX)))
    s = torch.where(a / s > E4M3_MAX, 2.0 * s, s)
    s = torch.where(a / (0.5 * s) <= E4M3_MAX, 0.5 * s, s)
    return torch.where(a > 0, s, torch.ones_like(s))


def e4m3_round(x: torch.Tensor) -> torch.Tensor:
    """fp64 `x` rounded once to the nearest e4m3 value (ties to even, saturating at +-448), still in fp64."""
    _, e = torch.frexp(x)
    q = torch.exp2((torch.clamp(e - 1, min=-6) - 3).to(torch.float64))    # spacing of the binade (subnormals: 2^-9)
    return torch.clamp(torch.round(x / q) * q, -E4M3_MAX, E4M3_MAX)


def pack_weight_e4m3(w: torch.Tensor, s_w: torch.Tensor, device: torch.device) -> torch.Tensor:
    """[Co,Ci,k,k] fp64 with per-output-channel scales s_w -> e4m3 K-major [Co_pad, k*k, Ci_pad] holding w / s_w,
    zero padded.  Ci_pad is a multiple of 128 (one 128-byte TMA row) once Ci > 64, else of 32 (the wgmma K step)."""
    co, ci, kh, kw = w.shape
    ci_pad, co_pad = (_round_up(ci, 128) if ci > 64 else _round_up(ci, 32)), _round_up(co, 16)
    p = torch.zeros((co_pad, kh * kw, ci_pad), dtype=torch.float64, device=w.device)
    p[:co, :, :ci] = e4m3_round(w / s_w.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(co, kh * kw, ci)
    return p.to(torch.float8_e4m3fn).to(device).contiguous()


def scale_groups(L: _Lowering) -> List[List[_Buf]]:
    """Buffers that share one activation scale: every channel window of a buffer (so every concat) by construction, and
    the source and destination of each op that moves values without arithmetic (SPP max-pool, nearest upsample), so
    that those ops are exact in e4m3.  Union-find over the op list, groups in buffer order."""
    parent = {id(b): id(b) for b in L.bufs}

    def find(k):
        while parent[k] != k:
            parent[k] = parent[parent[k]]
            k = parent[k]
        return k

    for op in L.ops:
        if op.kind in (_C.YB_OP_SPP_POOL, _C.YB_OP_UPSAMPLE2X):
            parent[find(id(op.src.buf))] = find(id(op.dst.buf))
    groups: Dict[int, List[_Buf]] = {}
    for b in L.bufs:
        groups.setdefault(find(id(b)), []).append(b)
    return list(groups.values())


def fp8_unsupported(model: nn.Module) -> Optional[str]:
    """Name of the model family when it has no FP8 plan (its ops have no e4m3 kernels), else None."""
    from .models._classifier import DarkNetClassifier
    from .models.yolo_lite import BackboneWithFPN

    if isinstance(model, DarkNetClassifier):
        return f"the DarkNet classifier {type(model).__name__}"
    if isinstance(getattr(model, "backbone", None), BackboneWithFPN):
        return "yolov5_mobilenet_v3_small_fpn"
    if any(isinstance(m, C3TR) for m in model.modules()):
        return "yolov5ts (C3TR transformer neck)"
    return None


def lower_fp8(model: nn.Module, dtype: torch.dtype, device: torch.device, amax: Dict[str, float],
              stem_variant: str = "auto"):
    """The FP8 plan of a YOLOv5 detection model: (lowering, input_buf, head_bufs, features, scale per buffer id).

    The walk is lower_yolo's (_Fp8Lowering).  The stem keeps its fp16 / bf16 kernel and a YB_OP_QUANTIZE converts its
    output; every later op runs on e4m3 buffers, the heads write fp16 / bf16 logits.  `amax` is the calibrated maximum
    of |x| per buffer name of the fp16 / bf16 plan (quantization.calibrate_fp8); a scale group takes the largest of its
    members.  Weights: one scale per output channel from the BN-folded fp64 weight, one rounding to e4m3."""
    why = fp8_unsupported(model)
    if why is not None:
        raise NotImplementedError(f"FP8 inference is not implemented for {why}")
    L, x0, head_bufs, feats = lower_yolo(model, dtype, device, stem_variant, fp8=True)
    qi = next(i for i, op in enumerate(L.ops) if op.kind == _C.YB_OP_QUANTIZE)
    stem_out, stem_q = L.ops[qi].src.buf, L.ops[qi].dst.buf
    wide = {id(x0), id(stem_out)} | {id(b) for b in head_bufs}
    for b in L.bufs:
        if id(b) not in wide:
            b.esz = 1
    missing = sorted(b.name for b in L.bufs if b.esz == 1 and b is not stem_q and b.name not in amax)
    if missing:
        raise ValueError(f"the calibration has no amax for {missing[:4]}... (calibrated for another architecture?)")
    scale: Dict[int, float] = {}
    for group in scale_groups(L):
        q = [b for b in group if b.esz == 1]
        if q:
            s = e4m3_scale(max(amax[stem_out.name if b is stem_q else b.name] for b in q))
            for b in q:
                scale[id(b)] = s
    head_ids = {id(b) for b in head_bufs}
    head_out = _C.YB_CONV_E4M3_BF16_OUT if dtype == torch.bfloat16 else _C.YB_CONV_E4M3_F16_OUT     # 16-bit logits
    for i, op in enumerate(L.ops[qi:], start=qi):
        if op.kind == _C.YB_OP_QUANTIZE:
            op.bias = torch.tensor([1.0 / scale[id(op.dst.buf)]], dtype=torch.float32, device=device)
            continue
        op.dtype = _C.YB_F8E4M3
        if op.kind != _C.YB_OP_CONV:
            continue
        s_w = L.s_w.pop(i)
        co, co_pad = s_w.shape[0], op.weight.shape[0]
        head = id(op.dst.buf) in head_ids
        tail = torch.zeros((2 * co_pad + 2,), dtype=torch.float64, device=s_w.device)
        tail[:co_pad] = op.bias.to(s_w.device)        # the fp32 bias
        tail[co_pad:co_pad + co] = s_w * scale[id(op.src.buf)]
        tail[2 * co_pad] = scale[id(op.residual.buf)] if op.residual is not None else 0.0
        tail[2 * co_pad + 1] = 1.0 if head else 1.0 / scale[id(op.dst.buf)]
        op.bias = tail.to(torch.float32).to(device).contiguous()
        op.reserved = head_out if head else 0
    return L, x0, head_bufs, feats, scale


def _split_conv_norm_act(name, m: nn.Sequential):
    """(conv, norm or None, activation code) of a torchvision Conv2dNormActivation."""
    mods = list(m)
    conv = mods[0]
    if not isinstance(conv, nn.Conv2d):
        raise NotImplementedError(f"{name}: expected a Conv2dNormActivation, got {type(m).__name__}")
    bn = None
    act = _C.YB_ACT_NONE
    for sub in mods[1:]:
        if hasattr(sub, "running_var"):
            bn = sub
        else:
            act = act_code(sub)
    return conv, bn, act


def _fold_conv_norm(conv: nn.Conv2d, bn) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv (optional bias) followed by an optional (Frozen)BatchNorm2d, folded in fp64."""
    w = conv.weight.detach().double()
    b = conv.bias.detach().double() if conv.bias is not None else torch.zeros(w.shape[0], dtype=torch.float64,
                                                                                device=w.device)
    if bn is None:
        return w, b
    scale, shift = bn_scale_shift(bn)
    return w * scale.view(-1, 1, 1, 1), b * scale + shift


def lower_lite(model: nn.Module, dtype: torch.dtype, device: torch.device):
    """Walk a YOLO whose backbone is BackboneWithFPN (MobileNetV3 features + FPN, yolort/models/yolo_lite.py) and emit
    (lowering, input_buf, head_bufs, features), like lower_yolo.

      * stem: the 3x3/s2/p1 convolution is an exact 3x3/s1/p1 convolution over the space-to-depth canvas
        (stem_s2_to_s2d), run over super-pixels of 4 (stem_superpixel);
      * InvertedResidual: expand -> YB_OP_DWCONV -> YB_OP_SE (in place) -> project, the projection's residual being
        the block input when use_res_connect;
      * FPN (torchvision ops/feature_pyramid_network.py), coarsest level first: inner[i](x_i) takes `last` as its
        residual when both sit at the same stride, and YB_OP_UPSAMPLE2X(last) when `last` is twice as coarse; the
        LastLevelMaxPool level (max_pool2d(k=1, s=2)) is a ksize-1 stride-2 YB_OP_DWCONV with unit weights;
      * the 1x1 head convolutions over "0", "1", "2" and "pool"."""
    from torchvision.ops.feature_pyramid_network import LastLevelMaxPool

    L = _Lowering(dtype, device)
    bb = model.backbone
    body, fpn = bb.body, bb.fpn
    return_layers = dict(body.return_layers)
    layers = list(body.named_children())
    if len(model.head.head) != len(return_layers) + 1 or not isinstance(fpn.extra_blocks, LastLevelMaxPool):
        raise NotImplementedError("lowering covers BackboneWithFPN with LastLevelMaxPool and one head per level")

    name0, stem = layers[0]
    conv, bn, act = _split_conv_norm_act(f"body.{name0}", stem)
    if conv.kernel_size != (3, 3) or conv.stride != (2, 2) or conv.padding != (1, 1) or conv.in_channels != 3 \
            or conv.groups != 1:
        raise NotImplementedError("stem must be a 3x3/s2/p1 convolution over RGB")
    w, b = _fold_conv_norm(conv, bn)
    x0, cur = L.s2d_stem(f"body.{name0}", w, b, stem_s2_to_s2d, act, "superpixel", what="3x3/s2 as 3x3")
    taps: Dict[str, _View] = {}
    if name0 in return_layers:
        taps[return_layers[name0]] = cur
    for name, m in layers[1:]:
        if hasattr(m, "use_res_connect"):
            cur = L.inverted_residual(f"body.{name}", m, cur)
        else:
            c = _split_conv_norm_act(f"body.{name}", m)[0]
            if c.kernel_size != (1, 1) or c.stride != (1, 1):
                raise NotImplementedError(f"body.{name}: expected the closing 1x1 convolution")
            dst = _View(L.buf(f"body.{name}", cur.buf.div, c.out_channels), 0, c.out_channels)
            L.conv_norm_act(f"body.{name}", m, cur, dst)
            cur = dst
        if name in return_layers:
            taps[return_layers[name]] = cur
    xs = [taps[k] for k in sorted(taps, key=int)]

    oc = bb.out_channels
    inner, layer = fpn.inner_blocks, fpn.layer_blocks
    nl = len(xs)
    results: List[Optional[_View]] = [None] * nl
    last = _View(L.buf(f"fpn.inner{nl - 1}", xs[-1].buf.div, oc), 0, oc)
    L.conv_norm_act(f"fpn.inner_blocks.{nl - 1}", inner[nl - 1], xs[-1], last)
    results[-1] = _View(L.buf(str(nl - 1), xs[-1].buf.div, oc), 0, oc)
    L.conv_norm_act(f"fpn.layer_blocks.{nl - 1}", layer[nl - 1], last, results[-1])
    for idx in range(nl - 2, -1, -1):
        div = xs[idx].buf.div
        if last.buf.div == div:          # F.interpolate to the same size: the identity
            top_down = last
        elif last.buf.div == 2 * div:
            top_down = _View(L.buf(f"fpn.up{idx}", div, oc), 0, oc)
            L.upsample(f"fpn.interpolate{idx}", last, top_down)
        else:
            raise NotImplementedError("FPN levels must be 1x or 2x apart")
        new = _View(L.buf(f"fpn.inner{idx}", div, oc), 0, oc)
        L.conv_norm_act(f"fpn.inner_blocks.{idx}", inner[idx], xs[idx], new, residual=top_down)
        last = new
        results[idx] = _View(L.buf(str(idx), div, oc), 0, oc)
        L.conv_norm_act(f"fpn.layer_blocks.{idx}", layer[idx], last, results[idx])
    pool = _View(L.buf("pool", 2 * results[-1].buf.div, oc), 0, oc)
    ones = torch.ones((oc, 1, 1, 1), dtype=torch.float64)
    L.dwconv("fpn.extra_blocks(max_pool2d k1 s2)", ones, torch.zeros(oc, dtype=torch.float64), results[-1], pool, 1, 2,
             _C.YB_ACT_NONE)
    feats = {str(i): r for i, r in enumerate(results)}
    feats["pool"] = pool
    return L, x0, L.heads(list(feats.values()), model.head.head), feats


def lower_darknet(model: nn.Module, dtype: torch.dtype, device: torch.device, stem_variant: str = "auto"):
    """Walk a DarkNetV4 / DarkNetV6 classifier (yolort/models/darknetv4.py:33-136, darknetv6.py:31-127) and emit
    (lowering, input_buf, head_bufs, features), like lower_yolo.

      * features: the stem and stages of the detection body (_Lowering.stem / stages), ending at stride 32;
      * avgpool: YB_OP_AVGPOOL into a GLOBAL buffer (one pixel per image);
      * classifier.0 + Hardswish: a 1x1 YB_OP_CONV over the [N,1,1,C] map (M = N rows) with the Hardswish epilogue;
        Dropout is the identity in eval mode and emits nothing;
      * classifier.3: a 1x1 YB_OP_CONV whose output channels are zero-padded to a multiple of 8 (callers slice
        [:, :num_classes]).
    `features` holds the final feature map and the pooled vector, so that the sub-modules can run on their own."""
    L = _Lowering(dtype, device)
    mods = list(model.features)
    x0, cur = L.stem("features", mods[0], stem_variant)
    cur = L.stages("features", mods[1:], cur, {})
    if cur.buf.div != 32:
        raise NotImplementedError(f"the features must end at stride 32, got {cur.buf.div}")
    cls = list(model.classifier)
    if not (len(cls) == 4 and isinstance(cls[0], nn.Linear) and isinstance(cls[2], nn.Dropout)
            and isinstance(cls[3], nn.Linear)):
        raise NotImplementedError("classifier must be Linear -> activation -> Dropout -> Linear")
    fc1, fc2 = cls[0], cls[3]
    C, hid, nc = cur.C, fc1.out_features, fc2.out_features
    pooled = _View(L.buf("avgpool", GLOBAL, C), 0, C)
    L.avgpool("avgpool", cur, pooled)
    hidden = _View(L.buf("classifier.0", GLOBAL, hid), 0, hid)
    L.conv("classifier.0", fc1.weight.detach().double().view(hid, C, 1, 1), fc1.bias.detach().double(), pooled, hidden,
           1, 1, 0, act_code(cls[1]))
    ncb = _round_up(nc, 8)
    logits = L.buf("classifier.3", GLOBAL, ncb)
    L.conv("classifier.3", fc2.weight.detach().double().view(nc, hid, 1, 1), fc2.bias.detach().double(), hidden,
           _View(logits, 0, ncb), 1, 1, 0, _C.YB_ACT_NONE)
    return L, x0, [logits], {"features": cur, "avgpool": pooled}


# ---------------------------------------------------------------------------------------------------
# plan instances
# ---------------------------------------------------------------------------------------------------
class Lowered:
    """Shape-independent part of a model's plans: the op list with BN-folded, packed weights on the device.  Built
    once per Engine and shared by every PlanInstance (a plan adds only an activation arena and TMA descriptors)."""

    def __init__(self, model: nn.Module, dtype: torch.dtype, device: torch.device, stem_variant: str = "auto",
                 fp8=None):
        from .models._classifier import DarkNetClassifier
        from .models.yolo_lite import BackboneWithFPN

        self.fp8 = fp8 is not None       # fp8: a quantization.Fp8Calibration
        self.feat_scales: Dict[str, float] = {}
        if fp8 is not None:
            self.L, self.x0, self.head_bufs, self.feats, scale = lower_fp8(model, dtype, device, fp8.amax, stem_variant)
            self.feat_scales = {k: scale[id(v.buf)] for k, v in self.feats.items()}
        elif isinstance(model, DarkNetClassifier):
            self.L, self.x0, self.head_bufs, self.feats = lower_darknet(model, dtype, device, stem_variant)
        elif isinstance(model.backbone, BackboneWithFPN):
            self.L, self.x0, self.head_bufs, self.feats = lower_lite(model, dtype, device)
        else:
            self.L, self.x0, self.head_bufs, self.feats = lower_yolo(model, dtype, device, stem_variant)
        self.n_heads = len(self.head_bufs)
        self._model = model
        self.weight_bytes = sum(op.weight.numel() * op.weight.element_size() + op.bias.numel() * 4
                                for op in self.L.ops if op.weight is not None)

    def head_convs(self) -> Optional[List[nn.Conv2d]]:
        """The detection head's nn.Conv2d layers in level order when the last n_heads ops of this (non-FP8) lowering are
        exactly them (YOLO models), else None."""
        head = getattr(getattr(self._model, "head", None), "head", None)
        if self.fp8 or not isinstance(head, nn.ModuleList) or len(head) != self.n_heads:
            return None
        ops = self.L.ops[len(self.L.ops) - self.n_heads:]
        if any(op.name != f"head.head.{i}" for i, op in enumerate(ops)):
            return None
        return list(head)

    def head_dgrad_packs(self) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """Per head level, from the parameters: the transposed head weight W^T [Cin, Cout] packed for the conv kernel
        with the rounding of the forward's packed weights, and a zero bias."""
        packs = []
        for c in self.head_convs():
            w = c.weight.detach().double().view(c.out_channels, c.in_channels)
            packs.append(self.L.pack(w.t()[:, :, None, None],
                                     torch.zeros(w.shape[1], dtype=torch.float64, device=w.device)))
        return packs

    def refresh_head(self) -> None:
        """Re-pack and round the head weights and biases from the parameters INTO the tensors every plan points at:
        the plain and fused-decode launch lists, the chunked front plans, captured CUDA graphs and the feature-gradient
        packs stay valid.  The bits equal those of a fresh lowering."""
        convs = self.head_convs()
        ops = self.L.ops[len(self.L.ops) - self.n_heads:]
        for op, conv in zip(ops, convs):
            wp, bp = self.L.pack(conv.weight.detach().double(), conv.bias.detach().double())
            op.weight.copy_(wp)
            op.bias.copy_(bp)
        packs = self.__dict__.get("_head_dgrad_w")
        if packs is not None:
            for (wt, _), (new, _) in zip(packs, self.head_dgrad_packs()):
                wt.copy_(new)


def front_op_count(L: _Lowering) -> int:
    """Number of leading ops that only touch the stride-2/4/8 levels (stem .. the first tapped C3): the part of the plan
    `YOLOv5.predict` can run per image chunk while later chunks are still crossing PCIe."""
    n = 0
    for op in L.ops:
        if op.dst.buf.div > 8 or op.src.buf.div > 8 or op.kind not in (_C.YB_OP_CONV, _C.YB_OP_QUANTIZE):
            break
        n += 1
    return n


def assign_offsets(L: _Lowering, x0: _Buf, keep: List[_Buf], N: int, H: int, W: int, reuse: bool,
                   front_ops: int = 0, launches: Optional[List[Tuple[int, ...]]] = None):
    """Arena layout for one (N, H, W): byte offset per buffer and the arena size.  `launches` groups the ops that run
    as ONE kernel (chained tails): liveness is tracked per launch, since everything a fused launch touches is live at
    the same time.

    With `reuse`, a buffer occupies its bytes only from its first writer to its last reader (launch order is the op
    order and every launch waits for the previous one, programmatic dependent launch included), so the arena is the
    peak of the live set instead of the sum of all activations (yolov5x batch 64 1280x1280: 56 GB -> a few GB).
    Buffers in `keep` (head logits, the PAN results) stay live to the end."""
    if launches is None:
        launches = [(i,) for i in range(len(L.ops))]
    step_of = {i: t for t, grp in enumerate(launches) for i in grp}
    n_ops = len(launches)          # time is counted in launches
    size = {id(b): _round_up(N * b.hw(H, W)[0] * b.hw(H, W)[1] * b.C * b.esz, 1024) for b in L.bufs}
    first = {id(b): n_ops for b in L.bufs}
    last = {id(b): -1 for b in L.bufs}
    first[id(x0)] = -1
    for i, op in enumerate(L.ops):
        t = step_of[i]
        first[id(op.dst.buf)] = min(first[id(op.dst.buf)], t)
        last[id(op.dst.buf)] = max(last[id(op.dst.buf)], t)
        for v in (op.src, op.residual):
            if v is not None:
                last[id(v.buf)] = max(last[id(v.buf)], t)
                first[id(v.buf)] = min(first[id(v.buf)], t)
    for b in keep:
        last[id(b)] = n_ops
    # chunked front (PlanInstance.run_front_chunk): the first `front_ops` ops run once per image chunk, so every buffer
    # they touch must keep its bytes until the last chunk has passed through all of them
    front_steps = step_of[front_ops - 1] + 1 if front_ops else 0
    for i, op in enumerate(L.ops[:front_ops]):
        for v in (op.dst, op.src, op.residual):
            if v is not None:
                first[id(v.buf)] = -1
                last[id(v.buf)] = max(last[id(v.buf)], front_steps - 1)
    offsets: Dict[int, int] = {}
    if not reuse:
        off = 0
        for b in L.bufs:
            offsets[id(b)] = off
            off += size[id(b)]
        return offsets, off
    order = sorted(L.bufs, key=lambda b: first[id(b)])
    free: List[List[int]] = []          # [offset, bytes], sorted by offset, coalesced
    live: List[Tuple[int, _Buf]] = []   # (last use, buffer)
    top = 0
    k = 0
    for step in range(-1, n_ops):
        # allocate what is first touched at this step (inputs of the step are still live: freed after it)
        while k < len(order) and first[id(order[k])] <= step:
            b = order[k]
            k += 1
            need = size[id(b)]
            best = None
            for blk in free:
                if blk[1] >= need and (best is None or blk[1] < best[1]):
                    best = blk
            if best is not None:
                offsets[id(b)] = best[0]
                best[0] += need
                best[1] -= need
                if best[1] == 0:
                    free.remove(best)
            elif free and free[-1][0] + free[-1][1] == top:   # grow the trailing free block
                offsets[id(b)] = free[-1][0]
                top = free[-1][0] + need
                free.pop()
            else:
                offsets[id(b)] = top
                top += need
            live.append((last[id(b)], b))
        # release what this step read last
        still = []
        for lu, b in live:
            if lu <= step:
                free.append([offsets[id(b)], size[id(b)]])
            else:
                still.append((lu, b))
        live = still
        free.sort()
        merged: List[List[int]] = []
        for blk in free:
            if merged and merged[-1][0] + merged[-1][1] == blk[0]:
                merged[-1][1] += blk[1]
            else:
                merged.append(blk)
        free = merged
    return offsets, top


def encode(op: _Op, dtype: torch.dtype, N: int, H: int, W: int, ptr: Callable[[_View], int], *,
           tail: Optional[_Op] = None, decode: Optional["_C.HeadDecode"] = None,
           keep_intermediates: bool = False) -> Tuple["_C.OpDesc", Optional["_C.ConvChain"]]:
    """The yb_op_desc of `op` over N images of an H x W canvas, in compute dtype `dtype` unless the op carries its own
    element type, with `ptr(view)` the address of a view.  Returns the descriptor and, with `tail` (the 1x1 convolution
    after `op`, riding on its launch), the yb_conv_chain it points at: the caller keeps that alive as long as the
    descriptor, and likewise `decode`, the fused decode epilogue of a head convolution.  With `keep_intermediates` a
    chained op stores its output even when only the tail reads it."""
    d = _C.OpDesc()
    hi, wi = op.src.buf.hw(H, W)
    ho, wo = op.dst.buf.hw(H, W)
    k = op.pack
    if wi % k or wo % k:
        raise ValueError(f"{op.name}: width {wi} not divisible by the pixel packing {k}")
    d.kind, d.dtype = op.kind, _C.dtype_code(dtype) if op.dtype is None else op.dtype
    d.N, d.H, d.W = N, hi, wi // k
    d.Cin, d.in_cstride, d.in_ = op.src.C * k, op.src.buf.C * k, ptr(op.src)
    d.Ho, d.Wo = ho, wo // k
    d.Cout, d.out_cstride, d.out = op.dst.C * k, op.dst.buf.C * k, ptr(op.dst)
    d.ksize, d.stride, d.pad, d.act = op.ksize, op.stride, op.pad, op.act
    if op.weight is not None:
        d.weight = op.weight.data_ptr()
    if op.bias is not None:
        d.bias = op.bias.data_ptr()
    if op.kind == _C.YB_OP_CONV:
        d.Cout_pad, _, d.Cin_pad = op.weight.shape
        if op.band:
            d.Cin_pad = 64     # [Cout_pad, 3, 2 x 64] banded stem matrix: one 64-channel chunk of super-pixels
    if op.dtype == _C.YB_F8E4M3:
        d.reserved = op.reserved
    elif op.kind == _C.YB_OP_CONV:
        if op.force_im2col:
            d.reserved |= _C.YB_CONV_FORCE_IM2COL
        if op.band:
            d.reserved |= _C.YB_CONV_BAND_STEM
        if os.environ.get("YB_NO_NSPLIT", "0") == "1":      # A/B timing: keep streamed weights + tile pairs
            d.reserved |= _C.YB_CONV_NO_NSPLIT
    if op.residual is not None:
        d.residual, d.res_cstride = ptr(op.residual), op.residual.buf.C
    if decode is not None:
        d.decode = ctypes.addressof(decode)
    chain = None
    if tail is not None:
        chain = _C.ConvChain()
        chain.weight, chain.bias = tail.weight.data_ptr(), tail.bias.data_ptr()
        chain.Cout_pad, _, chain.K_pad = tail.weight.shape
        chain.Cout, chain.act = tail.dst.C, tail.act
        chain.out, chain.out_cstride = ptr(tail.dst), tail.dst.buf.C
        chain.own_C = op.chain_own
        if op.chain_extra is not None:
            extra = op.chain_extra
            chain.extra, chain.extra_C, chain.extra_cstride = ptr(extra), extra.C, extra.buf.C
        # stage-wise inspection wants every activation in memory, also the one only the tail reads
        chain.store_first = 1 if (op.chain_store or keep_intermediates) else 0
        d.chain = ctypes.addressof(chain)
    return d, chain


def _tensor_ptr(*pairs: Tuple[_Buf, torch.Tensor]) -> Callable[[_View], int]:
    """`ptr` for encode() over stand-alone buffers, each held by its own tensor: (buffer, tensor) pairs."""
    addr = {id(b): t.data_ptr() for b, t in pairs}
    return lambda v: addr[id(v.buf)] + v.ch0 * v.buf.esz


def launch_groups(L: _Lowering, N: int, H: int, W: int, fuse_chains: bool, front_ops: int,
                  keep_intermediates: bool) -> List[Tuple[int, ...]]:
    """The launch list: groups of op indices that run as one kernel.  An op marked for a chained tail (chain_own) runs
    together with the next op when the library supports the pair, unless the pair would straddle the end of the
    chunked front (`front_ops`)."""
    launches: List[Tuple[int, ...]] = []
    i = 0
    while i < len(L.ops):
        n = 2 if (fuse_chains and i + 1 < len(L.ops) and i + 1 != front_ops and
                  _chainable(L.ops[i], L.ops[i + 1], L.dtype, N, H, W, keep_intermediates)) else 1
        launches.append(tuple(range(i, i + n)))
        i += n
    return launches


def _chainable(op: _Op, tail: _Op, dtype: torch.dtype, N: int, H: int, W: int, keep_intermediates: bool) -> bool:
    if not (op.chain_own > 0 and op.kind == _C.YB_OP_CONV and op.pack == 1 and tail.kind == _C.YB_OP_CONV
            and tail.ksize == 1 and tail.stride == 1 and tail.residual is None and tail.pack == 1):
        return False
    # support depends on shapes / alignment only, hence the dummy address; `chain` keeps d.chain valid for the query
    d, chain = encode(op, dtype, N, H, W, lambda v: 4096, tail=tail, keep_intermediates=keep_intermediates)
    return _C.conv_chain_supported(d)


def _op_flops(op: _Op, N: int, H: int, W: int) -> int:
    """Algorithmic work of one op over N images of an H x W canvas (the reference's, for convolutions)."""
    ho, wo = op.dst.buf.hw(H, W)
    if op.kind in (_C.YB_OP_CONV, _C.YB_OP_DWCONV):
        return N * ho * (wo // op.pack) * op.flops_per_pixel
    if op.kind == _C.YB_OP_ATTENTION:   # Q K^T and P V: 4 L E per token
        return N * (ho * wo) * 4 * (ho * wo) * op.dst.C
    return 0


class PlanInstance:
    """Arena + native plan for one (N, H, W); weights come from the Engine's shared `Lowered`."""

    def __init__(self, low: Lowered, N: int, H: int, W: int, post: Optional[dict] = None, keep_intermediates: bool = False,
                 chunked: bool = False, fuse_chains: bool = True):
        L, x0, head_bufs, feats = low.L, low.x0, low.head_bufs, low.feats
        grain = max(b.div for b in L.bufs)          # GLOBAL buffers fit any canvas
        if H % grain or W % grain:
            raise ValueError(f"canvas {H}x{W} must be a multiple of {grain}")
        self.N, self.H, self.W = N, H, W
        self.dtype, self.device = L.dtype, L.device
        self.keep_intermediates = keep_intermediates
        fuse_chains = fuse_chains and not low.fp8      # FP8 plans run every convolution as its own launch
        # the input canvas stays live too, so that a plan can be re-run (timing loops, tests) without re-letterboxing
        keep = [x0] + list(head_bufs) + [v.buf for v in feats.values()]
        # chunked front: 4 chunks when the batch divides (>= 4 images per chunk)
        front_ops = front_op_count(L) if (chunked and N % 4 == 0 and N >= 16 and not keep_intermediates) else 0
        self.front_chunks = 4 if front_ops else 0
        launches = launch_groups(L, N, H, W, fuse_chains, front_ops, keep_intermediates)
        self.launch_ops = launches
        step_of = {j: t for t, grp in enumerate(launches) for j in grp}
        self.front_ops = step_of[front_ops - 1] + 1 if front_ops else 0     # in launches (what the run_* methods count)
        self._front_op_count = front_ops                                       # in ops of the lowering
        self._offsets, total = assign_offsets(L, x0, keep, N, H, W, reuse=not keep_intermediates, front_ops=front_ops,
                                              launches=launches)
        self.arena = torch.zeros((max(total, 1024),), dtype=torch.uint8, device=L.device)
        self.arena_bytes = total
        self.unshared_bytes = sum(_round_up(N * b.hw(H, W)[0] * b.hw(H, W)[1] * b.C * b.esz, 1024) for b in L.bufs)

        self._low = low                     # keeps the shared weights alive
        self.n_heads = low.n_heads
        encoded = [self._encode(grp, N, self._ptr) for grp in launches]
        descs = [d for d, _ in encoded]
        self._chains = [c for _, c in encoded if c is not None]    # the yb_conv_chain blocks the descriptors point at
        self.op_names = [" -> ".join(L.ops[j].name for j in grp) for grp in launches]
        self.op_flops = [sum(_op_flops(L.ops[j], N, H, W) for j in grp) for grp in launches]
        self.plan = _C.Plan(descs, L.device)
        self._descs = descs
        self._front_plans: Optional[List[_C.Plan]] = None
        # Second launch list whose head convolutions decode + threshold in their epilogue and append candidates to a
        # fixed NMS arena instead of storing logits (box_head.py:68-82 + :328-360,418 fused).
        self.fused_post = None
        self.plan_fused = None
        if post is not None and post["n_anchors"] * (post["num_classes"] + 5) <= 256:
            level_hw = [(H // b.div, W // b.div) for b in head_bufs]
            self.fused_post = _C.FusedPost(N, level_hw, post["strides"], post["anchors_px"], post["num_classes"],
                                           post["score_thresh"], post["nms_thresh"], post["detections_per_img"],
                                           post["semantics"], L.device)
            heads = L.ops[len(L.ops) - self.n_heads:]
            fused = descs[:-self.n_heads] + [encode(op, L.dtype, N, H, W, self._ptr, decode=hd)[0]
                                             for op, hd in zip(heads, self.fused_post.head_decode)]
            self.plan_fused = _C.Plan(fused, L.device)

        self.input = self._nhwc(x0)                      # [N, H/2, W/2, 16] space-to-depth canvas
        self.heads = [self._nhwc(b) for b in head_bufs]  # [N, h, w, round_up(3*(nc+5), 16)]
        self.features = {k: self._nhwc(v.buf) for k, v in feats.items()}
        # every buffer by name; with arena reuse (the default) only `input`, `heads` and `features` hold their data
        # after a full run -- ask for `keep_intermediates=True` to inspect the others
        self.buffers = {b.name: self._nhwc(b) for b in L.bufs}

    def _encode(self, grp: Tuple[int, ...], N: int, ptr: Callable[[_View], int]):
        """encode() of launch `grp`: an op, or an op and its chained tail."""
        L = self._low.L
        return encode(L.ops[grp[0]], L.dtype, N, self.H, self.W, ptr, tail=L.ops[grp[1]] if len(grp) == 2 else None,
                      keep_intermediates=self.keep_intermediates)

    def _ptr(self, v: _View, image: int = 0) -> int:
        """Address of view `v` from image `image` on (activations are NHWC, image-major)."""
        h, w = v.buf.hw(self.H, self.W)
        return self.arena.data_ptr() + self._offsets[id(v.buf)] + (image * h * w * v.buf.C + v.ch0) * v.buf.esz

    def _nhwc(self, b: _Buf) -> torch.Tensor:
        h, w = b.hw(self.H, self.W)
        n = self.N * h * w * b.C
        o = self._offsets[id(b)]
        dtype = self.dtype if b.esz == 2 else torch.float8_e4m3fn
        return self.arena[o: o + n * b.esz].view(dtype).view(self.N, h, w, b.C)

    @property
    def device_bytes(self) -> int:
        return int(self.arena.numel())

    # -- e4m3 features of an FP8 plan (the hook path: YOLO.backbone / YOLO.head) ------------------------------------
    def dequantized_feature(self, key: str, dtype: torch.dtype) -> torch.Tensor:
        """Feature map `key` of an FP8 plan as its e4m3 values times their power-of-two scale, in `dtype` (exact for
        scales of 2^-15 and up in fp16, for any scale in bf16)."""
        return (self.features[key].to(torch.float32) * self._low.feat_scales[key]).to(dtype)

    def quantize_feature(self, key: str, x_nhwc: torch.Tensor) -> None:
        """x (NHWC, the plan's compute dtype) -> e4m3 feature buffer `key`, by one YB_OP_QUANTIZE launch with the
        feature's scale: a feature from dequantized_feature comes back as the same bytes."""
        x = x_nhwc.to(self.dtype).contiguous()
        dst = self.features[key]
        N, h, w, C = dst.shape
        inv = self.__dict__.setdefault("_inv_scales", {})
        if key not in inv:
            inv[key] = torch.tensor([1.0 / self._low.feat_scales[key]], dtype=torch.float32, device=self.device)
        xb, qb = _Buf("x", 1, C), _Buf(key, 1, C, esz=1)
        # ksize and stride are not read by YB_OP_QUANTIZE
        op = _Op(kind=_C.YB_OP_QUANTIZE, src=_View(xb, 0, C), dst=_View(qb, 0, C), ksize=0, stride=0, bias=inv[key],
                 name=f"{key}(quantize)")
        d, _ = encode(op, self.dtype, N, h, w, _tensor_ptr((xb, x), (qb, dst)))
        _C.Plan([d], self.device).run()

    def run(self, first: int = 0, count: Optional[int] = None) -> None:
        """Backbone + PAN + heads, logits stored in `self.heads`."""
        if first == 0 and count is None and self.use_graph:
            return self.run_graph()
        self.plan.run(first, count)

    # -- CUDA graph of the launch list ---------------------------------------------------------------------------
    use_graph = False      # opt-in per instance (Engine.graphs): the launch list is static, so it can be replayed as one graph

    def run_graph(self) -> None:
        """Replays the whole plan as ONE CUDA graph launch (captured on first use from the same launch list, programmatic
        dependent-launch edges included).  The ~55 cudaLaunchKernelEx calls of a yolov5s plan cost the host ~0.15 ms; at
        batch 32 the GPU needs 1.6 ms for them, so this matters for small batches / latency, not for throughput."""
        g = self.__dict__.get("_graph")
        if g is None:
            with _C.device_guard(self.device):
                self.plan.run()                      # eager once: lazy module loading must not happen under capture
                torch.cuda.synchronize(self.device)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.plan.run()
            self.__dict__["_graph"] = g
        g.replay()

    # -- chunked front ----------------------------------------------------------------------------------------------
    def _build_front_plans(self) -> None:
        """Launch lists of ops [0, front_ops) restricted to the images of one chunk: N = chunk and every view starting
        at the chunk's first image."""
        c = self.N // self.front_chunks
        plans = []
        for k in range(self.front_chunks):
            encoded = [self._encode(grp, c, lambda v: self._ptr(v, k * c)) for grp in self.launch_ops[: self.front_ops]]
            plans.append(_C.Plan([d for d, _ in encoded], self.device))   # the native plan copies what it needs here
        self._front_plans = plans

    def run_front_chunk(self, k: int) -> None:
        """Ops [0, front_ops) over the images of chunk k only (their slice of `self.input` must be written)."""
        if self._front_plans is None:
            with _C.device_guard(self.device):
                self._build_front_plans()
        self._front_plans[k].run()

    def run_rest(self) -> None:
        """Ops [front_ops, end) over the whole batch, after every chunk went through `run_front_chunk`."""
        self.plan.run(self.front_ops, self.plan.n_ops - self.front_ops)

    def run_backbone(self) -> None:
        """Everything but the detection-head convolutions (`YOLO.backbone`)."""
        self.plan.run(0, self.plan.n_ops - self.n_heads)

    def run_heads(self) -> None:
        """The detection-head 1x1 convolutions over `self.features` (`YOLO.head`)."""
        self.plan.run(self.plan.n_ops - self.n_heads, self.n_heads)

    def run_fused(self) -> None:
        """Backbone + PAN + heads with the decode epilogue (candidates land in `self.fused_post`'s arena)."""
        self.plan_fused.run()


class _HeadDgrad:
    """Feature gradient of head level `lvl` for one (N, h, w): dX = dY . W as a one-op plan (1x1 convolution, K = C_pad,
    no activation) on the conv kernel over the transposed, zero-padded head weight.  `dy` is the plan's input
    [N, h, w, C_pad] (the caller fills it, pad channels zero); run() returns a fresh [N, h, w, Cin] gradient."""

    def __init__(self, low: "Lowered", lvl: int, N: int, h: int, w: int, cin: int):
        L = low.L
        wt, bias = head_dgrad_weights(low)[lvl]
        cpad = low.head_bufs[lvl].C
        self.dy = torch.zeros((N, h, w, cpad), dtype=L.dtype, device=L.device)
        self.dx = torch.empty((N, h, w, cin), dtype=L.dtype, device=L.device)
        dy, dx = _Buf("dy", 1, cpad), _Buf("dx", 1, cin)
        op = _Op(kind=_C.YB_OP_CONV, src=_View(dy, 0, cpad), dst=_View(dx, 0, cin), weight=wt, bias=bias,
                 name=f"head.head.{lvl}(dgrad)")
        d, _ = encode(op, L.dtype, N, h, w, _tensor_ptr((dy, self.dy), (dx, self.dx)))
        self.plan = _C.Plan([d], L.device)
        self._keep = (wt, bias)

    def run(self) -> torch.Tensor:
        self.plan.run()
        return self.dx.clone()


def head_dgrad_weights(low: "Lowered") -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """Per head level: the transposed head weight W^T [Cin, Cout] packed for the conv kernel, and a zero bias.  Built
    once per lowering from the fp64 parameters, with the rounding of the forward's packed weights; refreshed in place
    with them (Engine._refresh_head)."""
    packs = low.__dict__.get("_head_dgrad_w")
    if packs is None:
        packs = low.__dict__["_head_dgrad_w"] = low.head_dgrad_packs()
    return packs


def head_dgrad(low: "Lowered", lvl: int, N: int, h: int, w: int, cin: int) -> _HeadDgrad:
    """The cached _HeadDgrad of (level, N, h, w) on this lowering."""
    cache = low.__dict__.setdefault("_head_dgrad", {})
    key = (lvl, N, h, w)
    inst = cache.get(key)
    if inst is None:
        with _C.device_guard(low.L.device):
            inst = cache[key] = _HeadDgrad(low, lvl, N, h, w, cin)
    return inst


class Engine:
    """Per-model state of the native path: the weights lowered ONCE (BN folded, packed, on the device) and an LRU
    cache of plan instances keyed by (N, H, W).  A new shape costs an arena allocation plus descriptor encoding
    (milliseconds), never a re-lowering; the cache is bounded by a plan count and a byte budget so that a serving
    process with dynamic canvases does not accumulate arenas without limit."""

    MAX_PLANS = 32

    def __init__(self, model: nn.Module, dtype: torch.dtype, device: torch.device, max_arena_bytes: Optional[int] = None):
        if device.type != "cuda":
            raise _C.NativeLibraryError(
                f"yolort_b200 runs on sm_90a GPUs only; model parameters are on {device} (no CPU fallback)")
        if dtype not in (torch.float16, torch.bfloat16):
            raise _C.NativeLibraryError(f"compute dtype must be float16 or bfloat16, got {dtype}")
        _C.lib()
        self.model, self.dtype, self.device = model, dtype, device
        import collections
        self._plans: "collections.OrderedDict[tuple, PlanInstance]" = collections.OrderedDict()
        self._low: Optional[Lowered] = None
        self._low8: Optional[Lowered] = None      # the FP8 lowering of `fp8`
        self.fp8 = None          # quantization.Fp8Calibration: plans run in FP8 (YOLO.set_fp8); None: in `dtype`
        self._tensors: List[torch.Tensor] = []
        self._versions: Tuple[int, ...] = ()
        self.max_arena_bytes = max_arena_bytes
        self.lowerings = 0       # how many times the weights were folded/packed (tests: stays 1 across shapes)
        self.head_refreshes = 0  # in-place refreshes of the head weights after head-only parameter edits
        self.stem_variant = "auto"
        self.graphs = False      # replay plans as CUDA graphs (PlanInstance.run_graph)
        # chained pointwise tails (yb_conv_chain); YB_NO_CHAIN=1 keeps every convolution its own launch (A/B timing)
        self.fuse_chains = os.environ.get("YB_NO_CHAIN", "0") != "1"

    # -- weights -------------------------------------------------------------------------------------------------
    def _fingerprint(self) -> Tuple[int, ...]:
        return tuple(t._version for t in self._tensors)

    def lowered(self, fp8: Optional[bool] = None) -> Lowered:
        """The shared lowering; rebuilt (and every plan dropped) when a parameter or BN statistic was modified in
        place since the last lowering (`_version` counters; `.to()` / `load_state_dict` go through YOLO's hooks).
        `fp8`: the FP8 (True) or the `dtype` (False) lowering; default: the one `self.fp8` selects."""
        if (self._low is not None or self._low8 is not None) and self._fingerprint() != self._versions:
            if not self._refresh_head():
                self.invalidate()
        use_fp8 = self.fp8 is not None if fp8 is None else fp8
        if use_fp8 and self.fp8 is None:
            raise ValueError("an FP8 lowering needs a calibration (set_fp8)")
        attr = "_low8" if use_fp8 else "_low"
        low = getattr(self, attr)
        if low is None:
            with _C.device_guard(self.device):
                if self._low is None and self._low8 is None:
                    self._tensors = [t for t in list(self.model.parameters()) + list(self.model.buffers())]
                    self._versions = self._fingerprint()
                low = Lowered(self.model, self.dtype, self.device, self.stem_variant, fp8=self.fp8 if use_fp8 else None)
            setattr(self, attr, low)
            self.lowerings += 1
        return low

    def _refresh_head(self) -> bool:
        """Head fine-tuning: after in-place edits of the head parameters only (an optimizer step) on a model whose
        other parameters are all frozen (requires_grad False), refresh the packed head weights in place instead of
        re-lowering; True when that was done.  Any other change, any change while a backbone or neck parameter still
        requires grad, and any change while an FP8 lowering exists take the full invalidation."""
        if self._low is None or self._low8 is not None or self.fp8 is not None:
            return False
        convs = self._low.head_convs()
        if convs is None:
            return False
        head_ids = {id(t) for c in convs for t in (c.weight, c.bias)}
        if any(p.requires_grad for p in self.model.parameters() if id(p) not in head_ids):
            return False
        cur = self._fingerprint()
        if any(a != b and id(t) not in head_ids for t, a, b in zip(self._tensors, cur, self._versions)):
            return False
        with _C.device_guard(self.device):
            self._low.refresh_head()
        self._versions = cur
        self.head_refreshes += 1
        return True

    def invalidate(self) -> None:
        self._plans.clear()
        self._low = None
        self._low8 = None

    def drop_plans(self) -> None:
        """Forget the plan instances (their fused head epilogues bake the post-processing constants) and keep the
        lowered weights."""
        self._plans.clear()

    def set_fp8(self, calib) -> None:
        """Run plans in FP8 with the scales of `calib` (None: in `dtype`).  FP8 plans are cached apart from the others,
        so switching back finds the `dtype` plans as they were."""
        if calib is not self.fp8:
            self.fp8 = calib
            self._low8 = None
            for key in [k for k in self._plans if k[-1]]:
                del self._plans[key]

    # -- plans ---------------------------------------------------------------------------------------------------
    def _budget(self) -> int:
        if self.max_arena_bytes is not None:
            return self.max_arena_bytes
        try:
            return int(0.6 * torch.cuda.get_device_properties(self.device).total_memory)
        except Exception:
            return 64 << 30

    def plan(self, N: int, H: int, W: int, post: Optional[dict] = None, keep_intermediates: bool = False,
             chunked: bool = False, slot: int = 0) -> PlanInstance:
        """`chunked`: a plan whose first ops can also run per image chunk (PlanInstance.run_front_chunk; the arena keeps
        the front buffers live, so it is a separate instance from the plain plan of the same shape).  `slot` > 0: another
        instance of the same shape with its own arena (test-time augmentation runs passes of equal canvas shape, each of
        which must keep its head logits until the joint decode)."""
        check_fp8 = getattr(self.model, "_check_fp8", None)     # YOLO: a stale FP8 calibration raises
        if check_fp8 is not None:
            check_fp8()
        low = self.lowered()
        pkey = None if post is None else (post["score_thresh"], post["nms_thresh"], post["detections_per_img"],
                                          post["semantics"], post["num_classes"])
        chunked = bool(chunked and N % 4 == 0 and N >= 16 and not keep_intermediates)
        key = (N, H, W, pkey, bool(keep_intermediates), chunked, bool(self.fuse_chains), int(slot), self.fp8 is not None)
        inst = self._plans.get(key)
        if inst is not None:
            self._plans.move_to_end(key)
            return inst
        with _C.device_guard(self.device):
            inst = PlanInstance(low, N, H, W, post, keep_intermediates, chunked, self.fuse_chains)
        inst.use_graph = bool(self.graphs)
        self._plans[key] = inst
        budget = self._budget()
        while len(self._plans) > 1 and (len(self._plans) > self.MAX_PLANS or
                                        sum(p.device_bytes for p in self._plans.values()) > budget):
            self._plans.popitem(last=False)      # least recently used
        return inst
