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
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _C
from .models.common import C3, BottleneckCSP, Conv, Focus, SPP


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


@dataclass
class _Buf:
    name: str
    div: int          # spatial divisor w.r.t. the canvas
    C: int            # total channels (pixel stride)
    offset: int = 0   # byte offset in the arena


@dataclass
class _View:
    buf: _Buf
    ch0: int
    C: int


@dataclass
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
        wp, _, co_pad = pack_weight(w, self.dtype, self.device)
        bp = pack_bias(b, co_pad, self.device)
        if ref_flops_per_pixel is None:
            ref_flops_per_pixel = 2 * w.shape[0] * w.shape[1] * k * k
        self.ops.append(_Op(_C.YB_OP_CONV, src, dst, k, s, p, act, wp, bp, residual, name, ref_flops_per_pixel, pack, force_im2col))

    def conv_band(self, name, w_band, b, src: _View, dst: _View, act, ref_flops_per_pixel):
        """Stem on the banded super-pixel weights (stem_band): pack 4, 3x3/s1/p1, handled by the patch kernel's
        kBand variant."""
        co4 = w_band.shape[0]
        assert src.C == 16 and src.ch0 == 0 and src.C == src.buf.C and dst.ch0 == 0 and dst.C == dst.buf.C and 4 * dst.C == co4
        assert co4 % 64 == 0 and co4 <= 256, "banded stem needs 64 | 4*Cout <= 256"
        wp = w_band.to(self.dtype).to(self.device).contiguous()
        bp = pack_bias(b, co4, self.device)
        self.ops.append(_Op(_C.YB_OP_CONV, src, dst, 3, 1, 1, act, wp, bp, None, name, ref_flops_per_pixel, 4, False, True))

    def conv_module(self, name, m: Conv, src: _View, dst: _View, residual=None):
        w, b = fold_conv_bn(m)
        k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
        self.conv(name, w, b, src, dst, k, s, p, act_code(m.act), residual)

    def block(self, name, m, src: _View, dst: _View):
        """C3 (r4.0 / r6.0 graphs) or BottleneckCSP (r3.1)."""
        if isinstance(m, C3):
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

    def spp(self, name, m: SPP, src: _View, dst: _View):
        if tuple(m.k) != (5, 9, 13):
            raise NotImplementedError("SPP pooling kernel implements k=(5,9,13) (the r6.0 neck)")
        div = src.buf.div
        c_ = m.cv1.conv.out_channels
        cat = self.buf(f"{name}.cat", div, 4 * c_)
        self.conv_module(f"{name}.cv1", m.cv1, src, _View(cat, 0, c_))
        self.ops.append(_Op(_C.YB_OP_SPP_POOL, _View(cat, 0, c_), _View(cat, c_, 3 * c_), name=f"{name}.pool"))
        self.conv_module(f"{name}.cv2", m.cv2, _View(cat, 0, 4 * c_), dst)

    def upsample(self, name, src: _View, dst: _View):
        self.ops.append(_Op(_C.YB_OP_UPSAMPLE2X, src, dst, name=name))


def lower_yolo(model: nn.Module, dtype: torch.dtype, device: torch.device, stem_variant: str = "auto"):
    """Walk YOLO.backbone / YOLO.head and emit (lowering, input_buf, head_bufs, features).
    `stem_variant`: "auto" | "band" | "superpixel" | "im2col" (the last two are kept for parity tests and A/B timing)."""
    L = _Lowering(dtype, device)
    bb = model.backbone
    body, pan = bb.body, bb.pan
    ch = list(bb.out_channels)
    nl = len(ch)                                   # detection levels: 3, or 4 with the P6 intermediate block
    has_p6 = getattr(pan, "intermediate_blocks", None) is not None
    if nl not in (3, 4) or len(model.head.head) != nl or has_p6 != (nl == 4):
        raise NotImplementedError("lowering covers the r6.0 topologies: 3 levels, or 4 levels with the P6 block")

    x0 = L.buf("input.s2d", 2, 16)
    stem = body["0"]
    if isinstance(stem, Focus):       # r3.1 / r4.0: Focus = 2x2 space-to-depth + 3x3/s1/p1 conv (darknetv4.py:82)
        stem = stem.conv
        if stem.conv.kernel_size != (3, 3) or stem.conv.stride != (1, 1) or stem.conv.padding != (1, 1):
            raise NotImplementedError("Focus stem must be the 3x3/s1/p1 convolution")
        w, b = fold_conv_bn(stem)
        w_s2d = focus_to_s2d(w)
    else:                             # r6.0: 6x6/s2/p2 conv == 3x3/s1/p1 over the same space-to-depth input
        if stem.conv.kernel_size != (6, 6) or stem.conv.stride != (2, 2) or stem.conv.padding != (2, 2):
            raise NotImplementedError("stem must be the r6.0 6x6/s2/p2 convolution")
        w, b = fold_conv_bn(stem)
        w_s2d = stem_to_s2d(w)
    t0 = L.buf("body.0", 2, w.shape[0])
    # The stem runs over "super-pixels" of 4 horizontally adjacent s2d pixels (128-byte TMA rows instead of 32).  Its
    # expanded weight matrix is block-banded, and when the band (6 slabs of 4*Cout x 64) fits in shared memory next to
    # two patches (4*Cout <= 128: yolov5n / s) the banded kernel variant multiplies only the band; wider stems
    # (m / l / x) use the dense super-pixel form.
    spk = 4
    co4 = spk * w.shape[0]
    if stem_variant == "band" or (stem_variant == "auto" and co4 % 64 == 0 and co4 <= 128
                                  and act_code(stem.act) in (_C.YB_ACT_SILU, _C.YB_ACT_NONE)):
        w_b, b_b = stem_band(w_s2d, b)
        L.conv_band("body.0(stem: banded 3x3 over s2d super-pixels)", w_b, b_b, _View(x0, 0, 16), _View(t0, 0, w.shape[0]),
                    act_code(stem.act), ref_flops_per_pixel=spk * 2 * w.shape[0] * 3 * 36)
    else:
        w_sp, b_sp = stem_superpixel(w_s2d, b, spk)
        L.conv("body.0(stem: 3x3 over s2d super-pixels)", w_sp, b_sp, _View(x0, 0, 16), _View(t0, 0, w.shape[0]), 3, 1, 1,
               act_code(stem.act), ref_flops_per_pixel=spk * 2 * w.shape[0] * 3 * 36, pack=spk,
               force_im2col=(stem_variant == "im2col"))

    # Concat buffers of the neck (path_aggregation_network.py:215-237), level l at stride 8 << l:
    #   cat_dn[l] = [up(lateral from level l+1) | body tap of level l]   (descending pass, l < nl-1)
    #   cat_up[l] = [down(result of level l-1) | lateral of level l]     (ascending pass,  l > 0)
    # lateral k (k = 1..nl-1) is the 1x1 conv output at level nl-k; producers write straight into these windows.
    taps = (4, 6, 8)
    cat_dn = {l: L.buf(f"pan.cat{nl - 1 - l}[up(lat{nl - 1 - l})|f{taps[l]}]", 8 << l, 2 * ch[l]) for l in range(nl - 1)}
    cat_up = {l: L.buf(f"pan.cat_p{l + 3}[down(p{l + 2})|lat{nl - l}]", 8 << l, 2 * ch[l - 1]) for l in range(1, nl)}

    cur = _View(t0, 0, w.shape[0])
    div = 2
    tap_dst = {taps[l]: _View(cat_dn[l], ch[l], ch[l]) for l in range(min(nl - 1, 3))}
    for i in range(1, 9):
        m = body[str(i)]
        if isinstance(m, Conv):
            div *= 2
            co = m.conv.out_channels
            t = L.buf(f"body.{i}", div, co)
            L.conv_module(f"body.{i}", m, cur, _View(t, 0, co))
            cur = _View(t, 0, co)
        elif isinstance(m, SPP):      # r3.1 / r4.0 keep the SPP as the last body module (darknetv4.py:97)
            co = m.cv2.conv.out_channels
            dst = _View(L.buf(f"body.{i}", div, co), 0, co)
            L.spp(f"body.{i}", m, cur, dst)
            cur = dst
        else:
            co = (m.cv3 if isinstance(m, C3) else m.cv4).conv.out_channels
            dst = tap_dst.get(i) or _View(L.buf(f"body.{i}", div, co), 0, co)
            assert dst.C == co
            L.block(f"body.{i}", m, cur, dst)
            cur = dst
    top = cur
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

    head_bufs = []
    for i, (feat, conv) in enumerate(zip(results, model.head.head)):
        co = conv.out_channels
        co_buf = _round_up(co, 16)
        hb = L.buf(f"head.{i}", feat.buf.div, co_buf)
        L.conv(f"head.head.{i}", conv.weight.detach().double(), conv.bias.detach().double(), feat,
               _View(hb, 0, co_buf), 1, 1, 0, _C.YB_ACT_NONE)
        head_bufs.append(hb)
    return L, x0, head_bufs, {f"p{l + 3}": r for l, r in enumerate(results)}


# ---------------------------------------------------------------------------------------------------
# plan instances
# ---------------------------------------------------------------------------------------------------
class Lowered:
    """Shape-independent part of a model's plans: the op list with BN-folded, packed weights on the device.  Built
    once per Engine and shared by every PlanInstance (a plan adds only an activation arena and TMA descriptors)."""

    def __init__(self, model: nn.Module, dtype: torch.dtype, device: torch.device, stem_variant: str = "auto"):
        self.L, self.x0, self.head_bufs, self.feats = lower_yolo(model, dtype, device, stem_variant)
        self.n_heads = len(self.head_bufs)
        self.weight_bytes = sum(op.weight.numel() * op.weight.element_size() + op.bias.numel() * 4
                                for op in self.L.ops if op.weight is not None)


def front_op_count(L: _Lowering) -> int:
    """Number of leading ops that only touch the stride-2/4/8 levels (stem .. the first tapped C3): the part of the plan
    `YOLOv5.predict` can run per image chunk while later chunks are still crossing PCIe."""
    n = 0
    for op in L.ops:
        if op.dst.buf.div > 8 or op.src.buf.div > 8 or op.kind != _C.YB_OP_CONV:
            break
        n += 1
    return n


def assign_offsets(L: _Lowering, x0: _Buf, keep: List[_Buf], N: int, H: int, W: int, reuse: bool, esz: int = 2,
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
    size = {id(b): _round_up(N * (H // b.div) * (W // b.div) * b.C * esz, 1024) for b in L.bufs}
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


class PlanInstance:
    """Arena + native plan for one (N, H, W); weights come from the Engine's shared `Lowered`."""

    def __init__(self, low: Lowered, N: int, H: int, W: int, post: Optional[dict] = None, keep_intermediates: bool = False,
                 chunked: bool = False, fuse_chains: bool = True):
        L, x0, head_bufs, feats = low.L, low.x0, low.head_bufs, low.feats
        grain = max(b.div for b in L.bufs)
        if H % grain or W % grain:
            raise ValueError(f"canvas {H}x{W} must be a multiple of {grain}")
        self.N, self.H, self.W = N, H, W
        self.dtype, self.device = L.dtype, L.device
        self.keep_intermediates = keep_intermediates
        esz = 2
        # the input canvas stays live too, so that a plan can be re-run (timing loops, tests) without re-letterboxing
        keep = [x0] + list(head_bufs) + [v.buf for v in feats.values()]
        # chunked front: 4 chunks when the batch divides (>= 4 images per chunk)
        front_ops = front_op_count(L) if (chunked and N % 4 == 0 and N >= 16 and not keep_intermediates) else 0
        self.front_chunks = 4 if front_ops else 0
        code = _C.dtype_code(L.dtype)
        self._chains: List[_C.ConvChain] = []    # yb_conv_chain blocks the descriptors point at (kept alive)
        no_nsplit = os.environ.get("YB_NO_NSPLIT", "0") == "1"    # A/B timing: keep streamed weights + tile pairs

        def make_desc(op: _Op, ptr) -> "_C.OpDesc":
            d = _C.OpDesc()
            hi, wi = H // op.src.buf.div, W // op.src.buf.div
            ho, wo = H // op.dst.buf.div, W // op.dst.buf.div
            d.kind, d.dtype = op.kind, code
            k = op.pack
            if wi % k or wo % k:
                raise ValueError(f"{op.name}: width {wi} not divisible by the pixel packing {k}")
            wi, wo = wi // k, wo // k
            d.N, d.H, d.W = N, hi, wi
            d.Cin, d.in_cstride, d.in_ = op.src.C * k, op.src.buf.C * k, ptr(op.src)
            d.Ho, d.Wo = ho, wo
            d.Cout, d.out_cstride, d.out = op.dst.C * k, op.dst.buf.C * k, ptr(op.dst)
            d.ksize, d.stride, d.pad, d.act = op.ksize, op.stride, op.pad, op.act
            if op.kind == _C.YB_OP_CONV:
                d.weight, d.bias = op.weight.data_ptr(), op.bias.data_ptr()
                d.Cout_pad, _, d.Cin_pad = op.weight.shape
                if op.band:
                    d.Cin_pad = 64     # [Cout_pad, 3, 2 x 64] banded stem matrix: one 64-channel chunk of super-pixels
            d.reserved = (1 if op.force_im2col else 0) | (2 if op.band else 0) | (8 if no_nsplit else 0)
            if op.residual is not None:
                d.residual, d.res_cstride = ptr(op.residual), op.residual.buf.C
            return d

        def make_chain(op: _Op, tail: _Op, ptr) -> "_C.ConvChain":
            """yb_conv_chain for `tail` (the 1x1 convolution after `op`) riding on `op`'s launch."""
            c = _C.ConvChain()
            c.weight, c.bias = tail.weight.data_ptr(), tail.bias.data_ptr()
            c.Cout_pad, _, c.K_pad = tail.weight.shape
            c.Cout, c.act = tail.dst.C, tail.act
            c.out, c.out_cstride = ptr(tail.dst), tail.dst.buf.C
            c.own_C = op.chain_own
            if op.chain_extra is not None:
                c.extra, c.extra_C, c.extra_cstride = ptr(op.chain_extra), op.chain_extra.C, op.chain_extra.buf.C
            # stage-wise inspection wants every activation in memory, also the one only the tail reads
            c.store_first = 1 if (op.chain_store or keep_intermediates) else 0
            return c

        def chainable(i: int) -> bool:
            op = L.ops[i]
            if not (fuse_chains and op.chain_own > 0 and i + 1 < len(L.ops) and i + 1 != front_ops):
                return False
            tail = L.ops[i + 1]
            if not (tail.kind == _C.YB_OP_CONV and tail.ksize == 1 and tail.stride == 1 and tail.residual is None
                    and tail.pack == 1 and op.pack == 1 and op.kind == _C.YB_OP_CONV):
                return False
            d = make_desc(op, lambda v: 4096)           # support depends on shapes / alignment only
            c = make_chain(op, tail, lambda v: 4096)
            d.chain = ctypes.addressof(c)
            return _C.conv_chain_supported(d)

        # launch list: groups of op indices that run as one kernel
        launches: List[Tuple[int, ...]] = []
        i = 0
        while i < len(L.ops):
            if chainable(i):
                launches.append((i, i + 1))
                i += 2
            else:
                launches.append((i,))
                i += 1
        self.launch_ops = launches
        step_of = {j: t for t, grp in enumerate(launches) for j in grp}
        self.front_ops = step_of[front_ops - 1] + 1 if front_ops else 0     # in launches (what the run_* methods count)
        self._front_op_count = front_ops                                       # in ops of the lowering
        offsets, total = assign_offsets(L, x0, keep, N, H, W, reuse=not keep_intermediates, esz=esz,
                                        front_ops=front_ops, launches=launches)
        self.arena = torch.zeros((max(total, 1024),), dtype=torch.uint8, device=L.device)
        self.arena_bytes = total
        self.unshared_bytes = sum(_round_up(N * (H // b.div) * (W // b.div) * b.C * esz, 1024) for b in L.bufs)
        base = self.arena.data_ptr()

        def ptr(v: _View) -> int:
            return base + offsets[id(v.buf)] + v.ch0 * esz

        descs = []
        self.op_names = []
        self.op_flops = []
        for grp in launches:
            op = L.ops[grp[0]]
            d = make_desc(op, ptr)
            name = op.name
            flops = N * (H // op.dst.buf.div) * (W // op.dst.buf.div // op.pack) * op.flops_per_pixel if op.kind == _C.YB_OP_CONV else 0
            if len(grp) == 2:
                tail = L.ops[grp[1]]
                c = make_chain(op, tail, ptr)
                self._chains.append(c)
                d.chain = ctypes.addressof(c)
                name = f"{op.name} -> {tail.name}"
                flops += N * (H // tail.dst.buf.div) * (W // tail.dst.buf.div) * tail.flops_per_pixel
            descs.append(d)
            self.op_names.append(name)
            self.op_flops.append(flops)
        self._low = low                     # keeps the shared weights alive
        self.n_heads = low.n_heads
        self.plan = _C.Plan(descs, L.device)
        self._descs = descs
        self._front_plans: Optional[List[_C.Plan]] = None
        # Second launch list whose head convolutions decode + threshold in their epilogue and append candidates to a
        # fixed NMS arena instead of storing logits (box_head.py:68-82 + :328-360,418 fused).
        self.fused_post = None
        self.plan_fused = None
        n_heads = len(head_bufs)
        if post is not None and post["n_anchors"] * (post["num_classes"] + 5) <= 256:
            level_hw = [(H // b.div, W // b.div) for b in head_bufs]
            self.fused_post = _C.FusedPost(N, level_hw, post["strides"], post["anchors_px"], post["num_classes"],
                                           post["score_thresh"], post["nms_thresh"], post["detections_per_img"],
                                           post["semantics"], L.device)
            fused = list(descs[:-n_heads])
            import ctypes as _ct
            for d, hd in zip(descs[-n_heads:], self.fused_post.head_decode):
                d2 = _C.OpDesc.from_buffer_copy(d)
                d2.decode = _ct.addressof(hd)
                fused.append(d2)
            self.plan_fused = _C.Plan(fused, L.device)

        def nhwc(b: _Buf) -> torch.Tensor:
            h, w = H // b.div, W // b.div
            n = N * h * w * b.C
            o = offsets[id(b)]
            return self.arena[o: o + n * esz].view(L.dtype).view(N, h, w, b.C)

        self.input = nhwc(x0)                      # [N, H/2, W/2, 16] space-to-depth canvas
        self.heads = [nhwc(b) for b in head_bufs]  # [N, h, w, round_up(3*(nc+5), 16)]
        self.features = {k: nhwc(v.buf) for k, v in feats.items()}
        # every buffer by name; with arena reuse (the default) only `input`, `heads` and `features` hold their data
        # after a full run -- ask for `keep_intermediates=True` to inspect the others
        self.buffers = {b.name: nhwc(b) for b in L.bufs}

    @property
    def device_bytes(self) -> int:
        return int(self.arena.numel())

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
        """Launch lists of ops [0, front_ops) restricted to the images of one chunk: same descriptors, N = chunk and
        every tensor pointer advanced by the chunk's images (activations are NHWC, image-major)."""
        L = self._low.L
        c = self.N // self.front_chunks
        esz = 2
        plans = []
        for k in range(self.front_chunks):
            ds = []
            chains = []
            for grp, d in zip(self.launch_ops[: self.front_ops], self._descs[: self.front_ops]):
                op = L.ops[grp[0]]
                d2 = _C.OpDesc.from_buffer_copy(d)
                d2.N = c

                def adv(view):
                    return k * c * (self.H // view.buf.div) * (self.W // view.buf.div) * view.buf.C * esz

                d2.in_ = d.in_ + adv(op.src)
                d2.out = d.out + adv(op.dst)
                if op.residual is not None:
                    d2.residual = d.residual + adv(op.residual)
                if len(grp) == 2:      # chained tail: its own block of pointers
                    tail = L.ops[grp[1]]
                    c2 = _C.ConvChain.from_buffer_copy(_C.ConvChain.from_address(d.chain))
                    c2.out = c2.out + adv(tail.dst)
                    if op.chain_extra is not None:
                        c2.extra = c2.extra + adv(op.chain_extra)
                    chains.append(c2)
                    d2.chain = ctypes.addressof(c2)
                ds.append(d2)
            plans.append(_C.Plan(ds, self.device))      # the native plan copies what it needs at creation
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
        self._tensors: List[torch.Tensor] = []
        self._versions: Tuple[int, ...] = ()
        self.max_arena_bytes = max_arena_bytes
        self.lowerings = 0       # how many times the weights were folded/packed (tests: stays 1 across shapes)
        self.stem_variant = "auto"
        self.graphs = False      # replay plans as CUDA graphs (PlanInstance.run_graph)
        # chained pointwise tails (yb_conv_chain); YB_NO_CHAIN=1 keeps every convolution its own launch (A/B timing)
        self.fuse_chains = os.environ.get("YB_NO_CHAIN", "0") != "1"

    # -- weights -------------------------------------------------------------------------------------------------
    def _fingerprint(self) -> Tuple[int, ...]:
        return tuple(t._version for t in self._tensors)

    def lowered(self) -> Lowered:
        """The shared lowering; rebuilt (and every plan dropped) when a parameter or BN statistic was modified in
        place since the last lowering (`_version` counters; `.to()` / `load_state_dict` go through YOLO's hooks)."""
        if self._low is not None and self._fingerprint() != self._versions:
            self.invalidate()
        if self._low is None:
            with _C.device_guard(self.device):
                self._tensors = [t for t in list(self.model.parameters()) + list(self.model.buffers())]
                self._versions = self._fingerprint()
                self._low = Lowered(self.model, self.dtype, self.device, self.stem_variant)
            self.lowerings += 1
        return self._low

    def invalidate(self) -> None:
        self._plans.clear()
        self._low = None

    # -- plans ---------------------------------------------------------------------------------------------------
    def _budget(self) -> int:
        if self.max_arena_bytes is not None:
            return self.max_arena_bytes
        try:
            return int(0.6 * torch.cuda.get_device_properties(self.device).total_memory)
        except Exception:
            return 64 << 30

    def plan(self, N: int, H: int, W: int, post: Optional[dict] = None, keep_intermediates: bool = False,
             chunked: bool = False) -> PlanInstance:
        """`chunked`: a plan whose first ops can also run per image chunk (PlanInstance.run_front_chunk; the arena keeps
        the front buffers live, so it is a separate instance from the plain plan of the same shape)."""
        low = self.lowered()
        pkey = None if post is None else (post["score_thresh"], post["nms_thresh"], post["detections_per_img"],
                                          post["semantics"], post["num_classes"])
        chunked = bool(chunked and N % 4 == 0 and N >= 16 and not keep_intermediates)
        key = (N, H, W, pkey, bool(keep_intermediates), chunked, bool(self.fuse_chains))
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
