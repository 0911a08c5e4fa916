"""Stage-wise parity at REAL shapes: every launch of a plan against a plain fp32 PyTorch op applied to the launch's
OWN input buffer -- "each conv block vs fp32 on the same rounded inputs/weights: |err| <= 2^-9 (fp16) / 2^-6 (bf16) x
(1 + |ref|)" (SURVEY.md 8c.1).  The fp32 reference runs on the GPU with TF32 disabled.

One reference per (op kind, element type) in REFERENCES, each returning (reference, bound); the stem is checked against
its own module (stem_reference), not against the space-to-depth rewrite the plan runs.  Bounds:

* fp16 / bf16 outputs: TOL x (1 + |ref|); the attention's scale is 1 + A(|V|) instead (its outputs are sums of values
  of both signs and can cancel), the global average pool's one ulp of the fp64 mean;
* e4m3 outputs of an FP8 plan: QUANTIZE, SPP and upsample exactly; a convolution within one e4m3 ulp of v / s_out
  (floor 2^-9, the subnormal spacing) plus 2^-10 of sum|x_i w_i| m / s_out, and exactly +-448 where |v / s_out| > 448
  (saturation; torch's float8 cast does not saturate, so references are clamped).  The second term is the tensor
  core's: Hopper's e4m3 wgmma does not add the products of an instruction in full fp32 (about 13 bits are kept after
  aligning them, as DeepSeek-V3's report, section 3.3.2, describes for the same hardware), so where the products
  cancel, the exact fp32 sum of the reference and the kernel's accumulator differ by a few 2^-13 of the magnitude sum.
  The heads' fp16 / bf16 logits take the 16-bit bound plus that term."""
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F
from torchvision.ops.misc import Conv2dNormActivation

from yolort_b200 import _C
from yolort_b200.engine import _fold_conv_norm, _split_conv_norm_act, act_code, fold_conv_bn
from yolort_b200.models.common import Conv, Focus

TOL = {torch.float16: 2.0 ** -9, torch.bfloat16: 2.0 ** -6}
MANT = {torch.float16: 10, torch.bfloat16: 7}
E4M3 = _C.YB_F8E4M3

_ACTS = {
    _C.YB_ACT_NONE: lambda y: y,
    _C.YB_ACT_SILU: F.silu,
    _C.YB_ACT_HARDSWISH: F.hardswish,
    _C.YB_ACT_LEAKY01: lambda y: F.leaky_relu(y, 0.1),
    _C.YB_ACT_RELU: F.relu,
}


def act_ref(y, code):
    """The epilogue activation YB_ACT_* `code` applied to y, in y's own precision."""
    if code not in _ACTS:
        raise ValueError(f"unknown activation code {code}")
    return _ACTS[code](y)


def to_e4m3(v):
    return v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def ulp_e4m3(v):
    _, e = torch.frexp(v.abs().clamp(min=2.0 ** -6))
    return torch.exp2((e - 4).float())


def ulp(r, dtype):
    """One unit in the last place of the (already rounded) fp16 / bf16 values r, as fp64."""
    e = torch.floor(torch.log2(r.double().abs().clamp_min(torch.finfo(dtype).tiny)))
    return torch.exp2(e - MANT[dtype])


def bound16(ref, dtype, mag=None):
    """fp16 / bf16 outputs: TOL x (1 + |ref|), plus the accumulation term 2^-10 mag of e4m3 operands when given."""
    b = TOL[dtype] * (1.0 + ref.abs())
    return b if mag is None else b + 2.0 ** -10 * mag


def e4m3_bound(ref, mag):
    """(clamped reference, bound) of e4m3 outputs from the fp32 reference and sum|x_i w_i| m, both already divided by
    the output scale (see the module docstring)."""
    slack = 2.0 ** -10 * mag
    sat = ref.abs() > 448.0 + slack
    refc = ref.clamp(-448.0, 448.0)
    return refc, torch.where(sat, 0.0, torch.maximum(ulp_e4m3(refc), torch.full_like(refc, 2.0 ** -9)) + slack)


def compare(got, ref, bound):
    """(violations, max |got - ref|, worst |got - ref| / bound) under `bound`, or exactly when `bound` is None (worst
    is then None).  A NaN counts as a violation."""
    err = (got - ref).abs()
    if bound is None:
        return int((~(err == 0)).sum()), float(err.max()), None
    worst = float(torch.where(err > 0, err / bound, 0.0).max())
    return int((~(err <= bound)).sum()), float(err.max()), worst


def _nchw(t):
    return t.float().permute(0, 3, 1, 2)


def _view(plan, v):
    return plan.buffers[v.buf.name][..., v.ch0: v.ch0 + v.C]


# ---- references: fn(op, x, res, dtype) -> (reference NCHW, bound or None), x / res the op's NHWC inputs -------------
def _conv(op, x, res, dtype):
    co, ci, k = op.dst.C, op.src.C, op.ksize
    w = op.weight[:co, :, :ci].float().view(co, k, k, ci).permute(0, 3, 1, 2).contiguous()
    ref = act_ref(F.conv2d(_nchw(x), w, op.bias[:co], op.stride, op.pad), op.act)
    if res is not None:
        ref = ref + _nchw(res)
    return ref, bound16(ref, dtype)


def _conv_e4m3(op, x, res, dtype):
    """fp32 on the dequantised operands: packed e4m3 weight, per-channel multiplier, fp32 bias and the residual scale
    from the op's tail (lower_fp8), then the output scale."""
    co, ci, k = op.dst.C, op.src.C, op.ksize
    co_pad = op.weight.shape[0]
    w = op.weight[:co, :, :ci].float().view(co, k, k, ci).permute(0, 3, 1, 2)
    tail = op.bias
    xs = _nchw(x)
    mul = tail[co_pad:co_pad + co].view(1, -1, 1, 1)
    v = act_ref(F.conv2d(xs, w, None, op.stride, op.pad) * mul + tail[:co].view(1, -1, 1, 1), op.act)
    if res is not None:
        v = v + _nchw(res) * float(tail[2 * co_pad])
    inv = float(tail[2 * co_pad + 1])
    mag = F.conv2d(xs.abs(), w.abs(), None, op.stride, op.pad) * mul * inv
    if op.dst.buf.esz == 1:
        return e4m3_bound(v * inv, mag)
    return v, bound16(v, dtype, mag)


def _spp(op, x, res, dtype):
    xs = _nchw(x)
    ref = torch.cat([F.max_pool2d(xs, k, 1, k // 2) for k in (5, 9, 13)], 1)
    return ref, (None if op.dtype == E4M3 else bound16(ref, dtype))


def _upsample(op, x, res, dtype):
    ref = F.interpolate(_nchw(x), scale_factor=2.0, mode="nearest")
    return ref, (None if op.dtype == E4M3 else bound16(ref, dtype))


def _quantize(op, x, res, dtype):
    return _nchw(to_e4m3(x.float() * float(op.bias[0]))), None


def _dwconv(op, x, res, dtype):
    """F.conv2d(groups=C) with the op's rounded [k*k][C] weights."""
    C, k = op.src.C, op.ksize
    w = op.weight.float().t().reshape(C, 1, k, k)
    ref = act_ref(F.conv2d(_nchw(x), w, op.bias, op.stride, op.pad, 1, C), op.act)
    return ref, bound16(ref, dtype)


def _se(op, x, res, dtype):
    """x * hardsigmoid(fc2(relu(fc1(mean_hw(x))))) with the op's fp32 fc1 / fc2 (transposed in the op)."""
    C, Sq = op.src.C, op.ksize
    w1 = op.weight[:C * Sq].view(C, Sq).t()
    w2 = op.weight[C * Sq:].view(Sq, C).t()
    b1, b2 = op.bias[:Sq], op.bias[Sq:]
    xf = _nchw(x)
    gate = F.hardsigmoid(F.relu(xf.mean((2, 3)) @ w1.t() + b1) @ w2.t() + b2)
    ref = xf * gate[:, :, None, None]
    return ref, bound16(ref, dtype)


def _attention(op, x, res, dtype):
    """fp32 SDPA on the op's own rounded q | k | v, under the scale 1 + A(|V|)."""
    n, h, w, _ = x.shape
    E, heads = op.dst.C, op.ksize
    q, k, v = x.float().reshape(n, h * w, 3, heads, E // heads).permute(2, 0, 3, 1, 4)

    def nchw(t):
        return t.permute(0, 2, 1, 3).reshape(n, h, w, E).permute(0, 3, 1, 2)

    ref = nchw(F.scaled_dot_product_attention(q, k, v))
    return ref, TOL[dtype] * (1.0 + nchw(F.scaled_dot_product_attention(q, k, v.abs())))


def _avgpool(op, x, res, dtype):
    """Within one ulp of the fp64 mean, rounded to the output type."""
    rounded = x.double().mean((1, 2), keepdim=True).to(dtype).double()
    return rounded.permute(0, 3, 1, 2), ulp(rounded, dtype).permute(0, 3, 1, 2)


# (op.kind, op.dtype): op.dtype is None for the plan's fp16 / bf16 compute type (an FP8 plan's QUANTIZE included: it
# carries its 16-bit source type), YB_F8E4M3 for the e4m3 ops of an FP8 plan
REFERENCES = {
    (_C.YB_OP_CONV, None): _conv,
    (_C.YB_OP_SPP_POOL, None): _spp,
    (_C.YB_OP_UPSAMPLE2X, None): _upsample,
    (_C.YB_OP_ATTENTION, None): _attention,
    (_C.YB_OP_DWCONV, None): _dwconv,
    (_C.YB_OP_SE, None): _se,
    (_C.YB_OP_AVGPOOL, None): _avgpool,
    (_C.YB_OP_QUANTIZE, None): _quantize,
    (_C.YB_OP_CONV, E4M3): _conv_e4m3,
    (_C.YB_OP_SPP_POOL, E4M3): _spp,
    (_C.YB_OP_UPSAMPLE2X, E4M3): _upsample,
}


def reference_for(op):
    """The reference of `op`.  An op without one is an error: no kind falls back to another kind's reference."""
    key = (op.kind, op.dtype)
    if key not in REFERENCES:
        raise KeyError(f"{op.name}: no stage-wise reference for op kind {op.kind} with element type {op.dtype}")
    return REFERENCES[key]


def stem_reference(stem, canvas, dtype):
    """The stem module's own output over the RGB canvas rebuilt from the plan's space-to-depth input `canvas`
    ([N, H/2, W/2, 16], channel (dy*2+dx)*4 + c): a Focus slices 2x2 and applies its 3x3/s1/p1 convolution, the r6.0
    Conv its 6x6/s2/p2 one, the lite model's Conv2dNormActivation its 3x3/s2/p1 one.  BN folded in fp64, the weight
    rounded to `dtype`, computed in fp32."""
    n, h2, w2, _ = canvas.shape
    x = canvas.float().view(n, h2, w2, 2, 2, 4)[..., :3].permute(0, 5, 1, 3, 2, 4).reshape(n, 3, 2 * h2, 2 * w2)
    if isinstance(stem, Focus):       # parity order (row, col) = (0,0), (1,0), (0,1), (1,1)
        x = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)
        stem = stem.conv
    if isinstance(stem, Conv):
        conv, (w, b), act = stem.conv, fold_conv_bn(stem), act_code(stem.act)
    elif isinstance(stem, Conv2dNormActivation):
        conv, bn, act = _split_conv_norm_act("stem", stem)
        w, b = _fold_conv_norm(conv, bn)
    else:
        raise NotImplementedError(f"no stem reference for {type(stem).__name__}")
    return act_ref(F.conv2d(x, w.to(dtype).float(), b.float(), conv.stride, conv.padding), act)


class Record(NamedTuple):
    name: str
    violations: int
    max_err: float
    worst: Optional[float]      # largest error / bound; None where the reference is exact


def check_plan_stagewise(plan, stem, verbose=True):
    """`plan` must have been created with keep_intermediates=True and its input canvas written; `stem` is the model's
    stem module.  Launches the plan ONE launch at a time and checks each op right after its launch ran.  The inputs of
    a launch's first op are snapshotted before it runs: SE, C3's last bottleneck (it writes over cv1's half of the
    concat buffer, its own residual) and C3TR work in place.  A 1x1 convolution that rides as the chained tail of its
    predecessor (PlanInstance.launch_ops) reads that output after the launch: keep_intermediates plans store it, so the
    tail is checked against fp32 applied to exactly the tile it consumed on chip.  Returns one Record per op of the
    lowering."""
    assert plan.keep_intermediates
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ops = plan._low.L.ops
    out = []
    for li, grp in enumerate(plan.launch_ops):
        x, res = (None if v is None else _view(plan, v).clone() for v in (ops[grp[0]].src, ops[grp[0]].residual))
        plan.run(li, 1)
        torch.cuda.synchronize()
        for i in grp:
            op = ops[i]
            if i != grp[0]:
                x, res = (None if v is None else _view(plan, v) for v in (op.src, op.residual))
            if op.pack > 1:
                ref = stem_reference(stem, x, plan.dtype)
                bound = bound16(ref, plan.dtype)
            else:
                ref, bound = reference_for(op)(op, x, res, plan.dtype)
            bad, mx, worst = compare(_nchw(_view(plan, op.dst)), ref, bound)
            if verbose and (bad or mx > 0.05):
                print(f"  stage {op.name}: violations {bad} max_abs_err {mx:.3e} ref_absmax {float(ref.abs().max()):.2f}")
            out.append(Record(op.name + (" [fused launch]" if len(grp) > 1 else ""), bad, mx, worst))
            del ref, bound
    if verbose:
        fracs = [r.worst for r in out if r.worst is not None]
        print(f"stage-wise N{plan.N} {plan.H}x{plan.W} {plan.dtype}: {len(out)} records for {len(ops)} ops, worst "
              f"max_abs_err {max(r.max_err for r in out):.3e}, worst {max(fracs):.3f} of the bound, ops with violations "
              f"{sum(1 for r in out if r.violations)}")
    return out
