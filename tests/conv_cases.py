"""One case table for the fp16/bf16 convolution kernels (csrc/conv_sm90.cu, csrc/conv3x3_patch_sm90.cu).

A `Case` describes one convolution launch (optionally with a chained 1x1 tail); `build_desc` turns it into the OpDesc
(and ConvChain) the library plans, from a pointer provider: fake 16-byte-aligned addresses on a machine without a GPU
(tests/test_conv_coverage.py asks `yb_conv_config` which kernel instance and plan path each case takes), real tensors
on the GPU (`check_case`, used by tests/test_gpu_conv_cases.py and by run_conv / run_chain in tests/test_gpu_conv.py).

`check_case` compares a launch with an fp64 convolution of the same fp16/bf16-rounded operands, under a bound that
scales with the operands' magnitude (see `tau`), and checks that nothing outside the destination view is written, that
a second launch gives the same bits and that a two-CTA launch gives the bits of the one-CTA launch.
"""
import ctypes
import dataclasses
from typing import Callable, Optional

import torch
import torch.nn.functional as F

from stagewise import act_ref
from yolort_b200 import _C
from yolort_b200.engine import pack_bias, pack_weight

F16, BF16 = torch.float16, torch.bfloat16
NONE, SILU, HSWISH, LEAKY, RELU = (_C.YB_ACT_NONE, _C.YB_ACT_SILU, _C.YB_ACT_HARDSWISH, _C.YB_ACT_LEAKY01,
                                   _C.YB_ACT_RELU)
SENTINEL = 7.0
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@dataclasses.dataclass(frozen=True)
class Chain:
    """Chained 1x1 tail over [first_out[:c_own] | extra (c_own channels)] -> C2 channels."""
    c_own: int
    C2: int
    extra: bool = False
    store_first: bool = True
    act2: int = SILU


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    N: int
    H: int
    W: int
    Cin: int
    Cout: int
    k: int = 1
    s: int = 1
    dtype: torch.dtype = F16
    act: int = SILU
    residual: bool = False
    res_cstride: int = 0     # channels of the residual buffer (0: Cout)
    res_off: int = 0         # first channel of the residual window
    in_cstride: int = 0      # channels of the input buffer (0: Cin)
    in_off: int = 0          # first channel of the input window
    out_cstride: int = 0     # channels of the output buffer (0: Cout, plus the extra operand of a chain)
    out_off: int = 0         # first channel of the output window
    reserved: int = 0
    seed: int = 0
    bias_scale: float = 0.5
    chain: Optional[Chain] = None

    @property
    def pad(self) -> int:
        return self.k // 2

    @property
    def Ho(self) -> int:
        return (self.H + 2 * self.pad - self.k) // self.s + 1

    @property
    def Wo(self) -> int:
        return (self.W + 2 * self.pad - self.k) // self.s + 1

    @property
    def in_cs(self) -> int:
        return self.in_cstride or self.Cin

    @property
    def res_cs(self) -> int:
        return self.res_cstride or self.Cout

    @property
    def out_cs(self) -> int:
        if self.out_cstride:
            return self.out_cstride
        return self.Cout + (self.chain.c_own if self.chain and self.chain.extra else 0)

    @property
    def extra_off(self) -> int:
        """First channel of a chain's extra operand: the window right of the first output (C3's concat)."""
        return self.out_off + self.Cout

    @property
    def out2_cs(self) -> int:
        return self.chain.C2 + 16        # the tail writes into a channel window too


def _pads(co: int, ci: int, dtype) -> tuple:
    _, ci_pad, co_pad = pack_weight(torch.zeros(co, ci, 1, 1, dtype=torch.float64), dtype, torch.device("cpu"))
    return ci_pad, co_pad


def build_desc(case: Case, ptr: Callable[[str], int]):
    """The OpDesc of `case`; `ptr(name)` gives the base address of buffer name ("x", "w", "b", "res", "out", "w2",
    "b2", "out2").  Returns (desc, chain struct or None); the chain struct must outlive the descriptor."""
    c = case
    ci_pad, co_pad = _pads(c.Cout, c.Cin, c.dtype)
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_CONV, _C.dtype_code(c.dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride = c.N, c.H, c.W, c.Cin, c.in_cs
    d.in_ = ptr("x") + 2 * c.in_off
    d.Ho, d.Wo, d.Cout, d.out_cstride = c.Ho, c.Wo, c.Cout, c.out_cs
    d.out = ptr("out") + 2 * c.out_off
    d.ksize, d.stride, d.pad, d.act = c.k, c.s, c.pad, c.act
    d.weight, d.Cin_pad, d.Cout_pad, d.bias = ptr("w"), ci_pad, co_pad, ptr("b")
    if c.residual:
        d.residual, d.res_cstride = ptr("res") + 2 * c.res_off, c.res_cs
    d.reserved = c.reserved
    ch = None
    if c.chain is not None:
        t = c.chain
        k2 = t.c_own * (2 if t.extra else 1)
        k2_pad, co2_pad = _pads(t.C2, k2, c.dtype)
        ch = _C.ConvChain()
        ch.weight, ch.bias, ch.Cout, ch.Cout_pad, ch.K_pad = ptr("w2"), ptr("b2"), t.C2, co2_pad, k2_pad
        ch.act = t.act2
        ch.out, ch.out_cstride, ch.own_C = ptr("out2"), c.out2_cs, t.c_own
        if t.extra:
            ch.extra, ch.extra_C, ch.extra_cstride = ptr("out") + 2 * c.extra_off, t.c_own, c.out_cs
        ch.store_first = 1 if t.store_first else 0
        d.chain = ctypes.addressof(ch)
    return d, ch


_FAKE = {n: 0x7F00_0000_0000 + ((i + 1) << 32) for i, n in enumerate(("x", "w", "b", "res", "out", "w2", "b2", "out2"))}


def fake_ptr(name: str) -> int:
    """16-byte (in fact 4 GiB) aligned addresses that are never dereferenced: host planning only."""
    return _FAKE[name]


# ---- what the planner does with a case (yb_conv_config) ----------------------------------------------------------------
def instance_key(case: Case, d, cfg: dict) -> tuple:
    """(kernel, dtype, N tile, fused decode, tail N, CTAs per SM): the template instance the launch runs."""
    kernel = "patch" if cfg["patch_kernel"] else "conv"
    return (kernel, "bf16" if case.dtype == BF16 else "f16", cfg["block_n"], bool(d.decode), cfg["tail_n"],
            cfg["ctas_per_sm"])


def plan_paths(case: Case, cfg: dict) -> set:
    """Named plan paths a case exercises."""
    p = set()
    res = "resident" if cfg["weights_resident"] else "streamed"
    if cfg["patch_kernel"]:
        tiling = cfg["patch_tiling"]
        p.add(f"patch {tiling}")
        if cfg["weights_resident"]:
            p.add("patch resident single N tile" if cfg["n_tiles"] == 1 else "patch resident N-split")
        elif cfg["tiles_per_pass"] == 2:
            p.add("patch streamed pairs")
            if cfg["m_tiles"] % 2:
                p.add("patch streamed odd last pair")
        if cfg["ctas_per_sm"] == 2:
            p.add(f"two CTAs patch {tiling}")
    else:
        if case.k == 1 and case.s == 1:
            p.add(f"conv 1x1 {res}")
        elif case.k == 3:
            p.add(f"conv im2col 3x3 s{case.s} {res}")
        else:
            p.add(f"conv im2col k{case.k}")
        if cfg["n_tiles"] > 1:
            p.add("conv several N tiles")
        if cfg["ctas_per_sm"] == 2:
            p.add("two CTAs conv")
    n = cfg["work_items"]
    if cfg["ctas_per_sm"] == 2 and n == 2 * SMS:
        p.add("two CTAs at 2 x SMs tiles")
    if cfg["ctas_per_sm"] == 1 and n == 2 * SMS - 1:
        p.add("one CTA at 2 x SMs - 1 tiles")
    if case.chain is not None:
        t = case.chain
        p.add("chain one own chunk" if t.c_own <= 64 else "chain two own chunks")
        if t.extra:
            p.add("chain extra operand")
        if not t.store_first:
            p.add("chain store_first=0")
    return p


# ---- the case table -------------------------------------------------------------------------------------------------
def _cases():
    S = SMS
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # ---- 1x1 / im2col kernel, one CTA per SM (fewer than 2 x SMs tiles) ----
            Case(f"{b} 1x1 Cout16", 2, 20, 20, 32, 16, dtype=dt, seed=1, residual=True, res_cstride=48, res_off=16),
            Case(f"{b} 1x1 Cout24 relu", 1, 17, 19, 64, 24, dtype=dt, act=RELU, seed=2, bias_scale=1.0),
            Case(f"{b} 1x1 Cout40 in-window", 2, 13, 11, 48, 40, dtype=dt, in_cstride=96, in_off=32, seed=3),
            Case(f"{b} 1x1 Cout72 leaky", 2, 16, 20, 80, 72, dtype=dt, act=LEAKY, seed=4, bias_scale=1.0,
                 out_cstride=96, out_off=8),
            Case(f"{b} 1x1 Cout200 none", 1, 20, 24, 64, 200, dtype=dt, act=NONE, seed=5),
            Case(f"{b} im2col 3x3 s1 128 resid-window", 2, 20, 20, 128, 128, k=3, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, residual=True, res_cstride=256, res_off=64, seed=6),
            Case(f"{b} im2col 3x3 s2 streamed", 1, 24, 16, 256, 128, k=3, s=2, dtype=dt, seed=7, act=HSWISH,
                 bias_scale=2.0),
            Case(f"{b} im2col 3x3 s1 resident hswish", 2, 18, 22, 32, 64, k=3, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, act=HSWISH, bias_scale=2.0, seed=42),
            Case(f"{b} im2col 5x5 Cin48", 2, 14, 18, 48, 64, k=5, dtype=dt, seed=8),
            Case(f"{b} 1x1 K1024 streamed 2 N tiles", 1, 16, 16, 1024, 512, dtype=dt, seed=9),
            # ---- 1x1 kernel at 2 x SMs tiles and more: N = 256 without decode, one and two CTAs ----
            Case(f"{b} 1x1 Cout256 >=2xSMs tiles", 2, 128, S, 64, 256, dtype=dt, seed=10),
            Case(f"{b} 1x1 Cout200 >=2xSMs tiles relu", 2, 128, S, 32, 200, dtype=dt, act=RELU, seed=11),
            Case(f"{b} 2cta 1x1 Cout16 ragged", 3, 91, S - 3, 32, 16, dtype=dt, seed=12, bias_scale=6.0),
            Case(f"{b} 2cta 1x1 Cout32 at 2xSMs", 2, 128, S, 64, 32, dtype=dt, seed=13, bias_scale=6.0,
                 residual=True, res_cstride=64, res_off=32),
            Case(f"{b} 1cta 1x1 Cout32 at 2xSMs-1", 1, 2 * S - 1, 128, 64, 32, dtype=dt, seed=14),
            Case(f"{b} 2cta im2col 3x3 s2 Cout64 leaky", 4, 2 * 96, 2 * 96, 32, 64, k=3, s=2, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, act=LEAKY, seed=15, bias_scale=2.0),
            Case(f"{b} 2cta 1x1 Cout64 in-window", 5, 57, S + 1, 64, 64, dtype=dt, in_cstride=128, in_off=64,
                 out_cstride=128, out_off=64, seed=16, bias_scale=6.0),
            # ---- 1x1 kernel with chained tails ----
            Case(f"{b} chain 1x1 64->[32]->32", 2, 24, 20, 64, 64, dtype=dt, chain=Chain(32, 32), seed=17),
            Case(f"{b} chain 1x1 64->[64]->64", 2, 24, 20, 128, 64, dtype=dt, chain=Chain(64, 64), seed=18),
            Case(f"{b} chain 1x1 64->[64]->128 sf0", 2, 24, 20, 64, 64, dtype=dt,
                 chain=Chain(64, 128, store_first=False, act2=NONE), seed=19),
            Case(f"{b} chain 1x1 128->[128]->32", 2, 24, 20, 64, 128, dtype=dt, chain=Chain(128, 32), seed=20),
            Case(f"{b} chain 1x1 128->[64]->64 resid", 2, 24, 20, 64, 128, dtype=dt, chain=Chain(64, 64),
                 residual=True, seed=21),
            Case(f"{b} chain im2col 3x3 128->[128]->128", 1, 20, 24, 64, 128, k=3, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, chain=Chain(128, 120, store_first=False), seed=22),
            Case(f"{b} 2cta chain 1x1 64->[32]->32", 2, 128, S, 64, 64, dtype=dt, chain=Chain(32, 32), seed=23,
                 bias_scale=6.0),
            Case(f"{b} 2cta chain 1x1 64->[64]->64 ragged", 3, 97, S - 1, 32, 64, dtype=dt,
                 chain=Chain(64, 56, store_first=False), seed=24),
            # ---- halo-patch kernel ----
            Case(f"{b} patch classic Cout24", 2, 32, 40, 32, 24, k=3, dtype=dt, seed=25, act=RELU),
            Case(f"{b} patch pairs Cin80 Cout40 in-window", 2, 24, 40, 80, 40, k=3, dtype=dt, in_cstride=128,
                 in_off=16, seed=26),
            Case(f"{b} patch pairs Cout72 resid-window", 1, 40, 44, 48, 72, k=3, dtype=dt, residual=True,
                 res_cstride=96, res_off=24, seed=27),
            Case(f"{b} patch N-split 64->256", 2, 40, 40, 64, 256, k=3, dtype=dt, seed=28),
            Case(f"{b} patch N-split 32->256 relu", 2, 40, 40, 32, 256, k=3, dtype=dt, seed=29, act=RELU),
            Case(f"{b} patch streamed odd pair", 1, 40, 40, 128, 128, k=3, dtype=dt, seed=30, act=LEAKY),
            Case(f"{b} patch wrap streamed pairs", 2, 20, 20, 256, 200, k=3, dtype=dt, seed=31),
            Case(f"{b} patch stride2 Cout72", 2, 64, 48, 48, 72, k=3, s=2, dtype=dt, seed=32, residual=True),
            Case(f"{b} patch chain 32->[32]->128", 2, 40, 44, 32, 32, k=3, dtype=dt,
                 chain=Chain(32, 128, extra=True, store_first=False), residual=True, seed=33),
            Case(f"{b} patch chain 32->[32]->64", 2, 40, 44, 32, 32, k=3, dtype=dt, chain=Chain(32, 64), seed=34),
            Case(f"{b} patch chain 64->[64]->64", 2, 20, 20, 64, 64, k=3, dtype=dt,
                 chain=Chain(64, 64, extra=True), seed=35),
            Case(f"{b} patch chain 64->[64]->128", 2, 40, 40, 64, 64, k=3, dtype=dt,
                 chain=Chain(64, 128, extra=True, store_first=False), residual=True, seed=36),
            # ---- halo-patch kernel, two CTAs per SM ----
            Case(f"{b} 2cta patch classic Cout32", (2 * S + 31) // 32 + 1, 64, 64, 32, 32, k=3, dtype=dt, seed=37,
                 bias_scale=6.0, residual=True, res_cstride=64, res_off=8),
            Case(f"{b} 2cta patch wrap Cout64", S // 2 + 3, 20, 20, 32, 64, k=3, dtype=dt, seed=38,
                 bias_scale=6.0),
            Case(f"{b} 2cta patch wrap ragged Cout40", S // 2 + 5, 19, 20, 32, 40, k=3, dtype=dt, seed=39,
                 act=RELU, bias_scale=2.0),
            Case(f"{b} 2cta patch stride2 Cout64", (2 * S + 7) // 8 + 1, 64, 64, 32, 64, k=3, s=2, dtype=dt,
                 seed=40, bias_scale=6.0),
            Case(f"{b} 2cta patch chain 32->[32]->64", (2 * S + 31) // 32 + 2, 64, 64, 32, 32, k=3, dtype=dt,
                 chain=Chain(32, 64, extra=True, store_first=False), residual=True, seed=41, bias_scale=6.0),
        ]
    return C


CASES = _cases()

# Instances no case of this table reaches, with the reason and the test that covers them.
EXCLUDED = {
    ("conv", "f16", 256, True, 0, 1): "fused decode needs a detection head and a candidate arena: "
                                      "tests/test_gpu_network.py::test_fused_head_decode_equals_unfused",
    ("conv", "bf16", 256, True, 0, 1): "fused decode needs a detection head and a candidate arena: "
                                       "tests/test_gpu_network.py::test_fused_head_decode_equals_unfused",
}


# ---- fp64 reference and bound ------------------------------------------------------------------------------------------
def tau(K: int) -> float:
    """Relative allowance, against mag = conv(|x|, |w|) + |b| (+ |res|), for everything but the final rounding.

    * Every product of two fp16 (11-bit) or bf16 (8-bit) significands is exact in fp32.
    * The K products are summed into fp32 accumulators.  The tensor core aligns the addends of a K-step to the
      largest exponent and truncates, so each addition may lose up to one fp32 ulp (2^-23, not the 2^-24 of
      round-to-nearest) of a partial sum, and every partial sum is at most mag: <= K * 2^-23 * mag.
    * The fp32 bias addition rounds once more: 2^-23 * mag (counted as one more term).
    * The activation multiplies the pre-activation error by at most its largest slope: 1.5 (Hardswish at v = 3;
      SiLU 1.1, LeakyReLU / ReLU 1).
    * SiLU evaluates v / (1 + 2^(-v log2 e)) with ex2.approx (relative error <= 2^-22) and rcp.approx (<= 2^-23),
      plus three fp32 roundings: <= 2^-20 * |v| <= 2^-20 * mag.
    * The fp32 residual addition: 2^-24 * mag.
    """
    return 1.5 * (K + 1) * 2.0 ** -23 + 2.0 ** -20 + 2.0 ** -24


def ulp_out(a: torch.Tensor, dtype) -> torch.Tensor:
    """One unit in the last place of the output format at |ref| (subnormal spacing below the normal range): covers the
    final rounding to fp16 / bf16, including a value that rounds up across a power of two."""
    mant, emin = (10, -14) if dtype == F16 else (7, -126)
    _, e = torch.frexp(torch.clamp(a, min=2.0 ** emin))
    return torch.ldexp(torch.ones_like(a), (e - 1 - mant).to(torch.int32))


def _nchw(t: torch.Tensor) -> torch.Tensor:
    return t.double().permute(0, 3, 1, 2)


def operands(case: Case, device) -> dict:
    """The case's tensors (seeded, generated on the CPU): fp16/bf16 activations, weights and residual, fp32 bias,
    output buffers of N + 1 images filled with the sentinel (the last image is a guard after the view)."""
    c = case
    g = torch.Generator().manual_seed(c.seed)
    t = {}
    t["x"] = torch.randn(c.N, c.H, c.W, c.in_cs, generator=g).to(c.dtype)
    w = (torch.randn(c.Cout, c.Cin, c.k, c.k, generator=g) * (2.0 / (c.Cin * c.k * c.k)) ** 0.5).to(c.dtype)
    t["b32"] = torch.randn(c.Cout, generator=g) * c.bias_scale
    t["w4"] = w
    t["w"], _, co_pad = pack_weight(w.double(), c.dtype, device)
    t["b"] = pack_bias(t["b32"].double(), co_pad, device)
    if c.residual:
        t["res"] = torch.randn(c.N, c.Ho, c.Wo, c.res_cs, generator=g).to(c.dtype)
    out = torch.full((c.N + 1, c.Ho, c.Wo, c.out_cs), SENTINEL, dtype=c.dtype)
    if c.chain is not None:
        ch = c.chain
        k2 = ch.c_own * (2 if ch.extra else 1)
        w2 = (torch.randn(ch.C2, k2, 1, 1, generator=g) * (2.0 / k2) ** 0.5).to(c.dtype)
        t["b2_32"] = torch.randn(ch.C2, generator=g) * 0.5
        t["w2_4"] = w2
        t["w2"], _, co2_pad = pack_weight(w2.double(), c.dtype, device)
        t["b2"] = pack_bias(t["b2_32"].double(), co2_pad, device)
        if ch.extra:      # the cv2 half of a C3 concat, right of the first output
            out[:c.N, ..., c.extra_off:c.extra_off + ch.c_own] = torch.randn(c.N, c.Ho, c.Wo, ch.c_own, generator=g)
        t["out2"] = torch.full((c.N + 1, c.Ho, c.Wo, c.out2_cs), SENTINEL, dtype=c.dtype)
    t["out"] = out
    return {k: v.to(device) for k, v in t.items()}


def _outside(buf: torch.Tensor, N: int, lo: int, hi: int) -> torch.Tensor:
    """Every element of `buf` outside channels [lo, hi) of images [0, N): the channel sentinels and the guard image."""
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[:N, ..., lo:hi] = False
    return buf[mask]


def _report(what, got, ref, mag, K, dtype, legacy_tol):
    """max |got - ref| / bound; prints and returns the worst fraction, asserts it is <= 1 (and the legacy stage-wise
    bound tol * (1 + |ref|) when given)."""
    err = (got.double() - ref).abs()
    bound = ulp_out(ref.abs(), dtype) + tau(K) * mag
    frac = err / bound
    worst = float(frac.max())
    i = tuple(int(v) for v in (frac == frac.max()).nonzero()[0])
    print(f"  {what}: worst {worst:.3f} of the bound at (n,c,y,x)={i}: got {float(got[i]):.6g} ref {float(ref[i]):.6g} "
          f"mag {float(mag[i]):.4g}; max_abs_err {float(err.max()):.3e}; violations {int((frac > 1).sum())}/{frac.numel()}")
    assert worst <= 1.0, f"{what}: error {worst:.3f} x the bound"
    if legacy_tol is not None:
        bad = int((err > legacy_tol * (1 + ref.abs())).sum())
        assert bad == 0, f"{what}: {bad} elements outside the stage-wise bound"
    return worst


def _launch(case, t, device):
    t["out"].copy_(t["out0"])
    if case.chain is not None:
        t["out2"].fill_(SENTINEL)
    d, ch = build_desc(case, lambda n: t[n].data_ptr())
    if case.chain is not None:
        assert _C.conv_chain_supported(d), _C.lib().yb_last_error().decode()
    plan = _C.Plan([d], device)
    plan.run()
    torch.cuda.synchronize()
    del plan, ch
    return t["out"].clone(), (t["out2"].clone() if case.chain is not None else None)


def check_case(case: Case, device=torch.device("cuda:0"), legacy_tol=None) -> dict:
    """Runs `case` on the GPU and checks it (see the module docstring).  Returns the worst fractions of the bound."""
    torch.backends.cudnn.allow_tf32 = False
    c = case
    t = operands(c, device)
    t["out0"] = t["out"].clone()
    sf = c.chain is not None and not c.chain.store_first
    stored = dataclasses.replace(c, chain=dataclasses.replace(c.chain, store_first=True)) if sf else c
    d, _ch = build_desc(stored, fake_ptr)
    cfg = _C.conv_config(d)
    key = instance_key(c, d, cfg)
    print(f"{c.name}: instance {key} grid {cfg['grid']} paths {sorted(plan_paths(c, cfg))}")
    out, out2 = _launch(stored, t, device)

    # ---- nothing outside the destination view(s) changed ----
    lo, hi = c.out_off, c.out_off + c.Cout
    assert torch.equal(_outside(out, c.N, lo, hi), _outside(t["out0"], c.N, lo, hi)), "wrote outside the output view"
    if c.chain is not None:
        assert torch.all(_outside(out2, c.N, 0, c.chain.C2) == SENTINEL), "tail wrote outside its output view"

    # ---- first output against fp64 ----
    x = _nchw(t["x"][..., c.in_off:c.in_off + c.Cin])
    w = t["w4"].double()
    b = t["b32"].double()
    pre = F.conv2d(x, w, b, c.s, c.pad)
    mag = F.conv2d(x.abs(), w.abs(), b.abs(), c.s, c.pad)
    ref = act_ref(pre, c.act)
    if c.residual:
        r = _nchw(t["res"][..., c.res_off:c.res_off + c.Cout])
        ref, mag = ref + r, mag + r.abs()
    got = out[:c.N, ..., lo:hi].permute(0, 3, 1, 2)
    worst = {"key": key, "first": _report("output", got, ref, mag, c.Cin * c.k * c.k, c.dtype, legacy_tol)}

    # ---- chained tail against fp64 applied to the STORED first output (= the tile the tail consumed on chip) ----
    if c.chain is not None:
        ch = c.chain
        own = out[:c.N, ..., lo:lo + ch.c_own]
        a2 = torch.cat([own, out[:c.N, ..., c.extra_off:c.extra_off + ch.c_own]], -1) if ch.extra else own
        a2 = _nchw(a2)
        w2, b2 = t["w2_4"].double(), t["b2_32"].double()
        ref2 = act_ref(F.conv2d(a2, w2, b2), ch.act2)
        mag2 = F.conv2d(a2.abs(), w2.abs(), b2.abs())
        got2 = out2[:c.N, ..., :ch.C2].permute(0, 3, 1, 2)
        worst["tail"] = _report("tail", got2, ref2, mag2, a2.shape[1], c.dtype, legacy_tol)

    # ---- a second launch gives the same bits ----
    again, again2 = _launch(stored, t, device)
    assert torch.equal(again, out), "second launch differs"
    if c.chain is not None:
        assert torch.equal(again2, out2), "second launch of the tail differs"

    # ---- two CTAs per SM: the bits of the one-CTA launch ----
    if cfg["ctas_per_sm"] == 2:
        one = dataclasses.replace(stored, reserved=stored.reserved | _C.YB_CONV_ONE_CTA)
        d1, _c1 = build_desc(one, fake_ptr)
        assert _C.conv_config(d1)["ctas_per_sm"] == 1
        o1, o21 = _launch(one, t, device)
        assert torch.equal(o1, out), "two-CTA launch differs from the one-CTA launch"
        if c.chain is not None:
            assert torch.equal(o21, out2), "two-CTA tail differs from the one-CTA launch"

    # ---- store_first = 0: the same tail bits, and nothing of the first output written ----
    if sf:
        o, o2 = _launch(c, t, device)
        assert torch.equal(o2, out2), "store_first=0 changes the tail"
        assert torch.equal(o, t["out0"]), "store_first=0 wrote the first output"
    return worst
