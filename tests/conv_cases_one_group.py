"""Cases for the one-consumer-warpgroup layout of the 1x1 / im2col kernel (csrc/conv_sm90.cu): two CTAs per SM, each
one producer and one consumer warpgroup over 64-row tiles (yb_conv_config: info[11] bit 2, `layout` "2x1").  The
layout takes layers whose one-CTA plan has a 256-column N tile, as two 128-column N tiles with resident weights, at
3 x SMs 128-row tiles and more.

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py.  Every case is sized from the
device's SM count so that it lands on the side of the planner's rule its name states.
"""
from conv_cases import BF16, F16, LEAKY, NONE, RELU, SMS, Case
from yolort_b200 import _C

ROWS = 128                                                # rows of the one-CTA tile the threshold counts


def one_group_key(case: Case, d, cfg: dict) -> tuple:
    """(kernel, dtype, N tile, fused decode, tail N, layout): the template instance the launch runs."""
    return ("conv", "bf16" if case.dtype == BF16 else "f16", cfg["block_n"], bool(d.decode), 0, cfg["layout"])


def one_group_paths(case: Case, cfg: dict) -> set:
    """Named plan paths of the one-group layout (and of the rule that keeps a launch off it)."""
    p = set()
    if cfg["patch_kernel"]:
        return p
    m_tiles = (case.N * case.Ho * case.Wo + ROWS - 1) // ROWS
    if cfg["layout"] == "2x1":
        p.add("2x1 1x1 resident" if case.k == 1 and case.s == 1 else "2x1 im2col")
        if case.Cout % 128:
            p.add("2x1 ragged second N tile")
        if case.N * case.Ho * case.Wo % 64:
            p.add("2x1 ragged M")
        if m_tiles == 3 * SMS:
            p.add("2x1 at 3 x SMs 128-row tiles")
    elif cfg["layout"] == "1x2" and m_tiles >= 2 * SMS:
        if m_tiles == 3 * SMS - 1 and cfg["block_n"] == 256:
            p.add("1x2 at 3 x SMs - 1 128-row tiles")
        if cfg["block_n"] == 256 and not cfg["weights_resident"]:
            p.add("1x2 streamed weights")
        if cfg["block_n"] == 128:
            p.add("1x2 N = 128")
    return p


def _cases():
    S = SMS
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            Case(f"{b} 2x1 1x1 64->256 at 3xSMs tiles", 3, 128, S, 64, 256, dtype=dt, seed=101, bias_scale=4.0,
                 residual=True, res_cstride=288, res_off=16),
            Case(f"{b} 1x2 1x1 64->256 at 3xSMs-1 tiles", 1, 3 * S - 1, 128, 64, 256, dtype=dt, seed=102),
            Case(f"{b} 2x1 1x1 256->256", 3, 128, S + 1, 256, 256, dtype=dt, seed=103, act=LEAKY, bias_scale=2.0),
            Case(f"{b} 2x1 1x1 96->200 ragged resid-window", 4, 103, S - 7, 96, 200, dtype=dt, seed=104,
                 act=RELU, residual=True, res_cstride=256, res_off=40, out_cstride=232, out_off=24),
            Case(f"{b} 2x1 im2col 3x3 s2 32->256 ragged", 7, 2 * 61, 2 * (S - 3), 32, 256, k=3, s=2, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, seed=105, act=NONE, bias_scale=2.0),
            Case(f"{b} 1x2 1x1 512->256 streamed", 3, 128, S, 512, 256, dtype=dt, seed=106),
            Case(f"{b} 1x2 1x1 128->128", 3, 128, S, 128, 128, dtype=dt, seed=107),
        ]
    return C


CASES = _cases()
