"""Cases for the split tail of the 1x1 / im2col kernel (csrc/conv_sm90.cu): when the tiles are not a whole number of
rounds of the persistent grid and the last round holds at most half a grid of 128-column tiles, each of those tiles runs
as two halves on CTAs that would otherwise idle: 64-row halves with two consumer warpgroups, 64-column halves with one
(yb_conv_config: `tail_tiles`, `tail_split`).

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py and are sized from the device's SM
count so that each lands on the side of the rule its name states.
"""
from conv_cases import BF16, F16, LEAKY, NONE, RELU, SMS, Case
from yolort_b200 import _C


def split_key(case: Case, cfg: dict) -> tuple:
    """(dtype, N tile, layout, slices per tail tile): the instance and the path a launch runs."""
    return ("bf16" if case.dtype == BF16 else "f16", cfg["block_n"], cfg["layout"], cfg["tail_split"])


def _cases():
    S = SMS
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # 3 x SMs + 4 128-row tiles: four tail tiles, eight slices
            Case(f"{b} split 1x2 1x1 128->128 r=4", 1, 128, 3 * S + 4, 128, 128, dtype=dt, seed=201, bias_scale=4.0,
                 residual=True, res_cstride=160, res_off=16),
            # ragged Cout (the second slice of a tile is partly past Cout) and ragged M, in a channel window
            Case(f"{b} split 1x2 1x1 96->120 ragged", 1, 125, 128 * (3 * S + 4) // 125, 96, 120, dtype=dt, seed=202,
                 act=RELU,
                 out_cstride=152, out_off=16),
            # im2col (4-D TMA) A tiles
            Case(f"{b} split 1x2 im2col 3x3 s2 64->128", 1, 2 * 64, 2 * (2 * S + 3), 64, 128, k=3, s=2, dtype=dt,
                 reserved=_C.YB_CONV_FORCE_IM2COL, seed=203, act=LEAKY),
            # four 128-column N tiles with streamed weights: halves take their rows of the streamed B sub-tiles
            Case(f"{b} split 1x2 1x1 128->512 streamed", 1, 128, S // 4 + 1, 128, 512, dtype=dt, seed=204,
                 bias_scale=2.0),
            # 64-row tiles, two CTAs per SM, two resident N tiles
            Case(f"{b} split 2x1 1x1 64->256", 2, 64, 3 * S + 2, 64, 256, dtype=dt, seed=205, act=NONE),
            # the rule's edges: exactly half a grid of tail tiles splits, one more does not
            Case(f"{b} split 1x2 1x1 64->128 r=G/2", 1, 128, 2 * S + S // 2, 64, 128, dtype=dt, seed=206),
            Case(f"{b} whole 1x2 1x1 64->128 r=G/2+1", 1, 128, 2 * S + S // 2 + 1, 64, 128, dtype=dt, seed=207),
            # streamed 256-column weights over 2-4 rounds: planned as two 128-column N tiles so the tail splits; at more
            # rounds the 256-column tile stays
            Case(f"{b} split 1x2 1x1 512->256 streamed few rounds", 1, 128, 3 * S + 4, 512, 256, dtype=dt, seed=209,
                 residual=True),
            Case(f"{b} whole256 1x2 1x1 512->256 streamed 4xSMs+4", 1, 128, 4 * S + 4, 512, 256, dtype=dt, seed=210),
            # a whole number of rounds has no tail
            Case(f"{b} whole 1x2 1x1 64->128 r=0", 1, 128, 3 * S, 64, 128, dtype=dt, seed=208),
        ]
    return C


CASES = _cases()
