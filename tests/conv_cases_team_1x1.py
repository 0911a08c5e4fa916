"""Cases for the two-team instance of the 1x1 / im2col kernel (csrc/conv_sm90.cu, conv_wgmma_team_kernel): 1x1 / s1
convolutions with a 128-column N tile of resident weights over whole 64-channel K chunks, chained to a 64-column tail
over one or two 64-channel boxes, run on one CTA of two consumer teams of two warpgroups when the launch has at least
8 tiles per SM (yb_conv_config: `consumer_groups` 4, layout "1x4", `chained` 1).

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py and are sized from the device's SM
count so that each lands on the side of the rule its name states ("team": two teams, "pair": two warpgroups).
"""
from conv_cases import BF16, F16, NONE, SMS, Case, Chain

MIN_TILES_PER_SM = 8


def images(px_per_image: int, odd: bool = False, S: int = SMS) -> int:
    """Images whose 128-row tiles just reach the threshold of 8 x S tiles (an odd tile count if `odd`)."""
    tiles = lambda n: -(-n * px_per_image // 128)  # noqa: E731
    n = 1
    while tiles(n) < MIN_TILES_PER_SM * S or (odd and tiles(n) % 2 == 0):
        n += 1
    return n


def _cases():
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # c2's body.4.cv1+cv2 -> body.4.m.0.cv1: two K chunks, the first output stored, a one-box tail operand
            Case(f"{b} team 1x1 128->[64]->64", images(80 * 80), 80, 80, 128, 128, dtype=dt, seed=501,
                 chain=Chain(64, 64)),
            # c2's pan.layer_blocks.0.cv1+cv2 -> m.0.cv1: four K chunks; ragged M, an odd tile count (one team runs
            # one tile more), the first output not stored
            Case(f"{b} team 1x1 256->[64]->64 sf0 ragged odd", images(40 * 40, odd=True), 40, 40, 256, 128,
                 dtype=dt, seed=502, chain=Chain(64, 64, store_first=False)),
            # a two-box tail operand, a shortcut on the first output, an input window, a 56-column linear tail
            Case(f"{b} team 1x1 64->[128]->56 resid in-window", images(16 * 8), 16, 8, 64, 128, dtype=dt, seed=503,
                 residual=True, in_cstride=128, in_off=64, chain=Chain(128, 56, act2=NONE)),
            # one tile fewer than the threshold: two consumer warpgroups
            Case(f"{b} pair 1x1 128->[64]->64 below", MIN_TILES_PER_SM * SMS - 1, 16, 8, 128, 128, dtype=dt,
                 seed=504, chain=Chain(64, 64)),
        ]
    return C


CASES = _cases()
