"""Cases for the four-consumer-warpgroup instance of the 1x1 / im2col kernel (csrc/conv_sm90.cu,
conv_wgmma_quad_kernel): 1x1 / s1 and stride-2 3x3 convolutions that stream their weights in 128-column N tiles over
whole 64-channel K chunks run as tasks of two consecutive 128-row M tiles sharing each weight slab (yb_conv_config:
`consumer_groups` 4, layout "1x4x2", `tiles_per_pass` 2) when they have at least 100 M tiles and either at most one per
SM, three or more N tiles, or at least 400 M tiles, and the grid is a multiple of the N tiles.

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py and are sized from the device's SM
count so that each lands on the side of the rule its name states ("quad": two-tile tasks on four warpgroups, "pair":
the two-warpgroup launch).
"""
from conv_cases import BF16, F16, LEAKY, NONE, SMS, Case

MIN_M_TILES = 100
WIDE_M_TILES = 400


def images(px_per_image: int, lo: int, odd: bool = False, ragged: bool = False) -> int:
    """The fewest images with at least `lo` 128-row M tiles (an odd count if `odd`, a partial last tile if `ragged`)."""
    n = 1
    while True:
        rows = n * px_per_image
        tiles = -(-rows // 128)
        if tiles >= lo and (not odd or tiles % 2 == 1) and (not ragged or rows % 128 != 0):
            return n
        n += 1


def _cases():
    S = SMS
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # c2's body.8 cv3: four N tiles, 100 M tiles, two rounds of pairs
            Case(f"{b} quad 1x1 512->512 four N tiles", images(400, MIN_M_TILES), 20, 20, 512, 512, dtype=dt, seed=601),
            # one M tile per SM at most, two N tiles, an odd tile count with a partial last tile (team 1 idle in the last
            # pair), an input and an output channel window
            Case(f"{b} quad 1x1 256->256 odd ragged windows", images(19 * 19, MIN_M_TILES, odd=True, ragged=True), 19, 19,
                 256, 256, dtype=dt, seed=602, act=LEAKY, in_cstride=384, in_off=64, out_cstride=320, out_off=64),
            # one N tile, an odd tile count, no activation
            Case(f"{b} quad 1x1 384->128 one N tile odd", images(21 * 21, MIN_M_TILES, odd=True), 21, 21, 384, 128,
                 dtype=dt, seed=603, act=NONE),
            # mode 1: c2's body.7, a stride-2 3x3 over the 4-D im2col map, four N tiles
            Case(f"{b} quad 3x3 s2 256->512", images(400, MIN_M_TILES), 40, 40, 256, 512, k=3, s=2, dtype=dt, seed=604),
            # mode 1 with an odd, partial last tile on one N tile
            Case(f"{b} quad 3x3 s2 128->128 odd ragged", images(11 * 11, MIN_M_TILES, odd=True, ragged=True), 22, 22, 128,
                 128, k=3, s=2, dtype=dt, seed=605),
            # one M tile too few: the two-warpgroup launch
            Case(f"{b} pair 1x1 512->512 below", images(400, MIN_M_TILES) - 1, 20, 20, 512, 512, dtype=dt, seed=606),
            # two N tiles, more M tiles than SMs but fewer than 400: the two-warpgroup launch
            Case(f"{b} pair 1x1 256->256 two N tiles past a round", images(400, S + 1), 20, 20, 256, 256, dtype=dt,
                 seed=607),
        ]
    return C


CASES = _cases()
