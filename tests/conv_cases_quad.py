"""Cases for the four-consumer-warpgroup instance of the halo-patch kernel (csrc/conv3x3_patch_sm90.cu,
conv3x3_patch_quad_kernel): stride-1 3x3 convolutions with streamed weights, run as pairs of M tiles times one
128-column N tile when Cout splits into 128-column N tiles, the grid is a multiple of them and the wider tasks cost no
extra round of the persistent grid (T >= G tasks on G CTAs with T mod G = 0 or T mod G > G / 2; yb_conv_config:
`groups` 4).

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py and are sized from the device's SM
count so that each lands on the side of the rule its name states ("quad": four consumer warpgroups, "pairs64": the
64-column pairs of two).
"""
from conv_cases import BF16, F16, LEAKY, NONE, SMS, Case


def images(tiles_per_image: int, n_tiles: int, S: int = SMS) -> int:
    """Images whose pair tasks just pass one and a half grids: T = ceil(tiles / 2) * n_tiles a little above 3S / 2."""
    n = 1
    while ((n * tiles_per_image + 1) // 2) * n_tiles <= S + S // 2 + 1:
        n += 1
    return n


def _cases():
    S = SMS
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # 40² classic tiles (15 per image, the last tile row ragged), residual in a channel window
            Case(f"{b} quad classic 40x40 128->128 residual", images(15, 1), 40, 40, 128, 128, k=3, dtype=dt, seed=301,
                 residual=True, res_cstride=192, res_off=64),
            # wrap tiles (20², 4 per image), two 128-column N tiles: 4 x (S/2 - 1) tasks
            Case(f"{b} quad wrap 20x20 256->256", S // 2 - 1, 20, 20, 256, 256, k=3, dtype=dt, seed=302, act=LEAKY,
                 bias_scale=1.0),
            # wrap tiles with an odd tile count: the last pair holds one tile; residual on the second N tile too
            Case(f"{b} quad wrap 23x20 odd last pair 128->256 residual", 2 * (images(5, 2) // 2) + 1, 23, 20, 128, 256,
                 k=3, dtype=dt, seed=303, residual=True),
            # in-window input and output channel strides
            Case(f"{b} quad classic 40x48 128->128 windows", images(18, 1), 40, 48, 128, 128, k=3, dtype=dt, seed=304,
                 act=NONE, in_cstride=256, in_off=64, out_cstride=256, out_off=128),
            # Cout not a multiple of 128: the 64-column pairs of two warpgroups
            Case(f"{b} pairs64 classic 40x40 128->192", images(15, 2), 40, 40, 128, 192, k=3, dtype=dt, seed=305),
            # fewer 128-column tasks than CTAs (c2's 20² level): the 64-column pairs
            Case(f"{b} pairs64 wrap 20x20 256->256 below a grid", S // 4 - 1, 20, 20, 256, 256, k=3, dtype=dt, seed=307),
            # too few tasks for half a grid: the 64-column pairs
            Case(f"{b} pairs64 classic 40x40 128->128 few tasks", 4, 40, 40, 128, 128, k=3, dtype=dt, seed=306),
        ]
    return C


CASES = _cases()
