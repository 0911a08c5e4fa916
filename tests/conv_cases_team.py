"""Cases for the two-team instance of the halo-patch kernel (csrc/conv3x3_patch_sm90.cu, conv3x3_patch_team_kernel):
stride-1 3x3 convolutions with resident weights in one N tile and classic single-tile tasks, chained after a 64-column
N tile over whole 64-channel chunks, run on one CTA of two consumer teams of two warpgroups when the launch has at
least 8 tasks per SM (yb_conv_config: `groups` 4, `tiles_per_pass` 1, `chained` 1).  The banded stem's team instance
needs the stem's band weights; tests/test_gpu_conv_team.py covers it through the yolov5s plan.

The cases use the Case / build_desc / check_case machinery of tests/conv_cases.py and are sized from the device's SM
count so that each lands on the side of the rule its name states ("team": two teams, "pair": two warpgroups).
"""
from conv_cases import BF16, F16, NONE, SMS, Case, Chain

MIN_TASKS_PER_SM = 8


def images(tiles_per_image: int, odd: bool = False, S: int = SMS) -> int:
    """Images whose tiles just reach the threshold of 8 x S tasks (an odd task count if `odd`)."""
    n = -(-MIN_TASKS_PER_SM * S // tiles_per_image)
    if odd and (n * tiles_per_image) % 2 == 0:
        n += 1
    return n


def _cases():
    C = []
    for dt in (F16, BF16):
        b = "bf16" if dt == BF16 else "f16"
        C += [
            # c2's body.4.m.0.cv2 -> body.4.m.1.cv1: shortcut, the first output stored, a 64-column tail
            Case(f"{b} team 80x80 64->[64]->64 residual", images(50), 80, 80, 64, 64, k=3, dtype=dt, seed=401,
                 residual=True, chain=Chain(64, 64)),
            # c2's body.4.m.1.cv2 -> body.4.cv3: the extra operand (cv2 half of the concat), first output not stored
            Case(f"{b} team 80x80 64->[64]->128 extra sf0", images(50), 80, 80, 64, 64, k=3, dtype=dt, seed=402,
                 residual=True, chain=Chain(64, 128, extra=True, store_first=False)),
            # ragged tiles, an odd task count (one team runs one task more), a 120-column tail, an input window
            Case(f"{b} team 76x84 64->[64]->120 extra ragged odd", images(55, odd=True), 76, 84, 64, 64, k=3,
                 dtype=dt, seed=403, act=NONE, in_cstride=96, in_off=32, chain=Chain(64, 120, extra=True)),
            # one task per SM fewer than the threshold: two consumer warpgroups
            Case(f"{b} pair 16x8 64->[64]->64 below", MIN_TASKS_PER_SM * SMS - 1, 16, 8, 64, 64, k=3, dtype=dt,
                 seed=404, chain=Chain(64, 64)),
        ]
    return C


CASES = _cases()
