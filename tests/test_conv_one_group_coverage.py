"""The one-consumer-warpgroup instances of the 1x1 / im2col kernel are all reached, and the rule that selects the layout
holds at its edges (host logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132 without a GPU).

Launches that now run the one-group layout report the same (N tile, tail, ctas_per_sm) as the one-CTA instance they
replaced, so this test also checks that every older instance is still reached by a case of tests/conv_cases.py that is
planned off the new layout.
"""
import os
import re

import conv_cases
import conv_cases_one_group as og
from conv_cases import build_desc, fake_ptr, instance_key
from yolort_b200 import _C

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolort_b200", "csrc")

REQUIRED_PATHS = {
    "2x1 1x1 resident", "2x1 im2col", "2x1 ragged second N tile", "2x1 ragged M", "2x1 at 3 x SMs 128-row tiles",
    "1x2 at 3 x SMs - 1 128-row tiles", "1x2 streamed weights", "1x2 N = 128",
}


def _selector():
    with open(os.path.join(CSRC, "conv_sm90.cu")) as f:
        return f.read()


def one_group_instances() -> set:
    """Every (kernel, dtype, N, decode, tail N, layout) of the one-group branch of select_conv_kernel_t."""
    src = _selector()
    out = set()
    for dt in ("f16", "bf16"):
        for m in re.finditer(r"conv_wgmma_kernel<kBf16, (\d+), false, (\d+), 2, 1>", src):
            out.add(("conv", dt, int(m[1]), False, int(m[2]), "2x1"))
    return out


def older_instances() -> set:
    """The 1x1 / im2col instances the older spelling names (the pattern of tests/test_conv_coverage.py)."""
    src = _selector()
    return {("conv", dt, int(m[1]), m[2] == "true", int(m[3]), int(m[4]))
            for dt in ("f16", "bf16")
            for m in re.finditer(r"conv_wgmma_kernel<kBf16, (\d+), (true|false), (\d+), (\d+)>", src)}


def _plan(c):
    d, _ch = build_desc(c, fake_ptr)
    return d, _C.conv_config(d)


def test_case_names_are_unique():
    names = [c.name for c in og.CASES]
    assert len(names) == len(set(names)) and not set(names) & {c.name for c in conv_cases.CASES}


def test_every_one_group_instance_is_reached():
    inst = one_group_instances()
    assert len(inst) == 2, sorted(inst)       # N = 128, f16 and bf16
    reached = {}
    for c in og.CASES + conv_cases.CASES:
        d, cfg = _plan(c)
        if cfg["layout"] == "2x1":
            assert cfg["epilogue_groups"] == 1 and cfg["resident_ctas"] == 2 and cfg["ctas_per_sm"] == 1, (c.name, cfg)
            assert cfg["weights_resident"] == 1 and cfg["grid"] == 2 * og.SMS, (c.name, cfg)
            reached.setdefault(og.one_group_key(c, d, cfg), []).append(c.name)
    for key in sorted(inst):
        print(f"  {key}: {reached.get(key, 'MISSING')}")
    assert set(reached) <= inst, sorted(set(reached) - inst)
    assert inst <= set(reached), sorted(inst - set(reached))


def test_every_plan_path_is_reached():
    seen = {}
    for c in og.CASES:
        _, cfg = _plan(c)
        for p in og.one_group_paths(c, cfg):
            seen.setdefault(p, c.name)
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: {seen.get(p, 'MISSING')}")
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))


def test_cases_take_the_layout_their_name_states():
    for c in og.CASES:
        _, cfg = _plan(c)
        assert cfg["layout"] == c.name.split()[1], (c.name, cfg)


def test_older_instances_are_reached_off_the_new_layout():
    """Every older instance is reached by a case of tests/conv_cases.py as actually planned (layout not 2x1)."""
    inst = older_instances()
    reached = {}
    for c in conv_cases.CASES:
        d, cfg = _plan(c)
        if cfg["layout"] != "2x1":
            reached.setdefault(instance_key(c, d, cfg), []).append(c.name)
    missing = inst - set(reached) - set(conv_cases.EXCLUDED)
    assert not missing, sorted(missing)


def test_keep_one_cta_bit_gives_the_two_group_layout():
    """Reserved bit 4 plans every one-group case on one CTA of two consumer warpgroups with one 256-column N tile."""
    for c in og.CASES:
        _, cfg = _plan(c)
        if cfg["layout"] != "2x1":
            continue
        d1, _ch = build_desc(c, fake_ptr)
        d1.reserved |= _C.YB_CONV_ONE_CTA
        one = _C.conv_config(d1)
        assert one["layout"] == "1x2" and one["epilogue_groups"] == 2 and one["grid"] <= og.SMS, (c.name, one)
        assert (cfg["block_n"], cfg["n_tiles"], one["block_n"], one["n_tiles"]) == (128, 2, 256, 1), (c.name, one)


def test_threshold_at_3x_sms_128_row_tiles():
    """The same 64 -> 256 layer plans the one-group layout at exactly 3 x SMs 128-row tiles and one CTA at one fewer."""
    by_name = {c.name: c for c in og.CASES}
    for dt in ("f16", "bf16"):
        for name, layout, grid in ((f"{dt} 2x1 1x1 64->256 at 3xSMs tiles", "2x1", 2 * og.SMS),
                                   (f"{dt} 1x2 1x1 64->256 at 3xSMs-1 tiles", "1x2", og.SMS)):
            _, cfg = _plan(by_name[name])
            assert (cfg["layout"], cfg["grid"]) == (layout, grid), (name, cfg)
