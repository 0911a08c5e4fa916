"""The rule that selects the one-consumer-warpgroup layout of the 1x1 / im2col kernel holds at its edges, and its cases
take the paths their names state (host logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132
without a GPU).  Instance coverage and the pinning bit are checked for every table in tests/test_conv_coverage.py."""
import conv_cases_one_group as og
from conv_cases import config
from yolort_b200 import _C

REQUIRED_PATHS = {
    "2x1 1x1 resident", "2x1 im2col", "2x1 ragged second N tile", "2x1 ragged M", "2x1 at 3 x SMs 128-row tiles",
    "1x2 at 3 x SMs - 1 128-row tiles", "1x2 streamed weights", "1x2 N = 128",
}


def test_every_plan_path_is_reached():
    seen = {}
    for c in og.CASES:
        for p in og.one_group_paths(c, config(c)):
            seen.setdefault(p, c.name)
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: {seen.get(p, 'MISSING')}")
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))


def test_cases_take_the_layout_their_name_states():
    for c in og.CASES:
        cfg = config(c)
        assert cfg["layout"] == c.name.split()[1], (c.name, cfg)
        if cfg["layout"] == "2x1":
            assert cfg["epilogue_groups"] == 1 and cfg["resident_ctas"] == 2 and cfg["ctas_per_sm"] == 1, (c.name, cfg)
            assert cfg["weights_resident"] == 1 and cfg["grid"] == 2 * og.SMS, (c.name, cfg)


def test_keep_one_cta_bit_gives_the_two_group_layout():
    """Reserved bit 4 plans every one-group case on one CTA of two consumer warpgroups with one 256-column N tile."""
    for c in og.CASES:
        cfg = config(c)
        if cfg["layout"] != "2x1":
            continue
        one = config(c, _C.YB_CONV_ONE_CTA)
        assert one["layout"] == "1x2" and one["epilogue_groups"] == 2 and one["grid"] <= og.SMS, (c.name, one)
        assert (cfg["block_n"], cfg["n_tiles"], one["block_n"], one["n_tiles"]) == (128, 2, 256, 1), (c.name, one)


def test_threshold_at_3x_sms_128_row_tiles():
    """The same 64 -> 256 layer plans the one-group layout at exactly 3 x SMs 128-row tiles and one CTA at one fewer."""
    by_name = {c.name: c for c in og.CASES}
    for dt in ("f16", "bf16"):
        for name, layout, grid in ((f"{dt} 2x1 1x1 64->256 at 3xSMs tiles", "2x1", 2 * og.SMS),
                                   (f"{dt} 1x2 1x1 64->256 at 3xSMs-1 tiles", "1x2", og.SMS)):
            cfg = config(by_name[name])
            assert (cfg["layout"], cfg["grid"]) == (layout, grid), (name, cfg)
