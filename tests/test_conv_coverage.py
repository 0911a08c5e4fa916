"""The case tables of the fp16/bf16 convolution kernels (tests/conv_cases.py and tests/conv_cases_*.py) reach every kernel
instance and every plan path, and every launch variant keeps to its own table (host logic, no GPU needed; SM-dependent
sizes follow the device's SM count, 132 without a GPU).

The instance list comes from the kernel selectors' source, so a new instance fails this test until a case reaches it.
"""
import conv_cases
import conv_cases_one_group
import conv_cases_quad
import conv_cases_quad_1x1
import conv_cases_tail_split
import conv_cases_team
import conv_cases_team_1x1
from conv_cases import EXCLUDED, SMS, VARIANTS, build_desc, check_pinned, config, fake_ptr, instance_key, plan_paths, \
    selector_instances, variants
from yolort_b200 import _C

TABLES = (conv_cases, conv_cases_one_group, conv_cases_quad, conv_cases_quad_1x1, conv_cases_tail_split, conv_cases_team,
          conv_cases_team_1x1)

# The tables whose cases may take each variant: a case of any other table that takes it has moved off the launch its
# table is about.
REACHED_BY = {
    "2x2": {conv_cases},
    "2x1": {conv_cases_one_group, conv_cases_tail_split},
    "split tail": {conv_cases_one_group, conv_cases_quad_1x1, conv_cases_tail_split},
    "patch quad": {conv_cases_quad},
    "patch team": {conv_cases_team},
    "1x1 team": {conv_cases_team_1x1},
    "1x1 quad": {conv_cases_quad_1x1},
}
assert set(REACHED_BY) == set(VARIANTS)

REQUIRED_PATHS = {
    # 1x1 / im2col kernel
    "conv 1x1 resident", "conv 1x1 streamed",
    "conv im2col 3x3 s1 resident", "conv im2col 3x3 s1 streamed",
    "conv im2col 3x3 s2 resident", "conv im2col 3x3 s2 streamed",
    "conv several N tiles", "conv im2col k5",
    # halo-patch kernel
    "patch classic", "patch wrap", "patch stride2",
    "patch resident single N tile", "patch resident N-split", "patch streamed pairs", "patch streamed odd last pair",
    # two CTAs per SM
    "two CTAs conv", "two CTAs patch classic", "two CTAs patch wrap", "two CTAs patch stride2",
    "two CTAs at 2 x SMs tiles", "one CTA at 2 x SMs - 1 tiles",
    # chained tails
    "chain one own chunk", "chain two own chunks", "chain extra operand", "chain store_first=0",
}


def _plans(tables=TABLES):
    for table in tables:
        for c in table.CASES:
            d, _ch = build_desc(c, fake_ptr)
            cfg = _C.conv_config(d)
            yield table, c, instance_key(c, d, cfg), cfg


def test_case_names_are_unique():
    names = [c.name for _, c, _, _ in _plans()]
    assert len(names) == len(set(names)), sorted(n for n in set(names) if names.count(n) > 1)


def test_every_instance_is_reached():
    inst = selector_instances()
    assert len(inst) == 68, sorted(inst)      # the patterns still match the selectors (34 instances per dtype today)
    reached = {}
    for _, c, key, _ in _plans():
        reached.setdefault(key, []).append(c.name)
    unknown = set(reached) - inst
    assert not unknown, f"cases planned onto instances the selectors do not list: {sorted(unknown)}"
    assert set(EXCLUDED) <= inst and not set(EXCLUDED) & set(reached)
    missing = inst - set(reached) - set(EXCLUDED)
    print(f"instance coverage: {len(inst & set(reached))} / {len(inst)} reached, {len(EXCLUDED)} excluded "
          f"({SMS} SMs)")
    for key in sorted(inst, key=str):
        print(f"  {key}: {reached[key][0] + (f' (+{len(reached[key]) - 1})' if len(reached[key]) > 1 else '') if key in reached else 'EXCLUDED: ' + EXCLUDED.get(key, 'MISSING')}")
    assert not missing, f"no case reaches {sorted(missing)}"


def test_every_plan_path_is_reached():
    seen = {}
    for _, c, _, cfg in _plans([conv_cases]):
        for p in plan_paths(c, cfg):
            seen.setdefault(p, c.name)
    for p in sorted(REQUIRED_PATHS):
        print(f"  {p}: {seen.get(p, 'MISSING')}")
    assert REQUIRED_PATHS <= set(seen), sorted(REQUIRED_PATHS - set(seen))


def test_variants_stay_in_their_tables():
    """Every variant is taken by a case of each table listed for it, and by no case of another table."""
    takers = {}
    for table, c, _, cfg in _plans():
        for v in variants(cfg):
            assert table in REACHED_BY[v], (v, table.__name__, c.name)
            takers.setdefault(v, set()).add(table)
    assert takers == REACHED_BY, {v: sorted(t.__name__ for t in ts) for v, ts in takers.items()}


def test_pinning_bits_give_the_reference_launch():
    """Each bit of a variant plans every case that takes it on the launch the variant names, with the same tiling."""
    for _, c, _, cfg in _plans():
        for v in variants(cfg):
            for bit in VARIANTS[v].bits:
                check_pinned(config(c, bit), cfg, v, bit, c.name)


def test_two_cta_threshold_at_2x_sms_tiles():
    """The same 1x1 layer plans two CTAs per SM at exactly 2 x SMs tiles and one CTA at one tile fewer."""
    by_name = {c.name: c for c in conv_cases.CASES}
    for dt in ("f16", "bf16"):
        for name, ctas, grid in ((f"{dt} 2cta 1x1 Cout32 at 2xSMs", 2, 2 * SMS), (f"{dt} 1cta 1x1 Cout32 at 2xSMs-1", 1, SMS)):
            c = by_name[name]
            d, _ = build_desc(c, fake_ptr)
            cfg = _C.conv_config(d)
            assert (cfg["ctas_per_sm"], cfg["grid"]) == (ctas, grid), (name, cfg)
