"""The two-team instance of the 1x1 / im2col kernel: every instance is reached, the cases take the path their names
state, the rule holds on both sides of its tile threshold, the plans fit in shared memory, and the reserved bits keep
the one-CTA tiling on two consumer warpgroups (host logic, no GPU needed; SM-dependent sizes follow the device's SM
count, 132 without a GPU)."""
import os
import re

import conv_cases
import conv_cases_one_group
import conv_cases_team_1x1 as t
from conv_cases import BF16, F16, SMS, Case, Chain, build_desc, fake_ptr
from yolort_b200 import _C

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolort_b200", "csrc")
STATIC_SMEM = 976     # ptxas -v of conv_wgmma_team_kernel


def _plan(c, extra=0):
    d, _ch = build_desc(c, fake_ptr)
    d.reserved |= extra
    return _C.conv_config(d)


def team_instances() -> set:
    with open(os.path.join(CSRC, "conv_sm90.cu")) as f:
        src = f.read()
    return {(dt, int(m[1]), int(m[2])) for dt in ("f16", "bf16")
            for m in re.finditer(r"conv_wgmma_team_kernel<kBf16, (\d+), (\d+)>", src)}


def _is_team(cfg) -> bool:
    return not cfg["patch_kernel"] and cfg["consumer_groups"] == 4 and cfg["layout"] == "1x4"


def test_case_names_are_unique():
    names = [c.name for c in t.CASES]
    assert len(names) == len(set(names))
    assert not set(names) & {c.name for c in conv_cases.CASES}


def test_cases_take_the_path_their_name_states():
    for c in t.CASES:
        cfg = _plan(c)
        team = c.name.split()[1] == "team"
        assert not cfg["patch_kernel"] and cfg["chained"] and cfg["weights_resident"] and cfg["n_tiles"] == 1, (c.name, cfg)
        assert cfg["block_n"] == 128 and cfg["tail_n"] == 64 and cfg["tiles_per_pass"] == 1, (c.name, cfg)
        assert _is_team(cfg) == team, (c.name, cfg)
        assert cfg["layout"] == ("1x4" if team else "1x2"), (c.name, cfg)
        if team:
            assert cfg["work_items"] >= t.MIN_TILES_PER_SM * SMS and cfg["grid"] == SMS, (c.name, cfg)
            assert cfg["ring"] == 1, (c.name, cfg)


def test_every_instance_is_reached():
    inst = team_instances()
    assert inst == {("f16", 128, 64), ("bf16", 128, 64)}, sorted(inst)
    reached = {("bf16" if c.dtype == BF16 else "f16", _plan(c)["block_n"], _plan(c)["tail_n"])
               for c in t.CASES if _is_team(_plan(c))}
    assert reached == inst, sorted(reached)
    team = [c for c in t.CASES if _is_team(_plan(c))]
    for dt in (F16, BF16):
        parities = {_plan(c)["work_items"] % 2 for c in team if c.dtype == dt}
        assert parities == {0, 1}, dt
        assert {c.chain.c_own for c in team if c.dtype == dt} == {64, 128}, dt        # one- and two-box tail operands
        assert {c.chain.store_first for c in team if c.dtype == dt} == {True, False}, dt


def test_reserved_bits_keep_the_one_cta_tiling():
    """YB_CONV_NO_TEAMS, YB_CONV_ONE_CTA and YB_CONV_PAIR_N64 (the two-warpgroup launch of every four-warpgroup one)
    keep the tiling of the team plan on two consumer warpgroups."""
    for c, bit in ((c, bit) for c in t.CASES
                   for bit in (_C.YB_CONV_NO_TEAMS, _C.YB_CONV_ONE_CTA, _C.YB_CONV_PAIR_N64)):
        cfg = _plan(c, bit)
        assert cfg["consumer_groups"] == 2 and cfg["layout"] == "1x2", (c.name, cfg)
        team = _plan(c)
        for k in ("block_n", "n_tiles", "weights_resident", "tiles_per_pass", "store_cols", "chained", "tail_n",
                  "grid", "m_tiles", "work_items", "tail_tiles", "tail_split"):
            assert cfg[k] == team[k], (c.name, k, cfg, team)


def test_threshold_edges():
    """Two teams exactly from 8 x SMs tiles on (one 128-pixel tile per image, so tiles = images)."""
    for dt in (F16, BF16):
        for cin, chain in ((128, Chain(64, 64)), (256, Chain(64, 64, store_first=False)), (64, Chain(128, 64))):
            for T in (SMS, 4 * SMS, 8 * SMS - 1, 8 * SMS, 8 * SMS + 1, 20 * SMS):
                cfg = _plan(Case("edge", T, 16, 8, cin, 128, dtype=dt, chain=chain))
                assert cfg["work_items"] == T
                assert _is_team(cfg) == (T >= 8 * SMS), (T, cin, chain, cfg)


def test_shared_memory_fit():
    """Each team plan fits 227 KB less the kernel's static shared memory with at least two 16 KB A stages per team:
    c2's op 5 (32 KB of weights) takes three per team, op 33 (64 KB of weights) two, both in 205 824 B."""
    for c in t.CASES:
        cfg = _plan(c)
        if _is_team(cfg):
            assert 2 <= cfg["slots"] <= 6 and cfg["smem_bytes"] <= 227 * 1024 - STATIC_SMEM, (c.name, cfg)
    assert [(_plan(c)["slots"], _plan(c)["smem_bytes"]) for c in t.CASES[:2]] == [(3, 205824), (2, 205824)]


def test_other_shapes_stay():
    """Chains after 64-column N tiles, 128-column tails, K chunks of 32 channels, unchained 1x1 launches, and the cases
    of the other tables never take two teams."""
    for c in (Case("n64", 8 * SMS, 16, 8, 128, 64, chain=Chain(64, 128)),
              Case("tail128", 8 * SMS, 16, 8, 128, 128, chain=Chain(64, 128)),
              Case("tail32", 8 * SMS, 16, 8, 128, 128, chain=Chain(64, 32)),
              Case("cin96", 8 * SMS, 16, 8, 96, 128, chain=Chain(64, 64)),
              Case("plain", 8 * SMS, 16, 8, 128, 128)):
        assert not _is_team(_plan(c)), c.name
    for c in conv_cases.CASES + conv_cases_one_group.CASES:
        assert not _is_team(_plan(c)), c.name
