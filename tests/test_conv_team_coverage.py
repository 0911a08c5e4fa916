"""The two-team instance of the halo-patch kernel: every instance is reached, the cases take the path their names state,
the rule holds on both sides of its task threshold, the plans fit in shared memory, and the reserved bit keeps two
consumer warpgroups (host logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132 without a GPU)."""
import os
import re

import conv_cases
import conv_cases_team as t
from conv_cases import BF16, F16, SMS, Case, Chain, build_desc, fake_ptr
from yolort_b200 import _C

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolort_b200", "csrc")

# instances no case of the table reaches: the banded stem needs band weights (engine.stem_band)
EXCLUDED = {(dt, 128, 0): "tests/test_gpu_conv_team.py::test_team_launches_match_two_warpgroups_bit_for_bit[yolov5s]"
            for dt in ("f16", "bf16")}


def _plan(c, extra=0):
    d, _ch = build_desc(c, fake_ptr)
    d.reserved |= extra
    return _C.conv_config(d)


def team_instances() -> set:
    with open(os.path.join(CSRC, "conv3x3_patch_sm90.cu")) as f:
        src = f.read()
    return {(dt, int(m[1]), int(m[2])) for dt in ("f16", "bf16")
            for m in re.finditer(r"conv3x3_patch_team_kernel<kBf16, (\d+), (\d+)>", src)}


def _is_team(cfg) -> bool:
    return cfg["patch_kernel"] == 1 and cfg["consumer_groups"] == 4 and cfg["tiles_per_pass"] == 1


def test_case_names_are_unique():
    names = [c.name for c in t.CASES]
    assert len(names) == len(set(names))
    assert not set(names) & {c.name for c in conv_cases.CASES}


def test_cases_take_the_path_their_name_states():
    for c in t.CASES:
        cfg = _plan(c)
        team = c.name.split()[1] == "team"
        assert cfg["patch_kernel"] and cfg["chained"] and cfg["weights_resident"] and cfg["n_tiles"] == 1, (c.name, cfg)
        assert cfg["patch_tiling"] == "classic" and cfg["block_n"] == 64, (c.name, cfg)
        assert _is_team(cfg) == team, (c.name, cfg)
        assert cfg["layout"] == ("1x4" if team else "1x2"), (c.name, cfg)
        if team:
            assert cfg["work_items"] >= t.MIN_TASKS_PER_SM * SMS and cfg["grid"] == SMS, (c.name, cfg)


def test_every_instance_is_reached():
    inst = team_instances()
    assert len(inst) == 6, sorted(inst)
    reached = {("bf16" if c.dtype == BF16 else "f16", _plan(c)["block_n"], _plan(c)["tail_n"])
               for c in t.CASES if _is_team(_plan(c))}
    assert reached == inst - set(EXCLUDED), sorted(reached)
    assert set(EXCLUDED) <= inst
    odd = {c.dtype for c in t.CASES if _is_team(_plan(c)) and _plan(c)["work_items"] % 2}
    assert odd == {F16, BF16}


def test_reserved_bits_keep_two_warpgroups():
    """YB_CONV_NO_TEAMS, and YB_CONV_PAIR_N64 (the two-warpgroup launch of every four-warpgroup one), keep the same
    tiling on two consumer warpgroups."""
    for c, bit in ((c, bit) for c in t.CASES for bit in (_C.YB_CONV_NO_TEAMS, _C.YB_CONV_PAIR_N64)):
        cfg = _plan(c, bit)
        assert cfg["consumer_groups"] == 2 and cfg["layout"] == "1x2", (c.name, cfg)
        team = _plan(c)
        for k in ("block_n", "n_tiles", "weights_resident", "tiles_per_pass", "store_cols", "chained", "tail_n",
                  "grid", "m_tiles", "work_items"):
            assert cfg[k] == team[k], (c.name, k, cfg, team)


def test_threshold_edges():
    """Two teams exactly from 8 x SMs tasks on (1-tile images, so tasks = images)."""
    for dt in (F16, BF16):
        for chain in (Chain(64, 64), Chain(64, 128, extra=True)):
            for T in (SMS, 4 * SMS, 8 * SMS - 1, 8 * SMS, 8 * SMS + 1, 20 * SMS):
                cfg = _plan(Case("edge", T, 16, 8, 64, 64, k=3, dtype=dt, chain=chain))
                assert cfg["work_items"] == T
                assert _is_team(cfg) == (T >= 8 * SMS), (T, chain, cfg)


def test_shared_memory_fit():
    """Each team plan fits 227 KB less the kernel's static shared memory with an even number of patch slots, so that
    every slot serves one team only (each team's parity waits then follow its own fills): the c2 chains take two slots
    next to a 64-column tail (195 584 B; a third would fit but would alternate between the teams) and next to a
    128-column one (220 160 B)."""
    for c in t.CASES:
        cfg = _plan(c)
        if _is_team(cfg):
            assert cfg["slots"] in (2, 4) and cfg["smem_bytes"] <= 227 * 1024 - 1120, (c.name, cfg)
    assert [(_plan(c)["slots"], _plan(c)["smem_bytes"]) for c in t.CASES[:2]] == [(2, 195584), (2, 220160)]


def test_other_shapes_stay():
    """Chains after 32-column N tiles, chains over a partial 64-channel chunk, tails over 32-channel chunks, and the
    other tables' cases never take two teams."""
    for c in (Case("n32", 8 * SMS, 16, 8, 32, 32, k=3, chain=Chain(32, 64)),
              Case("cin48", 8 * SMS, 16, 8, 48, 64, k=3, chain=Chain(64, 64)),
              Case("kc32", 8 * SMS, 16, 8, 64, 64, k=3, chain=Chain(32, 64))):
        cfg = _plan(c)
        assert cfg["chained"] and not _is_team(cfg), (c.name, cfg)
    for c in conv_cases.CASES:
        assert not _is_team(_plan(c)), c.name
