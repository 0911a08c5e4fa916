"""The two-team instance of the halo-patch kernel: the cases take the path their names state and reach an odd task
count, the rule holds on both sides of its task threshold, and the plans fit in shared memory (host logic, no GPU
needed; SM-dependent sizes follow the device's SM count, 132 without a GPU).  Instance coverage, the pinning bits and
the other tables are checked in tests/test_conv_coverage.py."""
import conv_cases_team as t
from conv_cases import BF16, F16, SMS, VARIANTS, Case, Chain, config

_is_team = VARIANTS["patch team"].takes


def test_cases_take_the_path_their_name_states():
    for c in t.CASES:
        cfg = config(c)
        team = c.name.split()[1] == "team"
        assert cfg["patch_kernel"] and cfg["chained"] and cfg["weights_resident"] and cfg["n_tiles"] == 1, (c.name, cfg)
        assert cfg["patch_tiling"] == "classic" and cfg["block_n"] == 64, (c.name, cfg)
        assert _is_team(cfg) == team, (c.name, cfg)
        assert cfg["layout"] == ("1x4" if team else "1x2"), (c.name, cfg)
        if team:
            assert cfg["work_items"] >= t.MIN_TASKS_PER_SM * SMS and cfg["grid"] == SMS, (c.name, cfg)


def test_every_instance_is_reached():
    """An odd task count (one team runs one task more) in each dtype."""
    odd = {c.dtype for c in t.CASES if _is_team(config(c)) and config(c)["work_items"] % 2}
    assert odd == {F16, BF16}


def test_threshold_edges():
    """Two teams exactly from 8 x SMs tasks on (1-tile images, so tasks = images)."""
    for dt in (F16, BF16):
        for chain in (Chain(64, 64), Chain(64, 128, extra=True)):
            for T in (SMS, 4 * SMS, 8 * SMS - 1, 8 * SMS, 8 * SMS + 1, 20 * SMS):
                cfg = config(Case("edge", T, 16, 8, 64, 64, k=3, dtype=dt, chain=chain))
                assert cfg["work_items"] == T
                assert _is_team(cfg) == (T >= 8 * SMS), (T, chain, cfg)


def test_shared_memory_fit():
    """Each team plan fits 227 KB less the kernel's static shared memory with an even number of patch slots, so that
    every slot serves one team only (each team's parity waits then follow its own fills): the c2 chains take two slots
    next to a 64-column tail (195 584 B; a third would fit but would alternate between the teams) and next to a
    128-column one (220 160 B)."""
    for c in t.CASES:
        cfg = config(c)
        if _is_team(cfg):
            assert cfg["slots"] in (2, 4) and cfg["smem_bytes"] <= 227 * 1024 - 1120, (c.name, cfg)
    assert [(config(c)["slots"], config(c)["smem_bytes"]) for c in t.CASES[:2]] == [(2, 195584), (2, 220160)]


def test_other_shapes_stay():
    """Chains after 32-column N tiles, chains over a partial 64-channel chunk and tails over 32-channel chunks never
    take two teams."""
    for c in (Case("n32", 8 * SMS, 16, 8, 32, 32, k=3, chain=Chain(32, 64)),
              Case("cin48", 8 * SMS, 16, 8, 48, 64, k=3, chain=Chain(64, 64)),
              Case("kc32", 8 * SMS, 16, 8, 64, 64, k=3, chain=Chain(32, 64))):
        cfg = config(c)
        assert cfg["chained"] and not _is_team(cfg), (c.name, cfg)
