"""The four-warpgroup instance of the 1x1 / im2col kernel (two-tile tasks over one streamed weight slab): the cases take
the path their names state and cover its shapes, the rule holds on both sides of each of its edges, and the plans fit in
shared memory (host logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132 without a GPU).  Instance
coverage, the YB_CONV_PAIR_N64 launch and the other tables are checked in tests/test_conv_coverage.py."""
import conv_cases_quad_1x1 as t
from conv_cases import BF16, F16, SMS, VARIANTS, Case, config
from yolort_b200 import _C

STATIC_SMEM = 704     # ptxas -v of conv_wgmma_quad_kernel
STAGE_BYTES = 3 * 16384
STAGING_BYTES = 4 * 16384


_is_quad = VARIANTS["1x1 quad"].takes


def test_cases_take_the_path_their_name_states():
    for c in t.CASES:
        cfg = config(c)
        quad = c.name.split()[1] == "quad"
        assert not cfg["patch_kernel"] and not cfg["weights_resident"] and cfg["block_n"] == 128, (c.name, cfg)
        assert _is_quad(cfg) == quad, (c.name, cfg)
        assert cfg["layout"] == ("1x4x2" if quad else "1x2"), (c.name, cfg)
        if quad:
            T = (cfg["m_tiles"] + 1) // 2 * cfg["n_tiles"]
            assert cfg["grid"] == min(T, SMS) and cfg["grid"] % cfg["n_tiles"] == 0, (c.name, cfg)
            assert cfg["ring"] == 1 and cfg["tail_split"] == 1 and cfg["tail_tiles"] == 0, (c.name, cfg)


def test_every_instance_is_reached():
    """Both dtypes, modes 0 and 1, 1, 2 and 4 N tiles, odd tile counts and partial last tiles in each dtype."""
    quad = [c for c in t.CASES if _is_quad(config(c))]
    for dt in (F16, BF16):
        mine = [c for c in quad if c.dtype == dt]
        assert {(c.k, c.s) for c in mine} == {(1, 1), (3, 2)}, dt
        assert {config(c)["n_tiles"] for c in mine} == {1, 2, 4}, dt
        assert {config(c)["m_tiles"] % 2 for c in mine} == {0, 1}, dt
        assert any((c.N * c.Ho * c.Wo) % 128 for c in mine), dt
        assert any(config(c)["grid"] < SMS for c in mine) and any(config(c)["grid"] == SMS for c in mine), dt


def test_rule_edges():
    """At least 100 M tiles (one 128-pixel tile per image, so tiles = images), and then at most one per SM, three or
    more N tiles or at least 400 M tiles; the grid must be a multiple of the N tiles."""
    for dt in (F16, BF16):
        for cout in (128, 256, 512):
            n = cout // 128
            for m in (99, 100, 101, SMS, SMS + 1, 2 * SMS + 1, 399, 400, 401):
                cfg = config(Case("edge", m, 16, 8, 512, cout, dtype=dt))
                assert cfg["m_tiles"] == m and not cfg["weights_resident"], (m, cout, cfg)
                if cfg["block_n"] != 128:   # 256-column N tiles from 2 x SMs tiles of them on: no quad instance
                    assert not _is_quad(cfg), (m, cout, cfg)
                    continue
                assert cfg["n_tiles"] == n, (m, cout, cfg)
                T = (m + 1) // 2 * n
                G = min(T, SMS)
                want = m >= 100 and G % n == 0 and (m <= SMS or n >= 3 or m >= 400)
                assert _is_quad(cfg) == want, (m, cout, cfg)
        # five N tiles: 132 CTAs are not a multiple of them
        assert not _is_quad(config(Case("n5", 400, 16, 8, 512, 640, dtype=dt)))


def test_shapes_outside_the_instance_stay():
    """Residuals, K chunks of 32 channels, a partial last K chunk, 64- and 256-column N tiles and resident weights never
    take two-tile tasks."""
    for c in (Case("residual", 400, 16, 8, 512, 512, residual=True),
              Case("cin96", 400, 16, 8, 96, 512),
              Case("cin200", 400, 16, 8, 200, 512),
              Case("n64", 400, 16, 8, 512, 64),
              Case("resident", 400, 16, 8, 128, 128)):
        assert not _is_quad(config(c)), (c.name, config(c))


def test_shared_memory_fit():
    """Three stages of two 16 KB A sub-tiles and one 16 KB weight slab next to both teams' two 16 KB staging boxes, in
    227 KB less the kernel's static shared memory."""
    for c in t.CASES:
        cfg = config(c)
        if _is_quad(cfg):
            assert cfg["slots"] == 3, (c.name, cfg)
            assert cfg["smem_bytes"] == 3 * STAGE_BYTES + STAGING_BYTES + 1024 <= 227 * 1024 - STATIC_SMEM, (c.name, cfg)


def test_reserved_bits_keep_the_one_cta_plan():
    """YB_CONV_ONE_CTA keeps today's one-CTA plan (split tail included), YB_CONV_NO_TAIL_SPLIT the one-CTA plan of whole
    tiles: neither takes two-tile tasks; the N tiling stays that of the quad plan.  YB_CONV_NO_TEAMS changes nothing."""
    for c in t.CASES:
        quad = config(c)
        for bit in (_C.YB_CONV_ONE_CTA, _C.YB_CONV_NO_TAIL_SPLIT):
            cfg = config(c, bit)
            assert cfg["consumer_groups"] == 2 and cfg["layout"] == "1x2" and cfg["tiles_per_pass"] == 1, (c.name, cfg)
            for k in ("block_n", "n_tiles", "weights_resident", "store_cols", "m_tiles", "work_items"):
                assert cfg[k] == quad[k], (c.name, bit, k, cfg, quad)
        assert config(c, _C.YB_CONV_NO_TEAMS) == quad, c.name
