"""The four-consumer-warpgroup instance of the halo-patch kernel: the cases take the path their names state and reach
an odd last pair, the rule holds on both sides of its edges, and the c2-c5 layers that take it are the ones the rule
names (host logic, no GPU needed; SM-dependent sizes follow the device's SM count, 132 without a GPU).  Instance
coverage, the pinning bit and the other tables are checked in tests/test_conv_coverage.py."""
import conv_cases
import conv_cases_quad as q
from conv_cases import BF16, F16, VARIANTS, Case, config

_is_quad = VARIANTS["patch quad"].takes


def test_cases_take_the_path_their_name_states():
    for c in q.CASES:
        cfg = config(c)
        quad = c.name.split()[1] == "quad"
        assert cfg["patch_kernel"] and cfg["tiles_per_pass"] == 2 and not cfg["weights_resident"], (c.name, cfg)
        assert _is_quad(cfg) == quad, (c.name, cfg)
        assert cfg["patch_tiling"] == c.name.split()[2], (c.name, cfg)
        if quad:
            assert cfg["block_n"] == 128 and cfg["n_tiles"] == c.Cout // 128 and cfg["layout"] == "1x4", (c.name, cfg)
            assert cfg["slots"] == 4 and cfg["ring"] >= 4 and cfg["smem_bytes"] <= 227 * 1024 - 768, (c.name, cfg)
            assert cfg["grid"] % cfg["n_tiles"] == 0
        else:
            assert cfg["block_n"] <= 64 and cfg["consumer_groups"] == 2, (c.name, cfg)


def test_every_instance_is_reached_and_the_odd_last_pair():
    reached = {("bf16" if c.dtype == BF16 else "f16", config(c)["m_tiles"] % 2) for c in q.CASES if _is_quad(config(c))}
    assert reached == {(dt, odd) for dt in ("f16", "bf16") for odd in (0, 1)}, sorted(reached)


def _tasks(cfg) -> int:
    return cfg["work_items"]


def test_rule_edges():
    """T tasks of 128 columns on G = SMs CTAs: four warpgroups exactly when T >= G and T mod G = 0 or > G / 2."""
    G = conv_cases.SMS
    # 1-tile images (16 x 8 classic tiles), Cout 128: T = ceil(N / 2)
    for T in (G // 2 + 1, G - 1, G, G + 1, G + G // 2, G + G // 2 + 1, 2 * G, 2 * G + G // 2 + 1):
        for dt in (F16, BF16):
            c = Case("edge", 2 * T, 16, 8, 128, 128, k=3, dtype=dt)
            cfg = config(c)
            r = T % G
            want = T >= G and (r == 0 or r > G // 2)
            assert cfg["tiles_per_pass"] == 2
            assert _is_quad(cfg) == want, (T, cfg)
            assert _tasks(cfg) == (T if want else 2 * T), (T, cfg)


# The stride-1 3x3 convolutions with streamed weights of the bench configs (the Bottleneck cv2 of the C3 blocks at
# strides 16 and 32; their shallower ones keep resident weights): (config, map side, channels, images, four warpgroups)
BENCH_LAYERS = [
    ("c2 yolov5s", 40, 128, 32, True),     # body.6.m.*, pan.inner_blocks.3.m.0, pan.layer_blocks.2.m.0: 240 tasks
    ("c2 yolov5s", 20, 256, 32, False),    # body.8.m.0, pan.layer_blocks.4.m.0: 128 tasks, fewer than CTAs
    ("c3 yolov5m", 40, 192, 128, False),   # Cout 192 is not a multiple of 128
    ("c3 yolov5m", 20, 384, 128, True),    # 768 tasks on three N tiles
    ("c4 yolov5l", 40, 256, 16, True),     # 240 tasks on two N tiles
    ("c4 yolov5l", 20, 512, 16, False),    # 128 tasks on four N tiles, fewer than CTAs
    ("c5 yolov5x", 80, 320, 64, False),    # Cout 320 is not a multiple of 128
    ("c5 yolov5x", 40, 640, 64, False),    # five N tiles do not divide a grid of 132
]


def test_bench_layers():
    if conv_cases.SMS != 132:
        return   # the expectations are those of a 132-SM H100
    for cfgname, side, c, n, want in BENCH_LAYERS:
        for dt in (F16, BF16):
            cfg = config(Case(cfgname, n, side, side, c, c, k=3, dtype=dt, residual=True))
            assert cfg["patch_kernel"] and cfg["tiles_per_pass"] == 2, (cfgname, side, c, cfg)
            assert _is_quad(cfg) == want, (cfgname, side, c, cfg)
