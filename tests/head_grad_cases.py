"""Head shapes of the shipped detection architectures, for the weight-gradient kernel (csrc/conv_wgrad_sm90.cu) and the
differentiable detection head: per level (P, Cout, Cin) with P = N * H * W at the level's stride."""
import functools

import torch

from yolort_b200.models import yolo as Y


def _arch(name: str):
    if name == "ts":
        return Y.yolov5_darknet_tan_s_r40()
    if name == "lite":
        from yolort_b200.models.yolo_lite import yolov5_mobilenet_v3_small_fpn

        m = yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False)
        return getattr(m, "model", m)
    return getattr(Y, f"yolov5_darknet_pan_{name}")()


ARCHS_640 = ["n_r60", "s_r60", "m_r60", "l_r60", "x_r60", "s_r40", "s_r31", "ts", "lite"]
ARCHS_1280 = ["n6_r60", "s6_r60", "m6_r60", "l6_r60", "x6_r60"]


@functools.lru_cache(maxsize=None)
def head_channels(name: str):
    """[(Cout, Cin, stride)] per head level of architecture `name` (built on the CPU, nothing is run)."""
    with torch.device("cpu"):
        m = _arch(name)
    strides = m.anchor_generator.strides
    return [(int(c.out_channels), int(c.in_channels), int(s)) for c, s in zip(m.head.head, strides)]


def head_problems(name: str, batch: int, size: int):
    """[(P, Cout, Cin)] of every head level at batch x size^2."""
    return [(batch * max(size // s, 1) ** 2, co, ci) for co, ci, s in head_channels(name)]


def all_head_problems():
    """(id, problems) of the shipped architectures at their training shapes: b32 640^2, P6 at b16 1280^2."""
    out = [(f"{a}-b32-640", head_problems(a, 32, 640)) for a in ARCHS_640]
    out += [(f"{a}-b16-1280", head_problems(a, 16, 1280)) for a in ARCHS_1280]
    return out


def edge_problems():
    """num_classes 1 / 3 / 20 / 80 heads, N = 1, a 64^2 canvas whose last level is 2x2, P a multiple of no tile."""
    out = []
    for nc in (1, 3, 20, 80):
        co = 3 * (nc + 5)
        out.append((f"nc{nc}", [(2 * 80 * 80, co, 128), (2 * 40 * 40, co, 256), (2 * 20 * 20, co, 512)]))
    out.append(("n1-640", head_problems("s_r60", 1, 640)))
    out.append(("canvas64", head_problems("s_r60", 2, 64)))
    out.append(("ragged", [(1 * 37 * 29, 255, 128), (3 * 7 * 11, 85, 320), (1, 18, 64), (4097, 255, 1280)]))
    return out
