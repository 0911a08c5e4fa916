"""Training-loss inputs shared by oracle/make_golden_loss.py, tests/test_loss.py (CPU) and tests/test_gpu_loss.py:
seeded head outputs (rounded to fp16-representable values, so an fp16 or bf16 head output of the same case holds the
same numbers where bf16 can) and targets, regenerated rather than stored.  A case is a dict of the SetCriterion
keyword arguments ("kw"), the head output shapes, and one (targets, head_outputs) per call."""
import numpy as np
import torch

P5_STRIDES = [8, 16, 32]
P5_ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
P6_STRIDES = [8, 16, 32, 64]
P6_ANCHORS = [[19, 27, 44, 40, 38, 94], [96, 68, 86, 152, 180, 137], [140, 301, 303, 264, 238, 542],
              [436, 615, 739, 380, 925, 792]]

# gradients stored per level: the matched cells, plus this many dense cells chosen by a fixed seed
DENSE_SAMPLE = 256


def head_shapes(n, h, w, strides, num_anchors, num_classes):
    return [(n, num_anchors, h // s, w // s, num_classes + 5) for s in strides]


def head_outputs(shapes, seed, dtype=torch.float32, device="cpu"):
    """Logits with the spread of a trained detector's: box terms ~N(0, 0.5), objectness ~N(-4, 2), classes
    ~N(-3, 2); every value fp16-representable."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for shp in shapes:
        x = torch.randn(shp, generator=g)
        x[..., :4] *= 0.5
        x[..., 4] = x[..., 4] * 2.0 - 4.0
        x[..., 5:] = x[..., 5:] * 2.0 - 3.0
        out.append(x.half().float().to(device=device, dtype=dtype).contiguous())
    return out


def random_targets(n_images, num_classes, count, seed):
    """[count, 6] fp32 (image, class, cx, cy, w, h), sizes log-uniform over 1 %-60 % of the canvas."""
    rs = np.random.RandomState(seed)
    t = np.zeros((count, 6), np.float32)
    t[:, 0] = rs.randint(0, n_images, count)
    t[:, 1] = rs.randint(0, num_classes, count)
    t[:, 2:4] = rs.uniform(0.0, 1.0, (count, 2))
    t[:, 4:6] = np.exp(rs.uniform(np.log(0.01), np.log(0.6), (count, 2)))
    return torch.from_numpy(t)


def edge_targets():
    """Targets on the assignment's boundaries for a 256 x 320 canvas at strides 8 / 16 / 32 (grids 40, 20, 10 wide
    and 32, 16, 8 high): gxy exactly x.5 and integral, gxy <= 1 and == 1, the far edges and beyond the canvas, an
    anchor ratio of exactly 4 (r and 1 / r), and zero-size boxes."""
    rows = [
        (0, 0, 0.3125, 0.265625, 0.1, 0.1),        # gx = 12.5 at W = 40, gy = 8.5 at H = 32
        (0, 1, 0.1, 0.125, 0.2, 0.15),             # gx ~ 1.0 at W = 10, gy = 1.0 at H = 8, integral at H = 16, 32
        (1, 2, 0.015625, 0.03125, 0.05, 0.05),     # gxy <= 1 at every level
        (1, 3, 1.0, 1.0, 0.3, 0.3),                # far edge: gi = W clamps to W - 1
        (0, 4, 0.0, 0.0, 0.05, 0.08),              # near edge
        (1, 5, 0.99, 0.9921875, 0.02, 0.03),
        (0, 6, -0.05, 0.5, 0.1, 0.1),              # centre outside the canvas
        (1, 7, 0.5, 0.5, 0.125, 0.05078125),       # gwh / anchor(10, 13) = (4.0, 1.0) exactly at stride 8
        (0, 0, 0.25, 0.75, 0.0078125, 0.05078125),  # 1 / r = 4.0 exactly at stride 8
        (1, 1, 0.4, 0.6, 0.0, 0.0),                # zero-size
        (0, 2, 0.6, 0.4, 0.0, 0.1),                # zero width
        (1, 3, 0.7, 0.2, 0.25, 0.5),
    ]
    return torch.tensor(rows, dtype=torch.float32)


def dup_targets():
    """Two targets per cell and anchor (the later one owns the objectness target; the gradients add)."""
    rows = [(0, 1, 0.30, 0.40, 0.10, 0.12), (0, 3, 0.301, 0.402, 0.11, 0.125),
            (1, 0, 0.62, 0.17, 0.30, 0.35), (1, 2, 0.621, 0.171, 0.31, 0.34), (1, 4, 0.6205, 0.1705, 0.29, 0.36)]
    return torch.cat([torch.tensor(rows, dtype=torch.float32), random_targets(2, 8, 6, 31)])


def cases():
    """name -> {"kw": SetCriterion kwargs, "shapes": head shapes, "calls": [(targets, head_outputs)]}."""
    c = {}
    s5 = head_shapes(2, 256, 320, P5_STRIDES, 3, 8)
    base = {"strides": P5_STRIDES, "anchor_grids": P5_ANCHORS, "num_classes": 8}
    c["basic"] = {"kw": dict(base), "shapes": s5, "calls": [(random_targets(2, 8, 40, 1), head_outputs(s5, 101))]}
    c["hyper"] = {"kw": dict(base, fl_gamma=1.5, box_gain=0.07, cls_gain=0.3, cls_pos=1.3, obj_gain=0.8, obj_pos=0.7,
                             anchor_thresh=2.9, label_smoothing=0.1),
                  "shapes": s5, "calls": [(random_targets(2, 8, 40, 2), head_outputs(s5, 102))]}
    c["empty"] = {"kw": dict(base), "shapes": s5, "calls": [(torch.zeros((0, 6)), head_outputs(s5, 103))]}
    c["edges"] = {"kw": dict(base), "shapes": s5, "calls": [(edge_targets(), head_outputs(s5, 104))]}
    c["dup"] = {"kw": dict(base), "shapes": s5, "calls": [(dup_targets(), head_outputs(s5, 105))]}
    s6 = head_shapes(2, 256, 320, P6_STRIDES, 3, 8)
    c["p6"] = {"kw": {"strides": P6_STRIDES, "anchor_grids": P6_ANCHORS, "num_classes": 8}, "shapes": s6,
               "calls": [(torch.cat([random_targets(2, 8, 40, 6), torch.tensor(
                   [(0, 1, 0.5, 0.5, 0.9, 0.95), (1, 2, 0.3, 0.6, 0.7, 0.9)], dtype=torch.float32)]),
                   head_outputs(s6, 106))]}
    s1 = head_shapes(2, 256, 320, P5_STRIDES, 3, 1)
    c["nc1"] = {"kw": dict(base, num_classes=1), "shapes": s1,
                "calls": [(random_targets(2, 1, 30, 7), head_outputs(s1, 107))]}
    c["autobal"] = {"kw": dict(base, auto_balance=True), "shapes": s5,
                    "calls": [(random_targets(2, 8, 20 + 5 * k, 80 + k), head_outputs(s5, 180 + k)) for k in range(3)]}
    return c


def dense_sample(shape, seed=0):
    """Fixed cell indices (flattened over N, A, H, W) at which the dense gradient is stored."""
    n = int(np.prod(shape[:4]))
    return np.sort(np.random.RandomState(seed).choice(n, min(n, DENSE_SAMPLE), replace=False)).astype(np.int64)
