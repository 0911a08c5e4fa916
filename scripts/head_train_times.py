"""CUDA-event times of head fine-tuning at yolov5s batch 32 640 x 640 and yolov5x6 batch 16 1280 x 1280: the weight-
gradient launch pair (yb_conv_wgrad) against its bound from the shapes, the layout copy of the incoming gradients, the
feature-gradient launch, one in-place head refresh against one full re-lowering, and a whole training step (train-mode
forward, SetCriterion, backward, GradScaler + SGD step) with a frozen backbone.  Prints one JSON line per measurement,
the card, its power limit and maximum SM clock first (queried in the same run).

    python scripts/head_train_times.py [--iters 20] [--out path.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loss_cases as LC  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.engine import Lowered, head_dgrad  # noqa: E402
from yolort_b200.models.box_head import SetCriterion  # noqa: E402
from yolort_b200.models.yolov5 import YOLOv5  # noqa: E402

DEV = "cuda:0"
HBM_BPS = 3.35e12        # H100 SXM data sheet
TENSOR_FLOPS = 989e12    # dense fp16 / bf16 with fp32 accumulation, data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def host_timed(fn, iters):
    ts = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = []
    emit(rows, {"card": card(), "torch": torch.__version__})
    for arch, n, size in (("yolov5_darknet_pan_s_r60", 32, 640), ("yolov5_darknet_pan_x6_r60", 16, 1280)):
        m = YOLOv5(arch=arch, size=(size, size))
        yolo = m.model.to(DEV)
        yolo.backbone.requires_grad_(False)
        ag = yolo.anchor_generator
        yolo.compute_loss = SetCriterion(ag.strides, ag.anchor_grids, yolo.num_classes)
        yolo.train()
        x = torch.rand(n, 3, size, size, generator=torch.Generator().manual_seed(0)).to(DEV)
        targets = LC.random_targets(n, yolo.num_classes, 7 * n, 1).to(DEV)
        tag = {"model": arch, "batch": n, "size": size}

        # inputs of one backward: features and incoming gradients at this shape
        feats = yolo.backbone(x)
        outs = yolo.head(feats)
        grads = [torch.randn_like(o) * 1e-3 for o in outs]
        low = yolo.engine().lowered()
        dt = low.L.dtype

        # wgrad launch pair over all levels
        specs, bytes_, flops = [], 0, 0
        dys = []
        for f, g, conv in zip(feats, grads, yolo.head.head):
            nn_, c, h, w = f.shape
            co = conv.out_channels
            dy = torch.zeros((nn_, h, w, (co + 15) // 16 * 16), dtype=dt, device=DEV)
            dys.append((dy, g, co))
            P = nn_ * h * w
            specs.append((dy.view(P, -1), f.permute(0, 2, 3, 1).reshape(P, c), torch.empty((co, c), device=DEV),
                          torch.empty((co,), device=DEV)))
            bytes_ += P * (co + c) * 2
            flops += 2 * P * co * (c + 1)
        t = timed(lambda: _C.conv_wgrad(specs, torch.device(DEV)), args.iters)
        bound = max(bytes_ / HBM_BPS, flops / TENSOR_FLOPS) * 1e3
        cfg = _C.conv_wgrad_config(_C.wgrad_problems(specs))
        emit(rows, dict(tag, what="wgrad launch pair", ms=round(t, 4), bound_ms=round(bound, 4),
                        share_of_bound=round(bound / t, 3), mbytes=round(bytes_ / 1e6, 1), gflop=round(flops / 1e9, 2),
                        items=cfg["items"], workspace_mb=round(cfg["workspace_bytes"] / 1e6, 1)))

        # layout copy of the incoming gradients into zero-padded [P, C_pad] rows
        A, K = ag.num_anchors, yolo.num_classes + 5

        def layout():
            for dy, g, co in dys:
                nn_, h, w = dy.shape[:3]
                dy[..., co:].zero_()
                dy[..., :co].view(nn_, h, w, A, K).copy_(g.permute(0, 2, 3, 1, 4))
        emit(rows, dict(tag, what="gradient layout copy", ms=round(timed(layout, args.iters), 4)))

        # feature-gradient launches (one 1x1 convolution per level)
        dg = [head_dgrad(low, l, f.shape[0], f.shape[2], f.shape[3], f.shape[1]) for l, f in enumerate(feats)]
        emit(rows, dict(tag, what="dgrad launches", ms=round(timed(lambda: [d.plan.run() for d in dg], args.iters), 4)))

        # one head refresh against one full re-lowering
        eng = yolo.engine()
        t_ref = host_timed(lambda: low.refresh_head(), args.iters)
        t_low = host_timed(lambda: Lowered(yolo, eng.dtype, eng.device, eng.stem_variant), max(3, args.iters // 4))
        emit(rows, dict(tag, what="head refresh vs re-lowering (host wall clock)", refresh_ms=round(t_ref, 3),
                        relower_ms=round(t_low, 3)))

        # a whole training step
        del feats, outs, grads, specs, dys, dg
        opt = torch.optim.SGD(yolo.head.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
        scaler = torch.amp.GradScaler("cuda")

        def step():
            loss = sum(yolo(x, targets).values())
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
            opt.zero_grad(set_to_none=True)
        t_step = timed(step, args.iters)
        emit(rows, dict(tag, what="training step", ms=round(t_step, 3), img_per_s=round(n / t_step * 1e3, 1),
                        lowerings=eng.lowerings))
        del m, yolo, opt
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
