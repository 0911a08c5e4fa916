"""CUDA-event times of the training loss (SetCriterion forward, and backward to the head outputs) at yolov5s batch 32
640 x 640 and yolov5x6 batch 16 1280 x 1280, with COCO's mean of about 7 targets per image and a 100-per-image stress
case, in fp16 and fp32 head outputs.  The comparator is the torch restatement (oracle/restate_loss.py) run eagerly on
the same GPU.  Prints one JSON line per configuration, the card and its power limit first.

    python scripts/loss_times.py [--iters 20] [--out path.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loss_cases as LC  # noqa: E402
from oracle import restate_loss as R  # noqa: E402
from yolort_b200.models.box_head import SetCriterion  # noqa: E402

DEV = "cuda:0"


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = [{"card": card(), "torch": torch.__version__}]
    print(json.dumps(rows[0]), flush=True)
    configs = [("yolov5s", 32, 640, LC.P5_STRIDES, LC.P5_ANCHORS), ("yolov5x6", 16, 1280, LC.P6_STRIDES, LC.P6_ANCHORS)]
    for model, n, size, strides, anchors in configs:
        shapes = LC.head_shapes(n, size, size, strides, 3, 80)
        for per_image in (7, 100):
            targets = LC.random_targets(n, 80, per_image * n, 1000 + per_image).to(DEV)
            for dtype in (torch.float16, torch.float32):
                heads = [h.requires_grad_(True) for h in LC.head_outputs(shapes, 11, dtype=dtype, device=DEV)]
                crit = SetCriterion(strides, anchors, 80)
                ones = [torch.ones(1, device=DEV)] * 3

                def fwd():
                    return crit(targets, heads)

                def fwd_bwd():
                    out = crit(targets, heads)
                    torch.autograd.grad(list(out.values()), heads, ones)

                def ref_fwd():
                    return R.loss(targets, heads, strides, anchors, 80)[0]

                def ref_fwd_bwd():
                    out = ref_fwd()
                    torch.autograd.grad(list(out.values()), heads, ones, allow_unused=True)

                with torch.no_grad():
                    t_fwd = timed(fwd, args.iters)
                t_all = timed(fwd_bwd, args.iters)
                with torch.no_grad():
                    r_fwd = timed(ref_fwd, max(3, args.iters // 4))
                r_all = timed(ref_fwd_bwd, max(3, args.iters // 4))
                row = {"model": model, "batch": n, "size": size, "targets_per_image": per_image,
                       "dtype": str(dtype).replace("torch.", ""),
                       "forward_ms": round(t_fwd, 4), "forward_backward_ms": round(t_all, 4),
                       "backward_ms": round(t_all - t_fwd, 4),
                       "eager_forward_ms": round(r_fwd, 3), "eager_forward_backward_ms": round(r_all, 3),
                       "speedup_forward_backward": round(r_all / t_all, 1)}
                rows.append(row)
                print(json.dumps(row), flush=True)
                del heads
                torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
