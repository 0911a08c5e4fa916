"""Test-time augmentation (`augment=True`) against the plain forward on one H100, CUDA-event medians.

For each config (yolov5s batch 32 640^2 fp16; yolov5x6 batch 16 1280^2 fp16; synthetic weights, random uint8 images
already on the device), reports: the canvas rescale kernel per pass and its fraction of the HBM bound at 3.35 TB/s
(bytes = source canvas read + pass canvas written), the three plan runs, the multi-pass decode + NMS, the whole
`forward(images, augment=True)` and the plain `forward(images)`.  Prints the card name, power limit and maximum SM
clock read in the same run, and writes everything as JSON to --out.

    python scripts/tta_times.py --out tta_times.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import parity_util as util  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.models import YOLOv5, yolov5s  # noqa: E402

DEV = torch.device("cuda:0")
HBM = 3.35e12


def yolov5x6(**kw):
    return YOLOv5(arch="yolov5_darknet_pan_x6_r60", size_divisible=64, **kw)


CFG = {"s_b32_640": (yolov5s, "s", 32, 640, None), "x6_b16_1280": (yolov5x6, "x6", 16, 1280, 1.3)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def median_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def run(name, reps):
    ctor, key, n, side, gain = CFG[name]
    lay = util.layouts()
    if key not in lay:        # x6 layout: the constructor's own state dict shapes
        shapes = {k: list(v.shape) for k, v in ctor().state_dict().items()}
    else:
        shapes = lay[key]
    kw = {} if gain is None else {"gain": gain}
    sd = util.synth_state_dict(shapes, knob_obj=0.0, knob_cls=0.0, seed=0, **kw)
    m = ctor(size=(side, side)).eval()
    m.load_state_dict(sd)
    m = m.to(DEV).half()
    g = torch.Generator().manual_seed(1)
    ims = [torch.randint(0, 256, (3, side, side), generator=g, dtype=torch.uint8).to(DEV) for _ in range(n)]
    with torch.no_grad():
        plain = median_ms(lambda: m(ims), reps)
        tta = median_ms(lambda: m(ims, augment=True), reps)
        yolo = m.model
        geo, plans = yolo.tta_plans(n, side, side)
        res = {"config": name, "batch": n, "canvas": side, "passes": geo, "plain_forward_ms": plain,
               "tta_forward_ms": tta, "tta_over_plain": tta / plain}
        for q in (1, 2):
            nh, nw, hp, wp = geo[q]
            ms = median_ms(lambda: _C.canvas_rescale(plans[0].input, plans[q].input, nh, nw, _C.TTA_FLIPS[q]), reps * 4)
            nbytes = plans[0].input.numel() * 2 + plans[q].input.numel() * 2
            res[f"canvas{q}_ms"] = ms
            res[f"canvas{q}_hbm_fraction"] = nbytes / (ms * 1e-3) / HBM
        for q in range(3):
            res[f"plan{q}_ms"] = median_ms(plans[q].run, reps)
        pc = yolo.post_config()
        nl = len(plans[0].heads)
        kept = [list(range(nl - 1)), list(range(nl)), list(range(1, nl))]
        passes = [(pl.heads, kept[q], _C.TTA_SCALES[q], _C.TTA_FLIPS[q]) for q, pl in enumerate(plans)]
        res["decode_nms_ms"] = median_ms(lambda: _C.decode_nms_tta_padded(
            passes, side, pc["strides"], pc["anchors_px"], pc["num_classes"], pc["score_thresh"], pc["nms_thresh"],
            pc["detections_per_img"], pc["semantics"]), reps)
        res["plain_plan_ms"] = res["plan0_ms"]
        res["three_plans_over_plain_plan"] = sum(res[f"plan{q}_ms"] for q in range(3)) / res["plan0_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=list(CFG))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "results": []}
    print("card (name, power limit, max SM clock):", out["card"])
    for c in a.configs:
        r = run(c, a.reps)
        print(json.dumps(r))
        out["results"].append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
