"""Device COCO box evaluation against the numpy restatement, on a seeded COCO-val-shaped workload (5000 images, 80
categories, about 7 GT per image, detections jittered from GT plus false positives, score ties, crowd GT; built by
tests/coco_corpus.py), in one process on one GPU:

  * `update` of device-resident detections in batches of 32 images: total and per call (CUDA events, synchronised);
  * `compute()`: the whole call (host clock, it ends in a device-to-host copy) and the kernels alone (CUDA events
    around the native evaluate), median over repeats; per-kernel times from a torch.profiler run of its own;
  * the CPU restatement (oracle/restate_cocoeval.py) on the same data, and whether the arrays are bit-identical.
Prints the card name, power limit and maximum SM clock with the numbers and writes them as JSON to --out.

    python scripts/eval_times.py --out eval_times.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from coco_corpus import corpus  # noqa: E402
from oracle import restate_cocoeval as O  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.data import COCOEvaluator  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-images", type=int, default=5000, help="images the CPU restatement is timed on")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    gt, calls = corpus(7, args.images, n_cats=80, batch=32)
    n_det = sum(len(s) for call in calls for _, (_, s, _) in call)
    preds = [[{"boxes": torch.from_numpy(b).to(dev), "scores": torch.from_numpy(s).to(dev),
               "labels": torch.from_numpy(l).to(dev)} for _, (b, s, l) in call] for call in calls]
    ids = [[i for i, _ in call] for call in calls]
    ev = COCOEvaluator(gt, device=dev)

    def feed():
        ev.reset()
        for p, i in zip(preds, ids):
            ev.update(p, i)

    feed()
    ev.compute()
    upd, host_compute, kern = [], [], []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        feed()
        e1.record()
        torch.cuda.synchronize()
        upd.append(e0.elapsed_time(e1))
        t0 = time.perf_counter()
        ev.compute()
        host_compute.append((time.perf_counter() - t0) * 1e3)
        records = ev._records[: ev._n]
        evaluated = torch.ones(ev._gt.n_images, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        e0.record()
        _C.coco_evaluate(ev._gt, records, evaluated, ev._params)
        e1.record()
        torch.cuda.synchronize()
        kern.append(e0.elapsed_time(e1))

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ev.compute()
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "device_time_total", 0) > 0:
            per_kernel[e.key[:90]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 4)
    device_stats, device_eval = ev.stats.copy(), {k: v.copy() for k, v in ev.eval.items()}

    n_or = min(args.oracle_images, args.images)
    keep = set(sorted({i for call in calls for i, _ in call})[:n_or])
    o_calls = [[(i, d) for i, d in call if i in keep] for call in calls]
    t0 = time.perf_counter()
    want, want_stats = O.evaluate(gt, o_calls)
    oracle_s = time.perf_counter() - t0
    identical = None
    if n_or == args.images:
        identical = bool(np.array_equal(want_stats, device_stats) and
                         all(np.array_equal(want[k], device_eval[k]) for k in want))
    res = {
        "card": card(), "images": args.images, "gt": len(gt["annotations"]), "detections": n_det,
        "update_calls": len(calls), "update_total_ms": statistics.median(upd),
        "update_per_call_ms": statistics.median(upd) / len(calls),
        "compute_ms_host": statistics.median(host_compute), "evaluate_kernels_ms": statistics.median(kern),
        "per_kernel_ms_profiled": per_kernel, "oracle_images": n_or, "oracle_s": oracle_s,
        "bit_identical_to_oracle": identical, "stats": device_stats.tolist(),
    }
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
