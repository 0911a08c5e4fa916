"""FP8 (e4m3) against fp16 on one H100, alternating the two precisions in one process.

For each config (c2: yolov5s batch 32 640^2, bench weights; c5: yolov5x batch 64 1280^2, zoo weights gain 1.3):
  * plan time per batch: CUDA-graph replay of the whole launch list, fp16 and FP8 alternated over several rounds;
  * per-op table: CUDA events around each launch (median of repeats), FLOP/s for the convolutions (the reference's
    algorithmic work), bytes/s (bytes read + written) for the pool / upsample / quantise ops;
  * the fraction of fp16 detections that FP8 reproduces (same label, IoU > 0.9) on the bench's images.
The calibration uses 4 other images of the same generator.  Prints the card name and power limit with the numbers and
writes everything as JSON to --out.

    python scripts/fp8_times.py --configs c2 c5 --out fp8_times.json
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

import bench  # noqa: E402
import parity_util as util  # noqa: E402
from yolort_b200 import _C, models  # noqa: E402
from yolort_b200.quantization import calibrate_fp8  # noqa: E402

DEV = torch.device("cuda:0")
CFG = {"c2": ("yolov5s", 32, 640, None, 0.25), "c5": ("yolov5x", 64, 1280, 1.3, 0.044)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def graph_ms(plan, iters):
    plan.use_graph = True
    plan.run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        plan.run()
    b.record()
    torch.cuda.synchronize()
    plan.use_graph = False
    return a.elapsed_time(b) / iters


def per_op(plan, reps):
    L = plan._low.L
    N, H, W = plan.N, plan.H, plan.W
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    rows = []
    plan.run()
    for li, grp in enumerate(plan.launch_ops):
        op = L.ops[grp[0]]
        for a, b in ev:
            a.record()
            plan.run(li, 1)
            b.record()
        torch.cuda.synchronize()
        us = 1e3 * statistics.median(a.elapsed_time(b) for a, b in ev)
        hi, wi = op.src.buf.hw(H, W)
        ho, wo = op.dst.buf.hw(H, W)
        nbytes = N * (hi * wi * op.src.C * op.src.buf.esz + ho * wo * op.dst.C * op.dst.buf.esz)
        flops = plan.op_flops[li]
        rows.append({"op": plan.op_names[li], "kind": op.kind, "us": us,
                     "tflops": flops / us / 1e6 if flops else None,
                     "gbps": None if flops else nbytes / us / 1e3})
    return rows


def detections(m, ims):
    return [util.to_np(d) for d in m(ims)]


def run(name, rounds, iters, reps):
    arch, batch, size, gain, thr = CFG[name]
    m = getattr(models, arch)(size=(size, size), score_thresh=thr).eval()
    m.load_state_dict(bench.make_state_dict(m) if gain is None else bench.zoo_state_dict(m, gain))
    m = m.to(DEV).half()
    calib = calibrate_fp8(m, [[im.to(DEV) for im in bench.make_images(4, 777, size)]])
    ims = [im.to(DEV) for im in bench.make_images(batch, 1234, size)]
    ref = detections(m, ims)
    m.set_fp8(calib)
    got = detections(m, ims)
    n_ref = sum(len(r["scores"]) for r in ref)
    matched = sum(util.match_fraction(g, r) * len(r["scores"]) for g, r in zip(got, ref)) / max(n_ref, 1)
    plans = {}
    for prec in ("fp16", "fp8"):
        m.set_fp8(calib if prec == "fp8" else None)
        plans[prec] = m.model.get_plan(batch, size, size)     # input canvas written by the detections() call
    times = {"fp16": [], "fp8": []}
    for _ in range(rounds):
        for prec in ("fp16", "fp8"):
            m.set_fp8(calib if prec == "fp8" else None)
            times[prec].append(graph_ms(plans[prec], iters))
    ops = {}
    for prec in ("fp16", "fp8"):
        m.set_fp8(calib if prec == "fp8" else None)
        ops[prec] = per_op(plans[prec], reps)
    m.set_fp8(None)
    res = {"config": name, "model": arch, "batch": batch, "size": size,
           "plan_ms": {p: statistics.median(t) for p, t in times.items()},
           "plan_ms_all": times, "matched_fp8_vs_fp16": matched, "fp16_detections": n_ref, "ops": ops}
    print(f"{name} {arch} b{batch} {size}^2: plan fp16 {res['plan_ms']['fp16']:.2f} ms  fp8 {res['plan_ms']['fp8']:.2f} ms"
          f"  speedup {res['plan_ms']['fp16'] / res['plan_ms']['fp8']:.3f}  matched {matched:.4f} of {n_ref}")
    f16 = {r["op"]: r for r in ops["fp16"]}
    print(f"  {'op':58s} {'fp16 us':>9s} {'fp8 us':>9s} {'fp16':>12s} {'fp8':>12s}")
    for r in ops["fp8"]:
        a = f16.get(r["op"])
        rate = (lambda x: "" if x is None else (f"{x['tflops']:.0f} TF/s" if x["tflops"] else f"{x['gbps']:.0f} GB/s"))
        print(f"  {r['op'][:58]:58s} {a['us'] if a else float('nan'):9.1f} {r['us']:9.1f} {rate(a):>12s} {rate(r):>12s}")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["c2", "c5"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_times.py measures on a GPU; none is visible")
    torch.backends.cudnn.allow_tf32 = False
    info = card()
    print("card (name, power limit, max SM clock):", info)
    out = {"card": info, "results": [run(c, args.rounds, args.iters, args.reps) for c in args.configs]}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
