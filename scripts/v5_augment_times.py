"""Times YOLOv5's hyp.scratch augmentations (random_perspective -> augment_hsv -> flipud -> fliplr) on 32 seeded
640x480 uint8 images: CUDA-event medians of 20 for the v5_augment kernel alone and for apply_batch end to end, and
the reference's cv2 path on the host's cores where cv2 imports.  Prints one JSON line (and writes it to --out).

    python scripts/v5_augment_times.py --out v5_augment_times.json
"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5aug_cases as VC  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.v5.utils import augmentations as A  # noqa: E402

N, H, W, REPS = 32, 480, 640, 20
HBM_BYTES_PER_S = 3.35e12


def median_ms(fn, reps=REPS):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ims_np = [VC.image(200 + k, H, W) for k in range(N)]
    ims = [torch.from_numpy(im).to(dev) for im in ims_np]
    labs = [VC.labels(200 + k, H, W, 6) for k in range(N)]
    targets = [{"boxes": torch.from_numpy(l[:, 1:].copy()).to(dev), "labels": torch.from_numpy(l[:, 0]).long().to(dev)}
               for l in labs]
    hyp = A.HYP_SCRATCH

    # the kernel alone: one batch's descriptors on the device, relaunched
    random.seed(0)
    np.random.seed(0)
    plans, _ = A.plan_batch([(H, W)] * N, [l.copy() for l in labs], hyp)
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
    descs = (_C.V5Image * N)()
    for d, im, o, p in zip(descs, ims, out, plans):
        A._fill(d, im, o, p, False)
    total = ctypes.c_int64(0)
    _C.check(_C.lib().yb_v5_augment_prepare(N, descs, ctypes.byref(total)), "prepare")
    raw = torch.frombuffer(bytearray(ctypes.string_at(ctypes.addressof(descs), ctypes.sizeof(descs))),
                           dtype=torch.uint8)
    d_descs = raw.to(dev)
    stream = _C.current_stream_ptr(dev)
    kernel_ms = median_ms(lambda: _C.check(_C.lib().yb_v5_augment(N, d_descs.data_ptr(), total.value, stream), "k"))
    warped = sum(p.inv is not None for p in plans)
    # bytes: every output byte written once, every source byte read at least once (the warp's taps hit L2 after)
    nbytes = 2 * N * H * W * 3

    def end_to_end():
        A.apply_batch(ims, targets, hyp)

    e2e_ms = median_ms(end_to_end)

    res = {"images": N, "size": [H, W], "kernel_ms": kernel_ms, "apply_batch_ms": e2e_ms, "warped_images": warped,
           "kernel_bytes": nbytes, "kernel_GBps": nbytes / kernel_ms / 1e6,
           "kernel_fraction_of_3.35TBps": nbytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S, "gpu": gpu_info()}
    try:
        import cv2

        def cv2_batch():
            for im, l in zip(ims_np, labs):
                im = im.copy()
                M, s, height, width = A._perspective_draw(im.shape, hyp["degrees"], hyp["translate"], hyp["scale"],
                                                          hyp["shear"], hyp["perspective"], (0, 0))
                im = cv2.warpAffine(im, M[:2], dsize=(width, height), borderValue=(114, 114, 114))
                A._warp_targets(l.copy(), M, s, width, height, 0.0)
                lut = A._hsv_draw(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
                hue, sat, val = cv2.split(cv2.cvtColor(im, cv2.COLOR_BGR2HSV))
                hsv = cv2.merge((cv2.LUT(hue, lut[0]), cv2.LUT(sat, lut[1]), cv2.LUT(val, lut[2])))
                cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR, dst=im)
                if random.random() < hyp["flipud"]:
                    im = np.flipud(im)
                if random.random() < hyp["fliplr"]:
                    im = np.fliplr(im)

        cv2_batch()
        t = []
        for _ in range(5):
            t0 = time.perf_counter()
            cv2_batch()
            t.append((time.perf_counter() - t0) * 1e3)
        res["cv2_ms"] = float(np.median(t))
        res["cv2_threads"] = cv2.getNumThreads()
    except ImportError:
        res["cv2_ms"] = None
    res["host_cpus"] = os.cpu_count()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
