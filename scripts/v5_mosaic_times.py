"""Times YOLOv5's mosaic training batches (yolort_b200.v5.utils.datasets.train_batch, hyp.scratch) for batch 32 at
img_size 640 on two seeded datasets: 640x480 images, and mixed sizes (downscales, upscales, exact 2x, the 319 -> 639
resize chain).  Reports, with the card's name, power limit and max SM clock read in the same run:

    kernels      median device times of v5_resize_kernel and v5_compose_kernel (torch.profiler, its own pass)
    bytes        the bytes each kernel must move (sources read once, outputs written once) over 3.35 TB/s
    train_batch  end to end, host clock around a synchronised call, median of REPS
    cpu          upstream's recipe with cv2 on the host (cv2.resize, the numpy canvas, warpAffine / warpPerspective,
                 BGR<->HSV with the LUTs, flips, HWC->CHW) on the same draws, single-threaded per sample over a pool
                 of os.cpu_count() workers; "not measured" where cv2 does not import

Prints one JSON line (and writes it to --out).

    python scripts/v5_mosaic_times.py --out v5_mosaic_times.json
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from v5aug_cases import image  # noqa: E402
from yolort_b200.v5.utils import datasets as D  # noqa: E402

N, S, REPS = 32, 640, 20
HBM_BYTES_PER_S = 3.35e12
MIXED = [(480, 640), (640, 480), (1280, 960), (319, 200), (300, 500), (700, 1200), (640, 320), (90, 160)]


def dataset(kind: str, n: int = 64):
    rng = np.random.default_rng(5)
    ims, labs = [], []
    for k in range(n):
        h, w = (480, 640) if kind == "640x480" else MIXED[k % len(MIXED)]
        ims.append(image(2000 + k, h, w))
        m = 1 + k % 6
        labs.append(np.concatenate([rng.integers(0, 80, (m, 1)), rng.uniform(0.2, 0.8, (m, 2)),
                                    rng.uniform(0.05, 0.4, (m, 2))], 1).astype(np.float32))
    return ims, labs


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in q.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not measured ({e})", "max_sm_clock": None}


def bytes_moved(planner: D.Planner, samples):
    """Resize: each source read once, each output written once.  Compose: each placed pixel read once per canvas,
    the [N, 3, s, s] batch written once."""
    resize = 0
    for key, (src, (h, w)) in planner.loads.items():
        sh, sw = planner.shapes[key] if src is None else planner.loads[src][1] if src in planner.loads else \
            planner.shapes[src]
        resize += 3 * (sh * sw + h * w)
    compose = 0
    for smp in samples:
        compose += 3 * smp.out_h * smp.out_w
        for cv in smp.canvases:
            compose += sum(3 * (y1 - y0) * (x1 - x0) for _, y0, x0, y1, x1, _, _ in cv.places)
    return resize, compose


def kernel_ms(fn):
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for k in ("v5_resize_kernel", "v5_compose_kernel"):
            if k in ev.name and ev.device_type.name == "CUDA":
                out.setdefault(k, []).append(ev.device_time_total / 1000.0)
    return {k: float(np.median(v)) for k, v in out.items()}


def cpu_recipe(ims, samples, s):
    """Upstream's cv2 steps on the host for the planned samples; returns ms for the batch."""
    import cv2

    from oracle import restate_v5mosaic as R

    cv2.setNumThreads(1)

    def loaded(key):
        if isinstance(key, tuple):
            im = loaded(key[1])
            (nh, nw), _ = R.letterbox_pad(*im.shape[:2], s)
            return cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR)
        im = ims[key]
        h, w = D.load_shape(*im.shape[:2], s)
        return im if (h, w) == im.shape[:2] else cv2.resize(im, (w, h), interpolation=cv2.INTER_LINEAR)

    def one(smp):
        outs = []
        for cv in smp.canvases:
            canvas = np.full((cv.h, cv.w, 3), 114, np.uint8)
            for key, y0, x0, y1, x1, oy, ox in cv.places:
                canvas[y0:y1, x0:x1] = loaded(key)[y0 - oy:y1 - oy, x0 - ox:x1 - ox]
            if cv.inv is not None:
                flags = cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP
                m = np.asarray(cv.inv, np.float64)
                canvas = (cv2.warpPerspective(canvas, m.reshape(3, 3), (smp.out_w, smp.out_h), flags=flags,
                                              borderValue=(114, 114, 114)) if cv.perspective else
                          cv2.warpAffine(canvas, m[:6].reshape(2, 3), (smp.out_w, smp.out_h), flags=flags,
                                         borderValue=(114, 114, 114)))
            outs.append(canvas)
        im = outs[0] if len(outs) == 1 else (outs[0] * smp.r + outs[1] * (1 - smp.r)).astype(np.uint8)
        if smp.lut is not None:
            hue, sat, val = cv2.split(cv2.cvtColor(im, cv2.COLOR_BGR2HSV))
            im_hsv = cv2.merge((cv2.LUT(hue, smp.lut[0]), cv2.LUT(sat, smp.lut[1]), cv2.LUT(val, smp.lut[2])))
            im = cv2.cvtColor(im_hsv, cv2.COLOR_HSV2BGR)
        if smp.flip_ud:
            im = np.flipud(im)
        if smp.flip_lr:
            im = np.fliplr(im)
        return np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])

    threads = os.cpu_count() or 1
    with ThreadPoolExecutor(threads) as pool:
        list(pool.map(one, samples))
        times = []
        for _ in range(5):
            t0 = time.perf_counter()
            np.stack(list(pool.map(one, samples)))
            times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times)), threads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("v5_mosaic_times: no CUDA device")
    dev = "cuda:0"
    result = {"card": card(), "batch": N, "img_size": S, "hyp": "hyp.scratch (mosaic 1.0, mixup 0.0)"}
    for kind in ("640x480", "mixed"):
        ims, labs = dataset(kind)
        srcs = [torch.from_numpy(im).to(dev) for im in ims]
        indices = list(range(N))

        def call(seed=0):
            random.seed(seed)
            np.random.seed(seed)
            return D.train_batch(srcs, labs, indices, img_size=S)

        kernels = kernel_ms(call)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        e2e = []
        for _ in range(REPS):
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            e2e.append((time.perf_counter() - t0) * 1e3)
        random.seed(0)
        np.random.seed(0)
        planner = D.Planner([im.shape[:2] for im in ims], labs, S, D.HYP_SCRATCH)
        samples = [planner.sample(i) for i in indices]
        rb, cb = bytes_moved(planner, samples)
        r = {"train_batch_ms": float(np.median(e2e)), "kernel_ms": kernels,
             "resize_bytes": rb, "compose_bytes": cb, "resized_images": len(planner.loads)}
        for k, b in (("v5_resize_kernel", rb), ("v5_compose_kernel", cb)):
            if k in kernels:
                r[f"{k}_share_of_3.35TBps"] = b / (kernels[k] * 1e-3) / HBM_BYTES_PER_S
        try:
            r["cpu_cv2_ms"], r["cpu_threads"] = cpu_recipe(ims, samples, S)
        except ImportError:
            r["cpu_cv2_ms"] = "not measured (cv2 does not import)"
        result[kind] = r
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
