"""Times YOLOv5's AutoAnchor on the GPU at a COCO-like seeded set of 860 k labels: kmean_anchors and check_anchors end
to end (host draws included), and their device parts alone (the 30 k-means trials, the 1000-generation evolution, one
metric pass), with CUDA events after warm-up.  Next to them, the same algorithm as restated on the CPU
(oracle/restate_autoanchor.py): one fitness evaluation and one vq + mean pass, the units the CPU repeats.  Prints the
card's name and power limit read in the same run.

    python scripts/autoanchor_times.py [--labels 860000] [--gen 1000]
"""
import argparse
import logging
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

import autoanchor_cases as AC  # noqa: E402
from oracle import restate_autoanchor as R  # noqa: E402


def _events(fn, reps=1):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def _wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels", type=int, default=860_000)
    ap.add_argument("--gen", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these are GPU timings")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}")
    from yolort_b200 import _C
    from yolort_b200.models import yolov5n
    from yolort_b200.v5.utils import autoanchor as AA

    logging.getLogger(AA.__name__).setLevel(logging.WARNING)
    images = args.labels // 20
    ds = AC.make(0, images, 27, scale=0.3, sigma=0.9)     # 20.25 labels per image on average
    shapes = 640 * ds.shapes / ds.shapes.max(1, keepdims=True)
    wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, ds.labels)])
    wh = wh0[(wh0 >= 2.0).any(1)]
    print(f"labels: {wh0.shape[0]} ({wh.shape[0]} after the 2 px filter)")

    obs = wh / wh.std(0)
    d_obs = torch.from_numpy(obs).cuda()
    np.random.seed(0)
    idx = torch.from_numpy(np.stack([np.random.choice(obs.shape[0], 9, replace=False) for _ in range(30)])).cuda()
    t_km, (books, sizes, dist, iters) = _events(lambda: _C.kmeans(d_obs, d_obs[idx]))
    best = int(torch.argmin(dist))
    codes, _ = R.vq(obs, books[best, :int(sizes[best])].cpu().numpy())
    chain = int(np.bincount(codes).max())
    print(f"gpu kmeans (30 trials at once): {t_km:.1f} ms, {iters} iterations launched, largest cluster of the best "
          f"trial {chain} points (its centroid sum is one dependent chain of that length)")

    wh_d = torch.from_numpy(wh.astype(np.float32)).cuda()
    k0 = np.sort(books[best, :9].cpu().numpy() * wh.std(0), axis=0)
    random.seed(0)
    np.random.seed(0)
    v = AA.draw_mutations(9, args.gen)
    t_ev, _ = _events(lambda: AA.evolve_anchors(wh_d, k0, v, 0.25))
    print(f"gpu evolution ({args.gen} generations, one cooperative launch): {t_ev:.1f} ms "
          f"({t_ev / max(args.gen, 1) * 1e3:.1f} us per generation)")
    wh0_d = torch.from_numpy(wh0.astype(np.float32)).cuda()
    t_m, _ = _events(lambda: _C.anchor_metric(wh0_d, torch.from_numpy(k0), 0.25, True), reps=20)
    print(f"gpu metric pass: {t_m * 1e3:.0f} us")

    random.seed(0)
    np.random.seed(0)
    AA.kmean_anchors(ds, n=9, gen=args.gen, verbose=False)          # warm-up
    random.seed(0)
    np.random.seed(0)
    t_all, _ = _wall(lambda: AA.kmean_anchors(ds, n=9, gen=args.gen, verbose=False))
    print(f"kmean_anchors end to end (host draws included): {t_all:.0f} ms")
    model = yolov5n(size=(128, 128))
    np.random.seed(0)
    t_chk, _ = _wall(lambda: AA.check_anchors(ds, model, thr=4.0, imgsz=640))
    print(f"check_anchors end to end (replaces the anchors when the fit is poor): {t_chk:.0f} ms")

    wh32 = wh.astype(np.float32)
    t = time.perf_counter()
    R.fitness(wh32, k0, 0.25)
    t_fit = (time.perf_counter() - t) * 1e3
    t = time.perf_counter()
    _, d = R.vq(obs, k0 / wh.std(0))
    R.np_mean(d)
    t_vq = (time.perf_counter() - t) * 1e3
    print(f"cpu restatement: one fitness evaluation {t_fit:.0f} ms (x {args.gen} generations = "
          f"{t_fit * args.gen / 1e3:.0f} s), one vq + mean pass {t_vq:.0f} ms")


if __name__ == "__main__":
    main()
