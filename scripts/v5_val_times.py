"""Times yolort_b200.v5.val.run on a COCO-val-shaped workload: 5000 seeded synthetic JPEG files (nine in ten with a long
side of 640 at COCO's common aspect ratios, the rest between 320 and 1024), up to 12 labels per image over 80 classes,
yolov5s with bench.py's synthetic weights, batch 32, img_size 640, conf 0.001, iou 0.6.

Prints, with the card's name and power limit:
  - run() end to end (files in, metrics out) with a host clock, after a warm-up pass, and its images/s;
  - the stages of the same loop with CUDA events between them, summed over the batches: decode (the ingest path of
    predict(paths)), resize (INTER_AREA / INTER_LINEAR), compose, plan (identity write + network), decode + NMS,
    rescale, update_padded, and compute() at the end.  Each stage's time runs from the event before its launches to
    the event after them, so host work that keeps the device waiting inside a stage is counted in it;
  - upstream's cv2 loader recipe (cv2.imread, cv2.resize INTER_AREA / INTER_LINEAR, copyMakeBorder, HWC -> CHW RGB) on
    8 host threads over the same files, for the loader's comparison with decode + resize + compose.

    python scripts/v5_val_times.py [--images 5000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_state_dict  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.models import yolov5s  # noqa: E402
from yolort_b200.v5 import val as V  # noqa: E402
from yolort_b200.v5.utils import datasets as D  # noqa: E402
from yolort_b200.v5.utils.general import rescale_params, scale_coords_padded  # noqa: E402
from yolort_b200.v5.utils.metrics import DetectionMetrics  # noqa: E402

STAGES = ("decode", "resize", "compose", "plan", "decode+nms", "rescale", "update_padded")
ASPECTS = ((480, 640), (640, 480), (427, 640), (640, 427), (360, 640), (640, 640), (424, 640), (640, 512))


def make_files(n, root):
    import cv2

    def one(i):
        rng = np.random.default_rng(i)
        if rng.random() < 0.9:
            h, w = ASPECTS[int(rng.integers(len(ASPECTS)))]
        else:
            long = int(rng.integers(320, 1025))
            short = int(long * rng.uniform(0.45, 1.0))
            h, w = (long, short) if rng.random() < 0.4 else (short, long)
        low = rng.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3), dtype=np.uint8)
        im = cv2.resize(low, (w, h), interpolation=cv2.INTER_CUBIC)
        im = np.clip(im.astype(np.int16) + rng.integers(-12, 13, im.shape), 0, 255).astype(np.uint8)
        path = os.path.join(root, f"{i:05d}.jpg")
        cv2.imwrite(path, im, [cv2.IMWRITE_JPEG_QUALITY, 90])
        k = int(rng.integers(0, 13))
        lab = np.concatenate([rng.integers(0, 80, (k, 1)), rng.uniform(0.1, 0.9, (k, 2)),
                              rng.uniform(0.02, 0.4, (k, 2))], 1).astype(np.float32)
        return path, lab

    with ThreadPoolExecutor(8) as pool:
        out = list(pool.map(one, range(n)))
    return [p for p, _ in out], [lab for _, lab in out]


def staged(model, paths, labels, bs, s, conf, iou, max_det):
    """run()'s loop with CUDA events between the stages; returns {stage: ms} and compute()'s ms."""
    yolo = model.model
    dev = next(yolo.parameters()).device
    sizes = V._image_sizes(paths)
    irect, bi, shapes_b = D.rect_batches(sizes, s, bs, int(max(yolo.anchor_generator.strides)))
    metrics = DetectionMetrics(yolo.num_classes, device=dev)
    marks = []
    for k in range(len(shapes_b)):
        idx = [int(i) for i in irect[bi == k]]
        H, W = (int(v) for v in shapes_b[k])
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        ev[0].record()
        images = [t.permute(1, 2, 0) for t in model._ingest_files([paths[i] for i in idx], dev)]
        ev[1].record()
        plan = D.ValPlan(images, [labels[i] for i in idx], range(len(idx)), (H, W), s, "rgb")
        plan.resize()
        ev[2].record()
        imgs = torch.empty((len(idx), 3, H, W), dtype=torch.uint8, device=dev)
        plan.compose(imgs)
        targets = plan.targets()
        ev[3].record()
        p = yolo.engine().plan(len(idx), H, W)
        yolo._write_samples(p, imgs)
        heads = yolo.run_plan(p)
        ev[4].record()
        pc = yolo.post_config()
        boxes, scores, cls, counts = _C.decode_nms_complete(heads, "nhwc", pc["strides"], pc["anchors_px"],
                                                            pc["num_classes"], conf, iou, max_det, pc["semantics"])[:4]
        ev[5].record()
        native = scale_coords_padded(boxes, counts, rescale_params(plan.shapes, dev), targets, (H, W))
        ev[6].record()
        metrics.update_padded(boxes, scores, cls, counts, native)
        ev[7].record()
        marks.append(ev)
    c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    c0.record()
    t = time.perf_counter()
    metrics.compute()
    compute_host = (time.perf_counter() - t) * 1e3
    c1.record()
    torch.cuda.synchronize()
    out = {st: sum(ev[j].elapsed_time(ev[j + 1]) for ev in marks) for j, st in enumerate(STAGES)}
    return out, c0.elapsed_time(c1), compute_host


def cv2_loader(paths, s, bs, threads=8):
    """Upstream's loader recipe per image, in rect order, on `threads` host threads: seconds for the whole set."""
    import cv2

    sizes = V._image_sizes(paths)
    irect, bi, shapes_b = D.rect_batches(sizes, s, bs)

    def one(j):
        i = int(irect[j])
        im = cv2.imread(paths[i])
        h0, w0 = im.shape[:2]
        r = s / max(h0, w0)
        if r != 1:
            im = cv2.resize(im, (int(w0 * r), int(h0 * r)), interpolation=cv2.INTER_AREA if r < 1 else cv2.INTER_LINEAR)
        (nh, nw), _, _, (top, bottom, left, right) = D.letterbox_arith(im.shape[:2], tuple(shapes_b[bi[j]]),
                                                                       auto=False, scaleup=False)
        if (nh, nw) != im.shape[:2]:
            im = cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR)
        im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        return np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])

    t = time.perf_counter()
    with ThreadPoolExecutor(threads) as pool:
        for _ in pool.map(one, range(len(paths)), chunksize=16):
            pass
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--img-size", type=int, default=640)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    model = yolov5s().eval()
    model.load_state_dict(make_state_dict(model))
    model = model.to("cuda:0")
    conf, iou, max_det, bs, s = 0.001, 0.6, 300, args.batch, args.img_size
    with tempfile.TemporaryDirectory() as root:
        t = time.perf_counter()
        paths, labels = make_files(args.images, root)
        gen_s = time.perf_counter() - t
        print(f"{len(paths)} files in {gen_s:.1f} s", file=sys.stderr, flush=True)
        with torch.no_grad():
            V.run(model, paths, labels, bs, s, conf, iou, max_det)           # warm-up: plans, arenas, decoders
            torch.cuda.synchronize()
            t = time.perf_counter()
            res = V.run(model, paths, labels, bs, s, conf, iou, max_det)
            torch.cuda.synchronize()
            run_s = time.perf_counter() - t
            print(f"run() {run_s:.2f} s", file=sys.stderr, flush=True)
            stages, compute_dev, compute_host = staged(model, paths, labels, bs, s, conf, iou, max_det)
        loader_s = cv2_loader(paths, s, bs)
    out = {
        "card": card, "images": args.images, "batch": bs, "img_size": s, "conf_thres": conf, "iou_thres": iou,
        "files_generated_s": round(gen_s, 1),
        "run_s": round(run_s, 3), "run_images_per_s": round(args.images / run_s, 1),
        "stages_ms": {k: round(v, 2) for k, v in stages.items()},
        "compute_ms_events": round(compute_dev, 2), "compute_ms_host": round(compute_host, 2),
        "staged_total_ms": round(sum(stages.values()) + compute_dev, 1),
        "loader_gpu_ms": round(stages["decode"] + stages["resize"] + stages["compose"], 1),
        "loader_cv2_8_threads_ms": round(loader_s * 1e3, 1),
        "map50": float(res["map50"]), "map": float(res["map"]),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
