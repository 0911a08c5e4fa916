"""COCO box AP of a model over an image directory and its annotation file, on one GPU: the counterpart of the
reference's tools/eval_metric.py.  Images go through `predict_stream(paths)` (baseline JPEGs decode on the device)
and the detections through `yolort_b200.data.COCOEvaluator`.  With --fp8-calib-batches N the model is calibrated on
the first N batches and fp16 and FP8 AP are reported side by side.

    python scripts/eval_coco.py --arch yolov5s --checkpoint yolov5s.pt \
        --images coco/val2017 --annotations coco/annotations/instances_val2017.json --batch-size 32
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import yolort_b200.models as M  # noqa: E402
from yolort_b200.data import COCOEvaluator  # noqa: E402


def evaluate(model, ann, paths, ids, batch_size, eval_type, device):
    ev = COCOEvaluator(ann, eval_type=eval_type, device=device)
    batches = [paths[i:i + batch_size] for i in range(0, len(paths), batch_size)]
    t0 = time.perf_counter()
    for b, out in enumerate(model.predict_stream(batches)):
        ev.update(out, ids[b * batch_size:(b + 1) * batch_size])
    res = ev.compute()
    res["seconds"] = time.perf_counter() - t0
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--arch", default="yolov5s")
    ap.add_argument("--checkpoint", default=None, help="an upstream YOLOv5 checkpoint (load_from_yolov5)")
    ap.add_argument("--version", default="r6.0", help="upstream release of the checkpoint")
    ap.add_argument("--images", required=True, help="directory holding the annotation file's file_names")
    ap.add_argument("--annotations", required=True, help="COCO annotation JSON")
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--score-thresh", type=float, default=0.005)
    ap.add_argument("--eval-type", default="yolov5", choices=["yolov5", "torchvision"])
    ap.add_argument("--fp8-calib-batches", type=int, default=0)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()

    dev = torch.device(args.device)
    if args.checkpoint:
        model = M.YOLOv5.load_from_yolov5(args.checkpoint, size=(args.size, args.size),
                                          score_thresh=args.score_thresh, version=args.version)
    else:
        model = getattr(M, args.arch)(score_thresh=args.score_thresh, size=(args.size, args.size))
        print(f"no --checkpoint: {args.arch} with its initial weights", file=sys.stderr)
    model = model.eval().to(dev)
    with open(args.annotations) as f:
        ann = json.load(f)
    images = sorted(ann["images"], key=lambda im: im["id"])
    paths = [os.path.join(args.images, im["file_name"]) for im in images]
    ids = [im["id"] for im in images]

    out = {"arch": args.arch, "checkpoint": args.checkpoint, "images": len(paths),
           "fp16": evaluate(model, ann, paths, ids, args.batch_size, args.eval_type, dev)}
    if args.fp8_calib_batches > 0:
        from torchvision.io import ImageReadMode, read_image

        from yolort_b200.quantization import calibrate_fp8

        n = args.fp8_calib_batches * args.batch_size
        calib = [[read_image(p, mode=ImageReadMode.RGB).to(dev) for p in paths[i:i + args.batch_size]]
                 for i in range(0, min(n, len(paths)), args.batch_size)]
        model.set_fp8(calibrate_fp8(model, calib))
        out["fp8"] = evaluate(model, ann, paths, ids, args.batch_size, args.eval_type, dev)
        out["fp8_calib_images"] = min(n, len(paths))
        model.set_fp8(None)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
