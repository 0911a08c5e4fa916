"""Fixtures of YOLOv5's test-time augmentation from the UNMODIFIED reference -- TEST INFRASTRUCTURE ONLY.

Calls the reference's own pieces (paths relative to the reference tree): scale_img (yolort/v5/utils/torch_utils.py:
288-300); DetectionModel._descale_pred and _clip_augmented (yolort/v5/models/yolo.py:178-205), unbound on stub
`self` objects (no DetectionModel is built); yolort's YOLOv5 transform, backbone, head, anchor generator and
PostProcess pieces (box_head.py:328-429, transform.py:332-367) on synth_state_dict weights.  Writes
tests/golden/{tta.npz, tta_geometry.json, e2e_tta_n.npz, e2e_tta_n6.npz}.
"""
import json
import math
import os
import types

import numpy as np
import torch

from . import ref_import
from .make_golden import GOLDEN, synth_image_u8, synth_state_dict
from .make_golden_p6 import GAIN_N6

SCALES, FLIPS = (1, 0.83, 0.67), (None, 3, None)        # yolo.py:154-155


def main():
    ref_import.import_reference()
    from yolort.models import yolov5n, yolov5n6
    from yolort.models.box_head import _concat_pred_logits, _decode_pred_logits
    from yolort.v5.models.yolo import DetectionModel
    from yolort.v5.utils.torch_utils import scale_img
    from torchvision.ops import boxes as box_ops

    torch.set_num_threads(8)
    stub = types.SimpleNamespace(inplace=True)

    # 1. pass geometry over a sweep of canvases ----------------------------------------------------------------------
    geo = []
    for gs in (32, 64):
        for h in range(gs, 1281, gs):
            for w in sorted({gs, h, 1280, 640, 608 if gs == 32 else 576}):
                x = torch.zeros(1, 1, h, w)
                entry = {"gs": gs, "H": h, "W": w, "passes": []}
                for s in SCALES:
                    y = scale_img(x, s, gs=gs)
                    entry["passes"].append([int(h * s), int(w * s), int(y.shape[2]), int(y.shape[3])])
                geo.append(entry)
    with open(os.path.join(GOLDEN, "tta_geometry.json"), "w") as f:
        json.dump(geo, f, separators=(",", ":"))

    # 2. canvases (mirrored and not), descale and clip ---------------------------------------------------------------
    z = {}
    g = torch.Generator().manual_seed(5)
    # one image each, small enough to keep the fixture small; width 608 gives the odd widths 504 / 407
    shapes = [(64, 64, 32), (64, 96, 32), (16, 608, 32), (64, 128, 64)]
    z["canvas_shapes"] = np.array(shapes, dtype=np.int64)
    for c, (h, w, gs) in enumerate(shapes):
        x = torch.rand(1, 3, h, w, generator=g)
        x[:, :, : h // 4] = 0.447                       # a letterbox-like flat band
        z[f"c{c}_x"] = x.numpy()
        for q, s in enumerate(SCALES):
            if q == 0:
                continue                                # scale 1 returns its input (torch_utils.py:291-292)
            for flip in (None, 3):
                z[f"c{c}_s{q}_f{flip or 0}"] = scale_img(x.flip(flip) if flip else x, s, gs=gs).numpy()
    p = torch.randn(2, 21 * 12, 7, generator=g) * 40.0 + 60.0
    z["pred"] = p.numpy()
    for q, (s, f) in enumerate(zip(SCALES, FLIPS)):
        z[f"descale{q}"] = DetectionModel._descale_pred(stub, p.clone(), f, s, (96, 160)).numpy()
    # per-pass predictions of a 3-level model: 8x8 / 4x4 / 2x2 maps twice, then 4x4 / 2x2 / 1x1
    ys = [torch.randn(2, n, 7, generator=g) for n in (3 * (64 + 16 + 4), 3 * (64 + 16 + 4), 3 * (16 + 4 + 1))]
    clip_stub = types.SimpleNamespace(model=[types.SimpleNamespace(nl=3)])
    clipped = DetectionModel._clip_augmented(clip_stub, [y.clone() for y in ys])
    for k, (y, c) in enumerate(zip(ys, clipped)):
        z[f"clip_in{k}"], z[f"clip_out{k}"] = y.numpy(), c.numpy()
    np.savez_compressed(os.path.join(GOLDEN, "tta.npz"), **z)

    # 3. end to end: two images of different sizes on a 128 x 128 canvas -------------------------------------------------
    with open(os.path.join(GOLDEN, "state_dict_layouts.json")) as f:
        lay_n = json.load(f)["n"]
    with open(os.path.join(GOLDEN, "state_dict_layouts_p6.json")) as f:
        lay_n6 = json.load(f)["n6"]
    cases = {"n": (yolov5n, lay_n, None, 32, (synth_image_u8(90, 128, 21), synth_image_u8(100, 75, 22))),
             "n6": (yolov5n6, lay_n6, GAIN_N6, 64, (synth_image_u8(128, 96, 31), synth_image_u8(70, 128, 32)))}
    for name, (ctor, lay, gain, gs, ims) in cases.items():
        kw = {} if gain is None else {"gain": gain}
        sd = synth_state_dict(lay, knob_obj=7.0, knob_cls=4.5, seed=0, **kw)
        m = ctor(size=(128, 128), score_thresh=0.15).eval()       # yolov5n6 pins size_divisible=64
        m.load_state_dict(sd)
        images = [im / 255.0 for im in ims]
        with torch.no_grad():
            samples, _ = m.transform(images)
            x = samples.tensors
            Hb, Wb = int(x.shape[2]), int(x.shape[3])
            assert int(max(m.model.anchor_generator.strides)) == gs
            y = []
            for s, f in zip(SCALES, FLIPS):
                xi = scale_img(x.flip(f) if f else x, s, gs=gs)
                feats = m.model.backbone(xi)
                heads = m.model.head(feats)
                grids, shifts = m.model.anchor_generator(feats)
                strides = torch.as_tensor(m.model.post_process.strides, dtype=torch.float32)
                pi = _concat_pred_logits(heads, grids, shifts, strides)
                y.append(DetectionModel._descale_pred(stub, pi, f, s, (Hb, Wb)))
            y = DetectionModel._clip_augmented(types.SimpleNamespace(model=[types.SimpleNamespace(nl=len(heads))]), y)
            pred = torch.cat(y, 1)
            pp = m.model.post_process
            dets = []
            for i in range(pred.shape[0]):
                boxes, scores = _decode_pred_logits(pred[i])
                inds, labels = torch.where(scores > pp.score_thresh)
                boxes, scores = boxes[inds], scores[inds, labels]
                keep = box_ops.batched_nms(boxes, scores, labels, pp.nms_thresh)[: pp.detections_per_img]
                dets.append({"scores": scores[keep], "labels": labels[keep], "boxes": boxes[keep]})
            out = m.transform.postprocess(dets, torch.tensor([Hb, Wb]), [(int(im.shape[-2]), int(im.shape[-1])) for im in ims])
        np.savez_compressed(os.path.join(GOLDEN, f"e2e_tta_{name}.npz"), img0=ims[0].numpy(), img1=ims[1].numpy(),
                            canvas=np.array([Hb, Wb]), n_pred=np.int64(pred.shape[1]),
                            **{f"det{i}_{k}": v.numpy() for i, d in enumerate(out) for k, v in d.items()})
        print(name, "canvas", (Hb, Wb), "passes", [tuple(int(v) for v in t.shape[1:]) for t in y],
              "dets", [len(d["scores"]) for d in out])


if __name__ == "__main__":
    main()
