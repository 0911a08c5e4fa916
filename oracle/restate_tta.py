"""CPU restatement of YOLOv5's test-time augmentation (`augment=True`) -- TEST INFRASTRUCTURE ONLY.

The reference composes it from `DetectionModel._forward_augment` (yolort/v5/models/yolo.py:152-163), `scale_img`
(yolort/v5/utils/torch_utils.py:288-300), `_descale_pred` (yolo.py:178-194), `_clip_augmented` (yolo.py:196-205) and
yolort's own letterbox, network and PostProcess pieces (yolort/models/transform.py, box_head.py:328-429).  The six
steps below follow that composition; the network is restate.Net, the NMS restate.batched_nms, the rescale
restate.scale_coords.  Paths are relative to the reference tree.
"""
import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import restate as R

f32 = np.float32
SCALES = (1.0, 0.83, 0.67)      # yolo.py:154
FLIPS = (None, 3, None)         # yolo.py:155 (3: left-right)
FILL = 0.447                    # torch_utils.py:300


def pass_geometry(Hb: int, Wb: int, gs: int) -> List[Tuple[int, int, int, int]]:
    """(nh, nw, Hp, Wp) per pass: torch_utils.py:293-299 (Python doubles); scale 1 returns the canvas (:292)."""
    out = []
    for s in SCALES:
        if s == 1.0:
            out.append((Hb, Wb, Hb, Wb))
        else:
            out.append((int(Hb * s), int(Wb * s), math.ceil(Hb * s / gs) * gs, math.ceil(Wb * s / gs) * gs))
    return out


def scale_img(x: np.ndarray, ratio: float, flip: Optional[int], gs: int) -> np.ndarray:
    """Step 2: scale_img(x.flip(3) if flip else x, ratio, gs) on an fp32 [N, 3, H, W] batch (torch_utils.py:288-300):
    bilinear resize to int(H*r) x int(W*r), then F.pad right / bottom with 0.447 to the gs-multiple.  The resize is
    torch's own CPU upsample_bilinear2d (align_corners=False): on whole batches its kernel rounds differently from
    restate.bilinear_resize in the last fp32 bit, and it is the reference's arithmetic."""
    x = np.asarray(x, dtype=np.float32)
    if flip == 3:
        x = x[..., ::-1]
    if ratio == 1.0:
        return np.ascontiguousarray(x)
    n, c, h, w = x.shape
    nh, nw, hp, wp = pass_geometry(h, w, gs)[SCALES.index(ratio)]
    out = np.full((n, c, hp, wp), f32(FILL), dtype=np.float32)
    t = torch.from_numpy(np.ascontiguousarray(x))
    out[:, :, :nh, :nw] = F.interpolate(t, size=(nh, nw), mode="bilinear", align_corners=False).numpy()
    return out


def concat_pred(head_outputs: List[torch.Tensor], strides, anchor_grids) -> np.ndarray:
    """Step 3: _concat_pred_logits (box_head.py:328-348) -> [N, n, K] = (cx, cy, w, h, obj, cls...), fp32; the same
    arithmetic as the first half of restate.decode."""
    per_level = []
    for lvl, t in enumerate(head_outputs):
        t = t.float()
        n, a, h, w, k = t.shape
        y = torch.sigmoid(t)
        gx = torch.arange(w, dtype=torch.int32).float().view(1, 1, 1, w).expand(1, a, h, w)
        gy = torch.arange(h, dtype=torch.int32).float().view(1, 1, h, 1).expand(1, a, h, w)
        grid = torch.stack((gx, gy), -1)
        anc = torch.tensor(anchor_grids[lvl], dtype=torch.float32).view(-1, 2)
        st = torch.tensor(float(strides[lvl]), dtype=torch.float32)
        shift = ((anc / st) * strides[lvl]).view(1, a, 1, 1, 2)
        xy = (y[..., 0:2] * 2.0 - 0.5 + grid) * st
        wh = (y[..., 2:4] * 2.0) ** 2 * shift
        per_level.append(torch.cat((xy, wh, y[..., 4:]), -1).view(n, -1, k))
    return torch.cat(per_level, 1).numpy()


def descale(p: np.ndarray, flip: Optional[int], scale: float, img_size: Tuple[int, int]) -> np.ndarray:
    """Step 4: _descale_pred with inplace=True (yolo.py:180-185): p[..., :4] /= scale (fp32 division by fp32(scale)),
    then x = W - x for the left-right flip."""
    p = np.array(p, dtype=np.float32, copy=True)
    p[..., :4] = p[..., :4] / f32(scale)
    if flip == 2:
        p[..., 1] = f32(img_size[0]) - p[..., 1]
    elif flip == 3:
        p[..., 0] = f32(img_size[1]) - p[..., 0]
    return p


def clip_augmented(y: List[np.ndarray], nl: int) -> List[np.ndarray]:
    """Step 5: _clip_augmented (yolo.py:196-205), its index arithmetic as written."""
    g = sum(4 ** x for x in range(nl))
    e = 1
    y = list(y)
    i = (y[0].shape[1] // g) * sum(4 ** x for x in range(e))
    y[0] = y[0][:, :-i]
    i = (y[-1].shape[1] // g) * sum(4 ** (nl - 1 - x) for x in range(e))
    y[-1] = y[-1][:, i:]
    return y


def postprocess_pred(pred: np.ndarray, score_thresh: float, nms_thresh: float, detections_per_img: int,
                     semantics: int = R.TV_AUTO):
    """Step 6: _decode_pred_logits (box_head.py:351-360) + PostProcess.forward's loop (:410-427) on [N, n, K]."""
    t = torch.from_numpy(np.ascontiguousarray(pred))
    scores_all = (t[..., 5:] * t[..., 4:5]).numpy()
    cx, cy, w, h = t[..., 0], t[..., 1], t[..., 2], t[..., 3]
    boxes_all = torch.stack((cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h), -1).numpy()
    thr = f32(score_thresh)
    out = []
    for i in range(pred.shape[0]):
        b, s = boxes_all[i], scores_all[i]
        inds, labels = np.nonzero(s > thr)
        cb, cs = b[inds], s[inds, labels]
        keep = R.batched_nms(cb, cs, labels, nms_thresh, semantics)[:detections_per_img]
        out.append({"scores": cs[keep], "labels": labels[keep].astype(np.int64), "boxes": cb[keep],
                    "n_candidates": int(inds.shape[0])})
    return out


def augmented_pred(net: "R.Net", samples: np.ndarray, strides, anchor_grids,
                   canvases: Optional[Sequence[np.ndarray]] = None) -> np.ndarray:
    """Steps 2-5 (_forward_augment, yolo.py:152-163): [N, n_total, K] in concatenation order.  `canvases` replaces the
    pass inputs (the GPU tests feed the canvases the device computed in fp16 / bf16)."""
    Hb, Wb = int(samples.shape[2]), int(samples.shape[3])
    gs = int(max(strides))
    y = []
    for q, (s, f) in enumerate(zip(SCALES, FLIPS)):
        xi = canvases[q] if canvases is not None else scale_img(samples, s, f, gs)
        with torch.no_grad():
            heads = net.head(net.backbone(torch.from_numpy(np.ascontiguousarray(xi, dtype=np.float32))),
                             num_anchors=len(anchor_grids[0]) // 2)
        y.append(descale(concat_pred(heads, strides, anchor_grids), f, s, (Hb, Wb)))
    return np.concatenate(clip_augmented(y, len(strides)), 1)


def detect(state_dict, images: Sequence[torch.Tensor], score_thresh: float = 0.005, nms_thresh: float = 0.45,
           detections_per_img: int = 300, size=(640, 640), size_divisible: int = 32, fill_color: int = 114,
           semantics: int = R.TV_AUTO, strides=R.DEFAULT_STRIDES, anchor_grids=R.DEFAULT_ANCHORS,
           net: Optional["R.Net"] = None):
    """YOLOv5.forward(images, augment=True) end to end on the CPU in fp32: step 1 (restate.letterbox), steps 2-6,
    scale_coords against (Hb, Wb) (transform.py:332-367).  `net`: the network restatement (default restate.Net of
    `state_dict`; e.g. restate_ts.NetTS for yolov5ts, restate_fp8.NetFP8 for the fake-quant FP8 network)."""
    batch, _, _ = R.letterbox(images, float(size[0]), float(size[1]), size_divisible, None, fill_color)
    samples = batch.numpy()
    net = R.Net(state_dict) if net is None else net
    pred = augmented_pred(net, samples, strides, anchor_grids)
    dets = postprocess_pred(pred, score_thresh, nms_thresh, detections_per_img, semantics)
    Hb, Wb = int(samples.shape[2]), int(samples.shape[3])
    for d, im in zip(dets, images):
        d["boxes"] = R.scale_coords(d["boxes"], Hb, Wb, int(im.shape[-2]), int(im.shape[-1]))
    return dets
