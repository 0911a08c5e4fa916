"""Torch restatement of YOLOv5's training loss: the reference's SetCriterion (yolort/models/box_head.py:85-325),
written from the rules below and checked against the unmodified reference by tests/golden/loss.npz
(oracle/make_golden_loss.py).  TEST INFRASTRUCTURE ONLY: it runs on any device, in fp32 or fp64, with autograd.

Rule 1 (anchors, box_head.py:167-171).  Anchors in grid units are anchor_px / stride, both fp32.
Rule 2 (ratio test, :271-281).  For level i with head shape [N, A, H, W, K] the gain is (W, H) (shape indices 3, 2);
    gwh = (w, h) * gain in fp32.  A target matches anchor a when max(r, 1 / r) over w and h is < anchor_thresh, with
    r = gwh / anchor and the comparison made in fp32 (the threshold is rounded to fp32 first).
Rule 3 (offsets, :284-298).  gxy = (cx, cy) * gain and gxi = gain - gxy, fp32.  Offset 0 (0, 0) always applies;
    offsets 1, 2 ((+0.5, 0), (0, +0.5)) when gxy % 1 < 0.5 and gxy > 1 for x, y; offsets 3, 4 ((-0.5, 0), (0, -0.5))
    when gxi % 1 < 0.5 and gxi > 1.  The matches of a level are ordered offset-major, then anchor, then target.
Rule 4 (indices, :304-323).  b and class are the target's columns truncated (`.long()`); (gi, gj) = (gxy - offset)
    truncated, then clamped to [0, W-1] and [0, H-1]; tbox = (gxy - (gi, gj), gwh) with the CLAMPED indices; the anchor
    is the match's anchor in grid units.
Rule 5 (box loss, :190-195, _utils.py:26-40, :65-108).  The logits at (b, a, gj, gi) are decoded as
    xy = 2 sigmoid - 0.5, wh = (2 sigmoid)^2 anchor; CIoU with eps 1e-7 against tbox, alpha = v / (v - iou + 1 + eps)
    held constant for the gradient; the level adds mean(1 - CIoU).
Rule 6 (objectness, :197-217).  target_obj[b, a, gj, gi] = (1 - gr) + gr * clamp(CIoU, 0), written in match order, so
    for a cell matched twice the later match wins; obj_i = BCE-with-logits(logit 4, target_obj, pos_weight=obj_pos)
    averaged over every cell of the level; the loss adds obj_i * balance[i].
Rule 7 (class loss, :205-212).  When num_classes > 1: targets smooth_neg everywhere and smooth_pos at the class,
    BCE-with-logits with pos_weight=cls_pos averaged over the level's matches x classes.
Rule 8 (gains, :223-225).  box, obj and cls are multiplied by box_gain, obj_gain and cls_gain.
"""
import math
from typing import Dict, List, Sequence

import torch

EPS = 1e-7
OFFSETS = ((0.0, 0.0), (0.5, 0.0), (0.0, 0.5), (-0.5, 0.0), (0.0, -0.5))
BALANCE_DEFAULTS = (4.0, 1.0, 0.4, 0.1)


def grid_anchors(anchor_grids: Sequence[Sequence[float]], strides: Sequence[int], device=None) -> torch.Tensor:
    """Rule 1: fp32 [L, A, 2]."""
    a = torch.tensor(anchor_grids, dtype=torch.float32, device=device).view(len(strides), -1, 2)
    s = torch.tensor([float(x) for x in strides], dtype=torch.float32, device=device).view(-1, 1, 1)
    return a / s


def assign(targets: torch.Tensor, shapes: Sequence[Sequence[int]], anchors: torch.Tensor,
           anchor_thresh: float) -> List[Dict[str, torch.Tensor]]:
    """Rules 2-4 in fp32.  targets [T, 6] = (image, class, cx, cy, w, h).  Returns per level the matches in order:
    b, a, gj, gi, cls (int64), tbox fp32 [M, 4], anchor fp32 [M, 2]."""
    t = targets.to(torch.float32)
    T, A = t.shape[0], anchors.shape[1]
    dev = t.device
    thresh = torch.tensor(anchor_thresh, dtype=torch.float32, device=dev)
    half = torch.tensor(0.5, dtype=torch.float32, device=dev)
    one = torch.tensor(1.0, dtype=torch.float32, device=dev)
    out = []
    for i, shp in enumerate(shapes):
        H, W = int(shp[2]), int(shp[3])
        gain = torch.tensor([W, H], dtype=torch.float32, device=dev)
        gxy = t[:, 2:4] * gain                                  # [T, 2]
        gwh = t[:, 4:6] * gain
        gxi = gain - gxy
        r = gwh[None] / anchors[i][:, None]                     # [A, T, 2]
        ratio_ok = torch.maximum(r, torch.reciprocal(r)).amax(2) < thresh       # [A, T]
        lo = (torch.remainder(gxy, 1.0) < half) & (gxy > one)                   # [T, 2]
        hi = (torch.remainder(gxi, 1.0) < half) & (gxi > one)
        take = torch.stack([torch.ones_like(lo[:, 0]), lo[:, 0], lo[:, 1], hi[:, 0], hi[:, 1]])   # [5, T]
        mask = ratio_ok[None] & take[:, None]                  # [5, A, T]: (offset, anchor, target) order
        o_idx, a_idx, t_idx = mask.nonzero(as_tuple=True)      # row-major: offset-major, then anchor, then target
        off = torch.tensor(OFFSETS, dtype=torch.float32, device=dev)[o_idx]
        mg = gxy[t_idx]
        gij = (mg - off).long()
        gi = gij[:, 0].clamp(0, W - 1)
        gj = gij[:, 1].clamp(0, H - 1)
        tbox = torch.cat([mg - torch.stack([gi, gj], 1), gwh[t_idx]], 1)
        out.append({"b": t[t_idx, 0].long(), "a": a_idx, "gj": gj, "gi": gi, "cls": t[t_idx, 1].long(),
                    "tbox": tbox, "anchor": anchors[i][a_idx]})
    return out


def ciou(pbox: torch.Tensor, tbox: torch.Tensor) -> torch.Tensor:
    """Rule 5: CIoU of xywh boxes [M, 4]; alpha carries no gradient."""
    px1, px2 = pbox[:, 0] - pbox[:, 2] / 2, pbox[:, 0] + pbox[:, 2] / 2
    py1, py2 = pbox[:, 1] - pbox[:, 3] / 2, pbox[:, 1] + pbox[:, 3] / 2
    tx1, tx2 = tbox[:, 0] - tbox[:, 2] / 2, tbox[:, 0] + tbox[:, 2] / 2
    ty1, ty2 = tbox[:, 1] - tbox[:, 3] / 2, tbox[:, 1] + tbox[:, 3] / 2
    inter = ((torch.minimum(px2, tx2) - torch.maximum(px1, tx1)).clamp(0)
             * (torch.minimum(py2, ty2) - torch.maximum(py1, ty1)).clamp(0))
    w1, h1 = px2 - px1, py2 - py1 + EPS
    w2, h2 = tx2 - tx1, ty2 - ty1 + EPS
    iou = inter / (w1 * h1 + w2 * h2 - inter + EPS)
    cw = torch.maximum(px2, tx2) - torch.minimum(px1, tx1)
    ch = torch.maximum(py2, ty2) - torch.minimum(py1, ty1)
    c2 = cw ** 2 + ch ** 2 + EPS
    rho2 = ((tx1 + tx2 - px1 - px2) ** 2 + (ty1 + ty2 - py1 - py2) ** 2) / 4
    v = (4 / math.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    with torch.no_grad():
        alpha = v / (v - iou + (1 + EPS))
    return iou - (rho2 / c2 + v * alpha)


def bce_logits(x: torch.Tensor, t, pos_weight: float) -> torch.Tensor:
    """Elementwise BCE-with-logits in torch's stable form."""
    lw = 1 + (pos_weight - 1) * t
    return (1 - t) * x + lw * (torch.log1p(torch.exp(-x.abs())) + (-x).clamp(min=0))


def loss(targets: torch.Tensor, head_outputs: Sequence[torch.Tensor], strides: Sequence[int],
         anchor_grids: Sequence[Sequence[float]], num_classes: int, box_gain: float = 0.05, cls_gain: float = 0.5,
         cls_pos: float = 1.0, obj_gain: float = 1.0, obj_pos: float = 1.0, anchor_thresh: float = 4.0,
         label_smoothing: float = 0.0, balance: Sequence[float] = None, gr: float = 1.0):
    """Rules 1-8.  Arithmetic in the head outputs' dtype (fp32 or fp64; the assignment stays fp32).  Returns
    ({"cls_logits", "bbox_regression", "objectness"} as shape-[1] tensors, [obj_i per level], assignment)."""
    dev = head_outputs[0].device
    dt = head_outputs[0].dtype
    if balance is None:
        balance = BALANCE_DEFAULTS[: len(strides)]
    smooth_pos, smooth_neg = 1.0 - 0.5 * label_smoothing, 0.5 * label_smoothing
    anchors = grid_anchors(anchor_grids, strides, dev)
    asg = assign(targets.to(dev), [p.shape for p in head_outputs], anchors, anchor_thresh)
    lbox = torch.zeros(1, dtype=dt, device=dev)
    lcls = torch.zeros(1, dtype=dt, device=dev)
    lobj = torch.zeros(1, dtype=dt, device=dev)
    objs = []
    for i, p in enumerate(head_outputs):
        m = asg[i]
        tobj = torch.zeros_like(p[..., 0]).detach()
        if m["b"].numel():
            sub = p[m["b"], m["a"], m["gj"], m["gi"]]
            s = sub[:, :4].sigmoid()
            pbox = torch.cat([s[:, :2] * 2.0 - 0.5, (s[:, 2:4] * 2) ** 2 * m["anchor"].to(dt)], 1)
            c = ciou(pbox, m["tbox"].to(dt))
            lbox = lbox + (1.0 - c).mean()
            score = (1.0 - gr) + gr * c.detach().clamp(0)
            # the later match of a cell wins, on any device: the owner is the largest match index of the cell
            cell = ((m["b"] * p.shape[1] + m["a"]) * p.shape[2] + m["gj"]) * p.shape[3] + m["gi"]
            idx = torch.arange(cell.numel(), device=dev)
            owner = torch.full((tobj.numel(),), -1, dtype=torch.int64, device=dev).scatter_reduce(0, cell, idx, "amax")
            own = owner[cell] == idx
            tobj.view(-1)[cell[own]] = score[own]
            if num_classes > 1:
                tc = torch.full_like(sub[:, 5:], smooth_neg).detach()
                tc[torch.arange(sub.shape[0], device=dev), m["cls"]] = smooth_pos
                lcls = lcls + bce_logits(sub[:, 5:], tc, cls_pos).mean()
        obji = bce_logits(p[..., 4], tobj, obj_pos).mean()
        objs.append(obji)
        lobj = lobj + obji * balance[i]
    return ({"cls_logits": lcls * cls_gain, "bbox_regression": lbox * box_gain, "objectness": lobj * obj_gain},
            objs, asg)


def update_balance(balance: Sequence[float], objs: Sequence[float], ssi: int) -> List[float]:
    """auto_balance (box_head.py:218-222) in Python floats."""
    b = [x * 0.9999 + 0.0001 / float(o) for x, o in zip(balance, objs)]
    return [x / b[ssi] for x in b]
