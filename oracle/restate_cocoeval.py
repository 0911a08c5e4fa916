"""COCO box evaluation restated in plain numpy, written from the published COCO detection protocol in the arithmetic
of its reference implementation.  Slow and obvious on purpose: it is the yardstick the device evaluator
(yolort_b200.data.COCOEvaluator) is compared with bit for bit.  The product never imports it.

The rules (the kernels in yolort_b200/csrc/coco_eval.cu cite these numbers):

1. Parameters.  iouThrs = np.linspace(.5, .95, 10), recThrs = np.linspace(0, 1, 101), maxDets = [1, 10, 100], area
   ranges [0, 1e10], [0, 32^2], [32^2, 96^2], [96^2, 1e10], both ends inclusive.  Computed once by numpy, never
   re-derived: iouThrs[8] is 0.8999999999999999 and several recall thresholds are not round decimals.
2. Which images count.  Only images passed to update are evaluated; a repeated image id keeps its first update call,
   and within one call its last entry.  Images are taken in ascending id.  A detection on an image id the file does
   not have is an error, and so is a label outside the label map ("yolov5": label l -> sorted(category ids)[l];
   "torchvision": label l -> category id l, for 0 <= l <= the largest id).  Categories are the file's, ascending;
   detections of another category id are not evaluated.
3. Detections.  xyxy -> xywh in fp32 (w = x2 - x1, h = y2 - y1 rounded to fp32), float64 from there on.  Area = w*h
   (float64), not crowd, not ignored.  Per (image, category): stable sort by score descending (ties keep the
   prediction-list order), keep the first 100.
4. GT.  ignore = iscrowd.  For area range a, gtIg = ignore or area < lo or area > hi, with `area` the annotation's
   area field.  Per (image, category) GT keep file order, then are stably sorted so that gtIg == 0 come first.
5. IoU, float64, each operation rounded: w = min(dx+dw, gx+gw) - max(dx, gx), likewise h; IoU 0 if w <= 0 or
   h <= 0.  i = w*h; u = da for a crowd GT, else (da + ga) - i, with da = dw*dh and ga = gw*gh; IoU = i / u.
6. Greedy matching per (image, category, area, threshold t), detections in sorted order.  Candidates: GT not yet
   matched at t (a crowd GT may match any number of times) with IoU >= min(t, 1 - 1e-10).  The detection takes the
   last index of the maximum IoU among the non-ignored candidates, or, when there is none, among the ignored ones.
   A match copies the GT's gtIg into dtIg.  "Matched" means the GT's id is nonzero (a GT with id 0 counts as no
   match); a detection without such a match also gets dtIg = 1 when its area is outside the range.
7. Accumulation per (category, area, maxDets m), over the evaluated images with a GT or a detection of the category:
   the first m sorted detections of each image, concatenated in image order, stably sorted by score descending.
   npig = number of gtIg == 0 GT; with no such image or npig == 0 the entries stay -1.  tp = matched and not dtIg,
   fp = not matched and not dtIg, cumulated as integers, then float64.  rc = tp / npig, pr = tp / ((fp + tp) +
   2^-52).  recall = rc[-1] (0 without detections).  pr becomes its suffix maximum; for each recall threshold r,
   i = searchsorted(rc, r, 'left'); precision = pr[i] and score = score[i] if i < nd, else 0.
8. Summary.  stats[n] = np.mean(s[s > -1]) (or -1) over the slices COCOeval.summarize takes, on the host.
"""
from collections import defaultdict

import numpy as np

# rule 1
IOU_THRS = np.linspace(.5, .95, 10)
REC_THRS = np.linspace(0, 1, 101)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0.0, 1e10], [0.0, 32.0 ** 2], [32.0 ** 2, 96.0 ** 2], [96.0 ** 2, 1e10]]
EPS = np.spacing(1)   # 2^-52


def category_map(gt, eval_type):
    """label -> category id, as a function that raises ValueError outside the map (rule 2)."""
    cat_ids = sorted(int(c["id"]) for c in gt["categories"])
    if eval_type == "yolov5":
        def f(label):
            if not 0 <= label < len(cat_ids):
                raise ValueError(f"label {label} is outside the yolov5 map of {len(cat_ids)} categories")
            return cat_ids[label]
    elif eval_type == "torchvision":
        def f(label):
            if not 0 <= label <= cat_ids[-1]:
                raise ValueError(f"label {label} is outside the torchvision map [0, {cat_ids[-1]}]")
            return label
    else:
        raise NotImplementedError(eval_type)
    return f


def select_images(calls):
    """rule 2: calls = [[(image_id, (boxes_xyxy, scores, labels)), ...], ...] -> {image_id: detections}."""
    kept = {}
    for call in calls:
        within = {}
        for image_id, det in call:
            within[int(image_id)] = det          # the last entry of a call wins
        for image_id, det in within.items():
            if image_id not in kept:             # the first call wins
                kept[image_id] = det
    return kept


def iou(d, g, crowd):
    """rule 5 (Python floats are IEEE float64 and Python never fuses a multiply-add)."""
    dx, dy, dw, dh = d
    gx, gy, gw, gh = g
    w = min(dx + dw, gx + gw) - max(dx, gx)
    if w <= 0:
        return 0.0
    h = min(dy + dh, gy + gh) - max(dy, gy)
    if h <= 0:
        return 0.0
    i = w * h
    u = dw * dh if crowd else (dw * dh + gw * gh) - i
    return i / u


def evaluate_pair(dts, gts):
    """rules 3, 4, 6 for one (image, category): per area, (scores [D], matched [T,D], dtIg [T,D], gtIg [G])."""
    order = sorted(range(len(dts)), key=lambda p: -dts[p]["score"])   # Python's sort is stable
    dts = [dts[p] for p in order][:MAX_DETS[-1]]
    ious = [[iou(d["bbox"], g["bbox"], g["crowd"]) for g in gts] for d in dts]
    out = []
    for lo, hi in AREA_RNG:
        gt_ig = [g["crowd"] or g["area"] < lo or g["area"] > hi for g in gts]
        groups = ([gi for gi in range(len(gts)) if not gt_ig[gi]], [gi for gi in range(len(gts)) if gt_ig[gi]])
        matched = np.zeros((len(IOU_THRS), len(dts)), bool)
        dt_ig = np.zeros((len(IOU_THRS), len(dts)), bool)
        for t, thr in enumerate(IOU_THRS):
            thr = min(thr, 1 - 1e-10)
            taken = [False] * len(gts)
            for di, d in enumerate(dts):
                m = -1
                for group in groups:
                    cands = [gi for gi in group if (gts[gi]["crowd"] or not taken[gi]) and ious[di][gi] >= thr]
                    if cands:
                        best = max(ious[di][gi] for gi in cands)
                        m = [gi for gi in cands if ious[di][gi] == best][-1]
                        break
                if m >= 0:
                    taken[m] = True
                    dt_ig[t, di] = gt_ig[m]
                    matched[t, di] = gts[m]["id"] != 0
                if not matched[t, di] and (d["area"] < lo or d["area"] > hi):
                    dt_ig[t, di] = True
        out.append((np.array([d["score"] for d in dts], np.float64), matched, dt_ig, np.array(gt_ig, bool)))
    return out


def evaluate(gt, calls, eval_type="yolov5"):
    """gt: a parsed COCO annotation dict.  calls: one list per update call of (image_id, (boxes xyxy, scores,
    labels)).  Returns (eval = {"precision", "recall", "scores"}, stats)."""
    to_cat = category_map(gt, eval_type)
    image_set = {int(im["id"]) for im in gt["images"]}
    cat_ids = sorted(int(c["id"]) for c in gt["categories"])
    kept = select_images(calls)
    img_ids = sorted(kept)
    dts = defaultdict(list)
    for image_id in img_ids:
        boxes, scores, labels = kept[image_id]
        boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
        scores = np.asarray(scores, np.float32).reshape(-1)
        labels = np.asarray(labels).reshape(-1)
        if len(scores) and image_id not in image_set:
            raise ValueError(f"detections on image id {image_id}, which the annotation file does not have")
        for p in range(len(scores)):
            cid = to_cat(int(labels[p]))
            x1, y1, x2, y2 = boxes[p]
            w, h = float(np.float32(x2 - x1)), float(np.float32(y2 - y1))     # rule 3: fp32 subtraction
            dts[(image_id, cid)].append({"bbox": (float(x1), float(y1), w, h), "area": w * h,
                                         "score": float(scores[p])})
    gts = defaultdict(list)
    evaluated = set(img_ids)
    for ann in gt["annotations"]:
        if int(ann["image_id"]) in evaluated:
            gts[(int(ann["image_id"]), int(ann["category_id"]))].append(
                {"bbox": tuple(float(v) for v in ann["bbox"]), "area": float(ann["area"]),
                 "crowd": bool(ann.get("iscrowd", 0)), "id": ann["id"]})
    T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(cat_ids), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    scores_out = -np.ones((T, R, K, A, M))
    for k, cid in enumerate(cat_ids):
        pairs = [evaluate_pair(dts.get((i, cid), []), gts.get((i, cid), []))
                 for i in img_ids if (i, cid) in dts or (i, cid) in gts]
        if not pairs:
            continue
        for a in range(A):
            npig = int(sum(np.count_nonzero(~p[a][3]) for p in pairs))
            if npig == 0:
                continue
            for mi, m in enumerate(MAX_DETS):
                sc = np.concatenate([p[a][0][:m] for p in pairs])
                order = np.argsort(-sc, kind="stable")
                sc = sc[order]
                matched = np.concatenate([p[a][1][:, :m] for p in pairs], axis=1)[:, order]
                dt_ig = np.concatenate([p[a][2][:, :m] for p in pairs], axis=1)[:, order]
                tp_sum = np.cumsum(matched & ~dt_ig, axis=1).astype(np.float64)
                fp_sum = np.cumsum(~matched & ~dt_ig, axis=1).astype(np.float64)
                nd = len(sc)
                for t in range(T):
                    tp, fp = tp_sum[t], fp_sum[t]
                    rc = tp / npig
                    pr = tp / ((fp + tp) + EPS)
                    recall[t, k, a, mi] = rc[-1] if nd else 0.0
                    pr = np.maximum.accumulate(pr[::-1])[::-1]          # suffix maximum
                    q = np.zeros(R)
                    s = np.zeros(R)
                    for r, i in enumerate(np.searchsorted(rc, REC_THRS, side="left")):
                        if i < nd:
                            q[r], s[r] = pr[i], sc[i]
                    precision[t, :, k, a, mi] = q
                    scores_out[t, :, k, a, mi] = s
    ev = {"precision": precision, "recall": recall, "scores": scores_out}
    return ev, summarize(precision, recall)


def summarize(precision, recall):
    """rule 8: COCOeval.summarize's twelve numbers for bbox."""
    def mean(s):
        s = s[s > -1]
        return float(np.mean(s)) if s.size else -1.0

    t50, t75 = np.where(IOU_THRS == .5)[0], np.where(IOU_THRS == .75)[0]
    return np.array([
        mean(precision[:, :, :, 0, 2]), mean(precision[t50][:, :, :, 0, 2]), mean(precision[t75][:, :, :, 0, 2]),
        mean(precision[:, :, :, 1, 2]), mean(precision[:, :, :, 2, 2]), mean(precision[:, :, :, 3, 2]),
        mean(recall[:, :, 0, 0]), mean(recall[:, :, 0, 1]), mean(recall[:, :, 0, 2]),
        mean(recall[:, :, 1, 2]), mean(recall[:, :, 2, 2]), mean(recall[:, :, 3, 2]),
    ])
