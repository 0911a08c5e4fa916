"""COCO evaluation inputs shared by tests/test_cocoeval.py (oracle, CPU) and tests/test_gpu_cocoeval.py (device):
hand-built known-answer cases and seeded COCO-shaped corpora.  A case is (gt dict, calls, eval_type), with calls =
one list per update call of (image_id, (boxes xyxy float32 [n,4], scores float32 [n], labels int64 [n]))."""
import numpy as np

EPS = 2.0 ** -52
ONE = 1.0 - EPS        # pycocotools' precision of a perfect detection: 1 / (1 + 2^-52)


def det(boxes, scores, labels):
    return (np.asarray(boxes, np.float32).reshape(-1, 4), np.asarray(scores, np.float32).reshape(-1),
            np.asarray(labels, np.int64).reshape(-1))


def gt_file(images, anns, cats=(1,)):
    """anns: (image_id, category_id, [x, y, w, h], area or None for w*h, iscrowd, id)."""
    out = []
    for n, (img, cat, bbox, area, crowd, aid) in enumerate(anns):
        out.append({"id": aid, "image_id": img, "category_id": cat, "bbox": [float(v) for v in bbox],
                    "area": float(bbox[2] * bbox[3] if area is None else area), "iscrowd": crowd})
    return {"images": [{"id": i} for i in images], "annotations": out, "categories": [{"id": c} for c in cats]}


def cases():
    """name -> (gt, calls, eval_type).  The expected values are in test_cocoeval.py."""
    c = {}
    c["identical"] = (gt_file([1], [(1, 1, [10, 10, 50, 40], None, 0, 1)]),
                      [[(1, det([[10, 10, 60, 50]], [0.9], [0]))]], "yolov5")
    c["iou_064"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]),
                    [[(1, det([[0, 0, 8, 8]], [0.9], [0]))]], "yolov5")
    # two detections inside a crowd region (IoU with a crowd GT = i / detection area = 1) score above the real TP
    c["crowd"] = (gt_file([1], [(1, 1, [0, 0, 100, 100], None, 1, 1), (1, 1, [200, 200, 20, 20], None, 0, 2)]),
                  [[(1, det([[10, 10, 30, 30], [50, 50, 70, 70], [200, 200, 220, 220]], [0.9, 0.8, 0.7], [0, 0, 0]))]],
                  "yolov5")
    # the normal GT (IoU 0.6) wins over the crowd GT (IoU 1) while it qualifies
    c["ignored_last"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], 100, 1, 1), (1, 1, [0, 0, 10, 6], None, 0, 2)]),
                         [[(1, det([[0, 0, 10, 10]], [0.9], [0]))]], "yolov5")
    # equal IoU: the later GT wins; with ids (0, 7) that is a real match, with (7, 0) a match to id 0 (no match)
    c["tie_later_real"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 0), (1, 1, [0, 0, 10, 10], None, 0, 7)]),
                           [[(1, det([[0, 0, 10, 10]], [0.9], [0]))]], "yolov5")
    c["tie_later_id0"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 7), (1, 1, [0, 0, 10, 10], None, 0, 0)]),
                          [[(1, det([[0, 0, 10, 10]], [0.9], [0]))]], "yolov5")
    c["id0"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 0)]), [[(1, det([[0, 0, 10, 10]], [0.9], [0]))]],
                "yolov5")
    # a 10x10 box whose area field (a segment area) is 5000: medium, not small
    c["area_field"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], 5000, 0, 1)]),
                       [[(1, det([[0, 0, 10, 10]], [0.9], [0]))]], "yolov5")
    c["area_1024"] = (gt_file([1], [(1, 1, [0, 0, 32, 32], None, 0, 1)]),
                      [[(1, det([[0, 0, 32, 32]], [0.9], [0]))]], "yolov5")
    # i = 50, u = (50 + 100) - 50 = 100: IoU exactly 0.5
    c["iou_equals_thr"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]),
                           [[(1, det([[0, 0, 10, 5]], [0.9], [0]))]], "yolov5")
    fps = [[300 + 20 * i, 300, 310 + 20 * i, 310] for i in range(100)]
    c["det101"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]),
                   [[(1, det(fps + [[0, 0, 10, 10]], [0.9] * 100 + [0.5], [0] * 101))]], "yolov5")
    c["det100"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]),
                   [[(1, det(fps[:99] + [[0, 0, 10, 10]], [0.9] * 99 + [0.5], [0] * 100))]], "yolov5")
    c["maxdets"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)] +
                            [(1, 1, [100 + 20 * i, 0, 10, 10], None, 0, 2 + i) for i in range(9)]),
                    [[(1, det([[500, 500, 510, 510]] + [[0, 0, 10, 10]] + [[100 + 20 * i, 0, 110 + 20 * i, 10]
                                                                           for i in range(9)],
                              [0.9] + [0.8] * 10, [0] * 11))]], "yolov5")
    # equal scores on images 2 (a TP) and 1 (an FP), given in that order: image 1 goes first
    c["tie_images"] = (gt_file([1, 2], [(1, 1, [0, 0, 10, 10], None, 0, 1), (2, 1, [0, 0, 10, 10], None, 0, 2)]),
                       [[(2, det([[0, 0, 10, 10]], [0.5], [0])), (1, det([[50, 50, 60, 60]], [0.5], [0]))]], "yolov5")
    # category 3 has GT and no detection, category 5 detections and no GT
    c["empty_cats"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1), (1, 3, [20, 20, 10, 10], None, 0, 2)],
                               cats=(1, 3, 5)),
                       [[(1, det([[0, 0, 10, 10], [20, 20, 30, 30]], [0.9, 0.8], [0, 2]))]], "yolov5")
    tp, fp = det([[0, 0, 10, 10]], [0.9], [0]), det([[50, 50, 60, 60]], [0.9], [0])
    c["first_call_wins"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]), [[(1, tp)], [(1, fp)]], "yolov5")
    c["last_in_call_wins"] = (gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)]), [[(1, fp), (1, tp)]], "yolov5")
    # torchvision labels are category ids: label 3 is category 3, label 2 is no category (not evaluated)
    c["torchvision"] = (gt_file([1], [(1, 3, [0, 0, 10, 10], None, 0, 1)], cats=(1, 3)),
                        [[(1, det([[0, 0, 10, 10], [0, 0, 10, 10]], [0.9, 0.95], [3, 2]))]], "torchvision")
    return c


def corpus(seed, n_images, n_cats=80, gt_per_image=7, fp_per_image=4, batch=32, crowd=0.02, max_gt=None,
           big_pair=0):
    """A seeded COCO-val-shaped workload: GT boxes over three size scales (area field = w*h, or a smaller segment
    area), crowd GT, detections jittered from GT with some label noise, random false positives, scores on a 1/64
    grid (ties within and across images), image ids out of order with gaps, a repeated image and an image without
    detections.  big_pair > 0 puts that many GT (and 100+ detections) into one (image, category)."""
    rng = np.random.default_rng(seed)
    img_ids = sorted(rng.choice(np.arange(1, 20 * n_images + 10), n_images, replace=False).tolist())
    cat_ids = sorted(rng.choice(np.arange(1, 2 * n_cats + 10), n_cats, replace=False).tolist())
    anns, dets = [], {}
    aid = 1
    for im in img_ids:
        ng = int(rng.poisson(gt_per_image))
        boxes, scores, labels = [], [], []
        for _ in range(ng):
            s = float(np.exp(rng.uniform(np.log(6), np.log(300))))
            w, h = s * rng.uniform(0.5, 1.5), s * rng.uniform(0.5, 1.5)
            x, y = rng.uniform(0, 640 - w / 2), rng.uniform(0, 480 - h / 2)
            k = int(rng.integers(n_cats))
            area = w * h if rng.random() < 0.7 else w * h * rng.uniform(0.4, 1.0)
            anns.append({"id": aid, "image_id": im, "category_id": cat_ids[k], "bbox": [x, y, w, h], "area": area,
                         "iscrowd": int(rng.random() < crowd)})
            aid += 1
            for _ in range(int(rng.integers(0, 3))):
                j = rng.normal(0, 0.08, 4) * [w, h, w, h]
                boxes.append([x + j[0], y + j[1], x + w + j[2], y + h + j[3]])
                scores.append(rng.integers(1, 64) / 64)
                labels.append(k if rng.random() < 0.9 else int(rng.integers(n_cats)))
        for _ in range(int(rng.poisson(fp_per_image))):
            x, y = rng.uniform(0, 600), rng.uniform(0, 440)
            boxes.append([x, y, x + rng.uniform(4, 200), y + rng.uniform(4, 200)])
            scores.append(rng.integers(1, 64) / 64)
            labels.append(int(rng.integers(n_cats)))
        dets[im] = (boxes, scores, labels)
    if big_pair:
        im, k = img_ids[0], 0
        boxes, scores, labels = list(dets[im][0]), list(dets[im][1]), list(dets[im][2])
        for i in range(big_pair):
            x, y = (i % 40) * 16.0, (i // 40) * 16.0
            anns.append({"id": aid, "image_id": im, "category_id": cat_ids[k], "bbox": [x, y, 12.0, 12.0],
                         "area": 144.0, "iscrowd": int(i % 97 == 5)})
            aid += 1
            if i < 150:
                boxes.append([x + 0.5, y + 0.5, x + 12.5, y + 12.0 + (i % 5)])
                scores.append(rng.integers(1, 64) / 64)
                labels.append(k)
        dets[im] = (boxes, scores, labels)
    order = list(rng.permutation(img_ids))
    if len(order) > 2:
        order.append(order[1])                      # a repeat: the first occurrence counts
        dets[order[2]] = ([], [], [])               # an evaluated image without detections
    calls, cur = [], []
    for i, im in enumerate(order):
        b, s, l = dets[im]
        if i == len(order) - 1 and len(order) > 2:
            b, s, l = b[:1], s[:1], l[:1]
        cur.append((int(im), det(np.reshape(np.asarray(b, np.float64), (-1, 4)), s, l)))
        if len(cur) == batch:
            calls.append(cur)
            cur = []
    if cur:
        calls.append(cur)
    gt = {"images": [{"id": int(i)} for i in rng.permutation(img_ids)], "annotations": anns,
          "categories": [{"id": int(c)} for c in rng.permutation(cat_ids)]}
    return gt, calls
