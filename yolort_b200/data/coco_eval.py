"""COCO box evaluation on the GPU: the reference's `yolort.data.coco_eval.COCOEvaluator` without pycocotools.

Detections are stored on the device as they arrive (`update` / `update_padded` never wait for the GPU), and
`compute()` runs pycocotools' per-image matching and accumulation as CUDA kernels (csrc/coco_eval.cu), reproducing
its `COCOeval.eval` arrays and `stats` bit for bit.  The protocol is restated rule by rule in
oracle/restate_cocoeval.py.
"""
import itertools
import json
import math
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from .. import _C

__all__ = ["COCOEvaluator"]

# COCOeval.Params for bbox (rule 1): computed by numpy and handed to the kernels as they are
IOU_THRS = np.linspace(.5, .95, 10)
REC_THRS = np.linspace(0, 1, 101)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0.0, 1e10], [0.0, 32.0 ** 2], [32.0 ** 2, 96.0 ** 2], [96.0 ** 2, 1e10]]
METRICS = ["AP", "AP50", "AP75", "APs", "APm", "APl"]


def _is_number(v) -> bool:
    return isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v)


def _validate(data) -> None:
    """Raises ValueError naming the first entry of a COCO annotation dict the evaluator cannot use."""
    if not isinstance(data, dict):
        raise ValueError("annotation file: expected a JSON object")
    for key in ("images", "annotations", "categories"):
        if not isinstance(data.get(key), list):
            raise ValueError(f"annotation file: '{key}' is missing or not a list")
    image_ids, cat_ids = set(), set()
    for key, ids in (("images", image_ids), ("categories", cat_ids)):
        for i, entry in enumerate(data[key]):
            if not isinstance(entry, dict) or not isinstance(entry.get("id"), int) or isinstance(entry["id"], bool):
                raise ValueError(f"annotation file: {key}[{i}] has no integer 'id'")
            if entry["id"] in ids:
                raise ValueError(f"annotation file: {key}[{i}] repeats id {entry['id']}")
            ids.add(entry["id"])
    if not cat_ids:
        raise ValueError("annotation file: 'categories' is empty")
    for i, ann in enumerate(data["annotations"]):
        where = f"annotation file: annotations[{i}]"
        if not isinstance(ann, dict):
            raise ValueError(f"{where} is not an object")
        if not isinstance(ann.get("id"), int) or isinstance(ann["id"], bool):
            raise ValueError(f"{where} has no integer 'id'")
        bbox = ann.get("bbox")
        if not isinstance(bbox, list) or len(bbox) != 4 or not all(_is_number(v) for v in bbox):
            raise ValueError(f"{where} (id {ann['id']}): 'bbox' must be 4 finite numbers, got {bbox!r}")
        if not _is_number(ann.get("area")):
            raise ValueError(f"{where} (id {ann['id']}): 'area' must be a finite number, got {ann.get('area')!r}")
        if ann.get("image_id") not in image_ids:
            raise ValueError(f"{where} (id {ann['id']}): image_id {ann.get('image_id')!r} is not in 'images'")
        if ann.get("category_id") not in cat_ids:
            raise ValueError(f"{where} (id {ann['id']}): category_id {ann.get('category_id')!r} is not in 'categories'")
        if not _is_number(ann.get("iscrowd", 0)):
            raise ValueError(f"{where} (id {ann['id']}): 'iscrowd' must be a number")


def summarize(precision: np.ndarray, recall: np.ndarray) -> np.ndarray:
    """COCOeval.summarize's twelve bbox numbers (rule 8): np.mean(s[s > -1]), or -1, over its slices."""
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


def merge_ranks(parts: Sequence[dict], img_index: Dict[int, int]):
    """The reference's `merge`: ranks in order, an image id keeps the first rank that evaluated it.  Each part is
    {"ids": image ids in first-evaluation order, "records": int32 [n, 8] stored detections, "status": int}.
    Returns (ids, records, status) of the union."""
    seen, ids, recs, status = set(), [], [], 0
    for part in parts:
        claimed = np.array(sorted(img_index[i] for i in seen if i in img_index), dtype=np.int32)
        rec = np.asarray(part["records"], dtype=np.int32).reshape(-1, _C.YB_COCO_RECORD_INT32)
        recs.append(rec[~np.isin(rec[:, 0], claimed)])
        new = [i for i in part["ids"] if i not in seen]
        ids.extend(new)
        seen.update(new)
        status |= int(part["status"])
    return ids, np.concatenate(recs) if recs else np.zeros((0, _C.YB_COCO_RECORD_INT32), np.int32), status


def all_gather_records(ids: List[int], records: np.ndarray, status: int, img_index: Dict[int, int], group=None):
    """Every rank's (ids, records, status) gathered over `group` and merged by `merge_ranks`."""
    import torch.distributed as dist

    parts = [None] * dist.get_world_size(group)
    dist.all_gather_object(parts, {"ids": list(ids), "records": records, "status": int(status)}, group=group)
    return merge_ranks(parts, img_index)


def label_to_category(cat_ids: List[int], eval_type: str) -> np.ndarray:
    """int32 [L]: label -> category index (-1: a category the file does not have); a label outside [0, L) is an
    error.  "yolov5": label l is the l-th smallest category id; "torchvision": label l is category id l."""
    if eval_type == "yolov5":
        return np.arange(len(cat_ids), dtype=np.int32)
    if eval_type != "torchvision":
        raise NotImplementedError(f"Currently not supports eval type {eval_type}")
    lut = np.full(max(cat_ids[-1] + 1, 0), -1, dtype=np.int32)
    for k, c in enumerate(cat_ids):
        if c >= 0:
            lut[c] = k
    return lut


def _image_id(target) -> int:
    if isinstance(target, dict):
        target = target["image_id"]
    if isinstance(target, torch.Tensor):
        if target.numel() != 1:
            raise ValueError(f"image_id must hold one value, got shape {tuple(target.shape)}")
        return int(target.item())   # a CUDA tensor costs one synchronisation here, as in the reference
    return int(target)


class COCOEvaluator:
    """Evaluate AP for box detection with COCO's metrics, on a CUDA device, in single or distributed mode.
    See http://cocodataset.org/#detection-eval.  The metrics range from 0 to 100; NaN means the metric cannot be
    computed (pycocotools' -1).

    Args:
        coco_gt: a COCO annotation JSON (path as str / Path) or the parsed dict.
        iou_type: "bbox" (the only type supported).
        eval_type: "yolov5" maps label l to the l-th smallest category id; "torchvision" maps label l to id l.
        device: the CUDA device the detections are stored and evaluated on.
    """

    def __init__(self, coco_gt: Union[str, Path, dict], iou_type: str = "bbox", eval_type: str = "yolov5",
                 device: Union[str, torch.device] = "cuda"):
        if iou_type != "bbox":
            raise ValueError(f"Unknown iou type {iou_type}: only 'bbox' is supported")
        if eval_type not in ("yolov5", "torchvision"):
            raise NotImplementedError(f"Currently not supports eval type {eval_type}")
        if isinstance(coco_gt, (str, Path)):
            with open(coco_gt) as f:
                coco_gt = json.load(f)
        elif not isinstance(coco_gt, dict):
            raise NotImplementedError(f"Currently not supports type {type(coco_gt)}")
        _validate(coco_gt)
        device = torch.device(device)
        if device.type != "cuda":
            raise _C.NativeLibraryError("COCOEvaluator runs on a CUDA device only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        self.iou_type = iou_type
        self.eval_type = eval_type

        img_ids = sorted(im["id"] for im in coco_gt["images"])
        self.cat_ids = sorted(c["id"] for c in coco_gt["categories"])
        self._img_index = {i: n for n, i in enumerate(img_ids)}
        cat_index = {c: k for k, c in enumerate(self.cat_ids)}
        anns = coco_gt["annotations"]
        n_img, K = len(img_ids), len(self.cat_ids)
        gi = np.array([self._img_index[a["image_id"]] for a in anns], dtype=np.int64)
        ci = np.array([cat_index[a["category_id"]] for a in anns], dtype=np.int64)
        order = np.lexsort((np.arange(len(anns)), ci, gi))   # by image, then category, then file order
        box = np.array([a["bbox"] for a in anns], dtype=np.float64).reshape(-1, 4)[order]
        area = np.array([a["area"] for a in anns], dtype=np.float64)[order]
        flags = np.array([(_C.YB_COCO_GT_CROWD if a.get("iscrowd", 0) else 0)
                          | (_C.YB_COCO_GT_ID_NONZERO if a["id"] != 0 else 0) for a in anns], dtype=np.uint8)[order]
        gi, ci = gi[order], ci[order]
        img_start = np.searchsorted(gi, np.arange(n_img + 1)).astype(np.int32)
        pair_counts = np.unique(gi * K + ci, return_counts=True)[1]

        def up(a):   # at least one element, so every pointer is valid
            a = np.ascontiguousarray(a)
            if a.size == 0:
                a = np.zeros((1,) + a.shape[1:], a.dtype)
            return torch.from_numpy(a).to(device)

        self._gt_tensors = [up(img_start), up(gi.astype(np.int32)), up(ci.astype(np.int32)), up(box), up(area),
                            up(flags)]
        t = self._gt_tensors
        self._gt = _C.CocoGt(n_img, K, len(anns), int(pair_counts.max()) if pair_counts.size else 0,
                             t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(),
                             t[5].data_ptr())
        label_map = label_to_category(self.cat_ids, eval_type)
        self._label_map = up(label_map)
        self._n_labels = len(label_map)
        self._params = torch.from_numpy(np.concatenate(
            [IOU_THRS, REC_THRS, np.array(AREA_RNG, np.float64).ravel()])).to(device)
        self.stats = None
        self.eval = None
        self.reset()

    # -- storage ------------------------------------------------------------------------------------------------
    def reset(self) -> None:
        """Forget every stored detection and evaluated image."""
        self._records = torch.empty((0, _C.YB_COCO_RECORD_INT32), dtype=torch.int32, device=self.device)
        self._n = 0
        self._ids: List[int] = []       # evaluated image ids, in first-evaluation order
        self._seen = set()
        self._status = torch.zeros((1,), dtype=torch.int32, device=self.device)

    def _to_device(self, t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
        t = t.to(dtype)
        if t.device == self.device:
            return t.contiguous()
        if t.device.type == "cpu":
            return t.contiguous().pin_memory().to(self.device, non_blocking=True)
        return t.to(self.device)

    def _reserve(self, extra: int) -> torch.Tensor:
        need = self._n + extra
        if need > self._records.shape[0]:
            grown = torch.empty((max(need, 2 * self._records.shape[0], 1 << 16), _C.YB_COCO_RECORD_INT32),
                                dtype=torch.int32, device=self.device)
            grown[: self._n].copy_(self._records[: self._n])
            self._records = grown
        return self._records[self._n: need]

    def update_padded(self, boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, counts: torch.Tensor,
                      image_ids) -> None:
        """Store `forward_padded`'s outputs as they are: boxes xyxy [n,D,4], scores [n,D], labels [n,D], counts [n],
        with the image ids of the n rows (host ints, or a tensor: a CUDA one costs one synchronisation).  Nothing
        waits for the device.  A repeated image id keeps its first update call, and the last row within a call."""
        if isinstance(image_ids, torch.Tensor):
            image_ids = image_ids.reshape(-1).tolist()
        ids = [_image_id(i) for i in image_ids]
        n = len(ids)
        if scores.dim() != 2 or scores.shape[0] != n or tuple(boxes.shape) != (n, scores.shape[1], 4) \
                or tuple(labels.shape) != tuple(scores.shape) or counts.numel() != n:
            raise ValueError("update_padded: expected boxes [n,D,4], scores [n,D], labels [n,D], counts [n] and n "
                             "image ids")
        last = {i: r for r, i in enumerate(ids)}
        rows = []
        for r, i in enumerate(ids):
            if last[i] != r or i in self._seen:
                rows.append(_C.YB_COCO_ROW_DROPPED)
            else:
                rows.append(self._img_index.get(i, -1))
        for i in last:
            if i not in self._seen:
                self._seen.add(i)
                self._ids.append(i)
        d = int(scores.shape[1])
        if n * d == 0:
            return
        records = self._reserve(n * d)
        row_image = torch.tensor(rows, dtype=torch.int32).pin_memory().to(self.device, non_blocking=True)
        _C.coco_append(self._to_device(boxes, torch.float32), self._to_device(scores, torch.float32),
                       self._to_device(labels, torch.int64), self._to_device(counts.reshape(-1), torch.int32),
                       row_image, self._label_map, records, self._status)
        self._n += n * d

    def update(self, preds: List[Dict[str, torch.Tensor]], targets) -> None:
        """Store the detections of `predict` / `forward` (device or host tensors) for the images of `targets`: dicts
        with "image_id" (an int or a one-element tensor) or plain ints.  Packs the lists and calls `update_padded`;
        only tensor shapes are read on the host."""
        preds, targets = list(preds), list(targets)
        if len(preds) != len(targets):
            raise ValueError(f"update: {len(preds)} predictions for {len(targets)} targets")
        ids = [_image_id(t) for t in targets]
        counts = [int(p["scores"].shape[0]) for p in preds]
        n, d = len(preds), max(counts, default=0)
        if n == 0:
            return
        if d == 0:
            self.update_padded(torch.empty((n, 0, 4)), torch.empty((n, 0)), torch.empty((n, 0), dtype=torch.int64),
                               torch.zeros(n, dtype=torch.int32), ids)
            return
        # one concatenation per field, then one scatter into the padded slots
        flat_b = torch.cat([p["boxes"].reshape(-1, 4) for p in preds])
        flat_s = torch.cat([p["scores"].reshape(-1) for p in preds])
        flat_l = torch.cat([p["labels"].reshape(-1) for p in preds])
        slot = torch.tensor(list(itertools.chain.from_iterable(range(r * d, r * d + c) for r, c in enumerate(counts))),
                            dtype=torch.int64)
        slot = self._to_device(slot, torch.int64)
        boxes = torch.empty((n * d, 4), dtype=torch.float32, device=self.device)
        scores = torch.empty((n * d,), dtype=torch.float32, device=self.device)
        labels = torch.empty((n * d,), dtype=torch.int64, device=self.device)
        boxes.index_copy_(0, slot, self._to_device(flat_b, torch.float32))
        scores.index_copy_(0, slot, self._to_device(flat_s, torch.float32))
        labels.index_copy_(0, slot, self._to_device(flat_l, torch.int64))
        self.update_padded(boxes.view(n, d, 4), scores.view(n, d), labels.view(n, d),
                           torch.tensor(counts, dtype=torch.int32), ids)

    # -- evaluation ---------------------------------------------------------------------------------------------
    def compute(self, group=None) -> dict:
        """Evaluate everything stored (under torch.distributed with more than one rank: every rank's detections, an
        image keeping the first rank that evaluated it) and return `derive_coco_results()`.  Sets `self.stats` and
        `self.eval` ({"precision", "recall", "scores"} float64 arrays in COCOeval's layout)."""
        import torch.distributed as dist

        records, ids, status = self._records[: self._n], self._ids, None
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            local = records.cpu().numpy()
            local = local[local[:, 2] >= 0]
            ids, merged, status = all_gather_records(ids, local, int(self._status.item()), self._img_index, group)
            records = self._to_device(torch.from_numpy(merged), torch.int32)
        if status is None:
            status = int(self._status.item())
        if status & _C.YB_COCO_ST_UNKNOWN_IMAGE:
            raise ValueError("detections on an image id that the annotation file does not have")
        if status & _C.YB_COCO_ST_BAD_LABEL:
            raise ValueError(f"a detection label is outside the {self.eval_type} label map of {self._n_labels} labels")
        evaluated = np.zeros(self._gt.n_images, dtype=np.uint8)
        for i in ids:
            if i in self._img_index:
                evaluated[self._img_index[i]] = 1
        evaluated = torch.from_numpy(evaluated if evaluated.size else np.zeros(1, np.uint8)).to(self.device)
        if self._gt.n_images == 0:
            evaluated = evaluated[:0]
        precision, recall, scores = _C.coco_evaluate(self._gt, records.contiguous(), evaluated, self._params)
        # pinned buffers: the arrays are about 16 MB at K = 80, and a pageable copy of them costs more than the kernels
        host = {k: torch.empty(t.shape, dtype=t.dtype, pin_memory=True).copy_(t, non_blocking=True)
                for k, t in (("precision", precision), ("recall", recall), ("scores", scores))}
        torch.cuda.current_stream(self.device).synchronize()
        self.eval = {k: t.numpy() for k, t in host.items()}
        self.stats = summarize(self.eval["precision"], self.eval["recall"])
        return self.derive_coco_results()

    def derive_coco_results(self, class_names: Optional[List[str]] = None) -> dict:
        """{"AP", "AP50", "AP75", "APs", "APm", "APl"} x 100 (NaN where pycocotools gives -1), plus "AP-<name>" per
        category when `class_names` (one per category, ascending id) is given."""
        if self.stats is None:
            return {m: float("nan") for m in METRICS}
        results = {m: float(self.stats[i] * 100) if self.stats[i] >= 0 else float("nan") for i, m in enumerate(METRICS)}
        if class_names is None or len(class_names) <= 1:
            return results
        precisions = self.eval["precision"]
        if len(class_names) != precisions.shape[2]:
            raise ValueError(f"{len(class_names)} class names for {precisions.shape[2]} categories")
        for k, name in enumerate(class_names):
            p = precisions[:, :, k, 0, -1]
            p = p[p > -1]
            results["AP-" + name] = float(np.mean(p) * 100) if p.size else float("nan")
        return results
