"""COCO box evaluation on the host: the numpy restatement's known answers (each derived from the protocol's rules in
oracle/restate_cocoeval.py), annotation-file validation, the label maps, and the multi-rank merge over gloo."""
import json
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from coco_corpus import EPS, ONE, cases, corpus, det, gt_file
from oracle import restate_cocoeval as O
from yolort_b200.data import coco_eval as E

C = cases()


def run(name):
    gt, calls, eval_type = C[name]
    return O.evaluate(gt, calls, eval_type)


def mean_of(*parts):
    return np.mean(np.concatenate([np.full(n, v) for n, v in parts]))


def test_parameters_are_numpys():
    assert O.IOU_THRS[8] == 0.8999999999999999
    assert O.REC_THRS[35] == 0.35000000000000003
    assert np.array_equal(O.IOU_THRS, E.IOU_THRS) and np.array_equal(O.REC_THRS, E.REC_THRS)
    assert O.AREA_RNG == E.AREA_RNG


def test_identical_detection():
    ev, stats = run("identical")
    # 10 thresholds x 101 recall thresholds x 1 category, each 1 / (1 + 2^-52)
    assert stats[0] == np.mean(np.full(1010, ONE)) == 0.9999999999999998
    assert stats[4] == stats[0] and stats[3] == -1 and stats[5] == -1        # area 2000: medium only
    assert np.all(ev["recall"][:, 0, 0, :] == 1.0)


def test_iou_064():
    ev, stats = run("iou_064")
    # IoU 64/100 = 0.64 clears 0.5, 0.55, 0.6: 3 of 10 rows of 101 ones
    assert stats[0] == mean_of((303, ONE), (707, 0.0)) == 0.29999999999999993
    assert stats[1] == np.mean(np.full(101, ONE)) == 0.9999999999999999
    assert stats[2] == 0.0


def test_crowd_absorbs_detections():
    ev, stats = run("crowd")
    # the two detections inside the crowd box match it (IoU = 400 / 400) and are ignored: only the real TP counts
    assert stats[0] == np.mean(np.full(1010, ONE))
    assert np.all(ev["recall"][:, 0, 0, 2] == 1.0)


def test_ignored_gt_only_without_a_normal_match():
    ev, stats = run("ignored_last")
    p = ev["precision"][:, :, 0, 0, 2]
    assert np.all(p[:3] == ONE)        # IoU 0.6 with the normal GT: a TP at 0.5, 0.55, 0.6
    assert np.all(p[3:] == 0.0)        # above: the crowd GT takes it, so it is ignored, and nothing is found
    assert stats[0] == 0.29999999999999993


def test_equal_iou_later_gt_wins():
    ev, _ = run("tie_later_real")
    # npig = 2, one TP: rc = 0.5, precision 1 / (1 + 2^-52) up to recall 0.5
    assert np.array_equal(ev["precision"][:, :, 0, 0, 2], np.tile(np.where(O.REC_THRS <= 0.5, ONE, 0.0), (10, 1)))
    ev, _ = run("tie_later_id0")
    # the later GT has id 0, so the detection counts as unmatched: an FP
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 0.0) and np.all(ev["recall"][:, 0, 0, 2] == 0.0)


def test_gt_id_zero_counts_as_unmatched():
    ev, stats = run("id0")
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 0.0) and stats[0] == 0.0 and stats[8] == 0.0


def test_area_field_sets_the_range():
    _, stats = run("area_field")
    assert stats[3] == -1                          # small: the GT is ignored (area field 5000), npig = 0
    assert stats[4] == np.mean(np.full(1010, ONE))  # medium: the detection (area 100) matches a non-ignored GT


def test_area_1024_is_small_and_medium():
    _, stats = run("area_1024")
    assert stats[3] == stats[4] == np.mean(np.full(1010, ONE)) and stats[5] == -1


def test_iou_equal_to_threshold_matches():
    ev, stats = run("iou_equals_thr")
    assert np.all(ev["precision"][0, :, 0, 0, 2] == ONE) and np.all(ev["precision"][1:, :, 0, 0, 2] == 0.0)
    assert stats[1] == np.mean(np.full(101, ONE))
    assert stats[0] == mean_of((101, ONE), (909, 0.0))


def test_only_100_detections_per_image_and_category():
    ev, _ = run("det101")
    assert np.all(ev["recall"][:, 0, 0, 2] == 0.0)        # the 101st (the TP) is dropped
    ev, _ = run("det100")
    assert np.all(ev["recall"][:, 0, 0, 2] == 1.0)
    # 99 FPs then the TP: pr = 1 / ((99 + 1) + 2^-52) at recall 1
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 1.0 / ((99.0 + 1.0) + EPS))


def test_maxdets_1_and_10():
    ev, _ = run("maxdets")
    r = ev["recall"][0, 0, 0]
    assert r[0] == 0.0                       # maxDets 1: only the top-scoring FP
    assert r[1] == 9 / 10 and r[2] == 1.0    # maxDets 10: the FP and 9 of the 10 TPs; 100: all 10


def test_score_ties_across_images_lower_id_first():
    ev, _ = run("tie_images")
    # image 1's FP goes before image 2's TP: pr = [0, 1 / (2 + 2^-52)], rc = [0, 0.5]
    want = np.where(O.REC_THRS <= 0.5, 1.0 / ((1.0 + 1.0) + EPS), 0.0)
    assert np.array_equal(ev["precision"][0, :, 0, 0, 2], want)


def test_categories_without_detections_or_gt():
    ev, stats = run("empty_cats")
    assert np.all(ev["precision"][:, :, 1, 0, 2] == 0.0) and np.all(ev["recall"][:, 1, 0, 2] == 0.0)
    assert np.all(ev["precision"][:, :, 2] == -1) and np.all(ev["recall"][:, 2] == -1)
    assert np.all(ev["precision"][:, :, 0, 0, 2] == ONE)


def test_image_repeats():
    assert run("first_call_wins")[1][0] == np.mean(np.full(1010, ONE))
    assert run("last_in_call_wins")[1][0] == np.mean(np.full(1010, ONE))


def test_torchvision_map_drops_unknown_categories():
    ev, stats = run("torchvision")
    assert stats[0] == np.mean(np.full(1010, ONE))   # label 2 is no category: its higher score is ignored
    assert np.all(ev["precision"][:, :, 0] == -1)             # category 1 has neither GT nor detections


def test_oracle_errors():
    gt = gt_file([1], [(1, 1, [0, 0, 10, 10], None, 0, 1)])
    with pytest.raises(ValueError, match="image id 9"):
        O.evaluate(gt, [[(9, det([[0, 0, 1, 1]], [0.5], [0]))]])
    with pytest.raises(ValueError, match="label 1"):
        O.evaluate(gt, [[(1, det([[0, 0, 1, 1]], [0.5], [1]))]])
    O.evaluate(gt, [[(9, det(np.zeros((0, 4)), [], []))]])      # an unknown image without detections is fine


def test_corpus_oracle_is_consistent():
    gt, calls = corpus(3, 40, n_cats=6)
    ev, stats = O.evaluate(gt, calls)
    assert ev["precision"].shape == (10, 101, 6, 4, 3) and ev["recall"].shape == (10, 6, 4, 3)
    assert 0.0 < stats[0] < 1.0
    assert np.array_equal(stats, E.summarize(ev["precision"], ev["recall"]))


def test_pycocotools_agrees_when_available():
    pytest.importorskip("pycocotools")
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval

    for seed in (0, 1):
        gt, calls = corpus(seed, 30, n_cats=5)
        ev, stats = O.evaluate(gt, calls)
        coco = COCO()
        coco.dataset = gt
        coco.createIndex()
        kept = O.select_images(calls)
        cat_ids = sorted(c["id"] for c in gt["categories"])
        res = []
        for im, (b, s, l) in kept.items():
            for p in range(len(s)):
                x1, y1, x2, y2 = b[p]
                res.append({"image_id": im, "category_id": cat_ids[int(l[p])], "score": float(s[p]),
                            "bbox": [float(x1), float(y1), float(np.float32(x2 - x1)), float(np.float32(y2 - y1))]})
        e = COCOeval(coco, coco.loadRes(res), "bbox")
        e.params.imgIds = sorted(kept)
        e.evaluate()
        e.accumulate()
        e.summarize()
        for k in ("precision", "recall", "scores"):
            assert np.array_equal(e.eval[k], ev[k]), k
        assert np.array_equal(e.stats, stats)


# -- the annotation file and the label maps ------------------------------------------------------------------
GOOD = {"images": [{"id": 3}], "categories": [{"id": 7}, {"id": 2}],
        "annotations": [{"id": 1, "image_id": 3, "category_id": 7, "bbox": [0, 0, 4, 4], "area": 16}]}


@pytest.mark.parametrize("mutate,match", [
    (lambda d: d.pop("images"), "'images' is missing"),
    (lambda d: d.pop("categories"), "'categories' is missing"),
    (lambda d: d["annotations"][0].pop("bbox"), r"annotations\[0\].*'bbox'"),
    (lambda d: d["annotations"][0].update(bbox=[0, 0, 4]), "'bbox' must be 4"),
    (lambda d: d["annotations"][0].update(bbox=[0, 0, float("nan"), 4]), "'bbox' must be 4 finite"),
    (lambda d: d["annotations"][0].update(area=float("inf")), "'area' must be a finite"),
    (lambda d: d["annotations"][0].pop("area"), "'area'"),
    (lambda d: d["annotations"][0].update(image_id=4), "image_id 4 is not in 'images'"),
    (lambda d: d["annotations"][0].update(category_id=1), "category_id 1 is not in 'categories'"),
    (lambda d: d["images"].append({"id": 3}), r"images\[1\] repeats id 3"),
])
def test_validation_names_the_bad_entry(mutate, match):
    d = json.loads(json.dumps(GOOD))
    mutate(d)
    with pytest.raises(ValueError, match=match):
        E._validate(d)


def test_iscrowd_is_optional_and_type_checks():
    E._validate(GOOD)
    with pytest.raises(ValueError, match="iou type"):
        E.COCOEvaluator(GOOD, iou_type="segm")
    with pytest.raises(NotImplementedError):
        E.COCOEvaluator(GOOD, eval_type="detectron")
    with pytest.raises(NotImplementedError):
        E.COCOEvaluator(42)


def test_label_maps():
    assert E.label_to_category([2, 7], "yolov5").tolist() == [0, 1]          # label l -> sorted ids[l]
    assert E.label_to_category([2, 7], "torchvision").tolist() == [-1, -1, 0, -1, -1, -1, -1, 1]   # label = id


def test_merge_ranks_first_rank_wins():
    idx = {10: 0, 20: 1, 30: 2}
    r0 = np.array([[0, 0, 0, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0]], np.int32)
    r1 = np.array([[1, 0, 5, 0, 0, 0, 0, 0], [2, 0, 0, 0, 0, 0, 0, 0]], np.int32)
    ids, rec, st = E.merge_ranks([{"ids": [10, 20], "records": r0, "status": 0},
                                  {"ids": [30, 20, 99], "records": r1, "status": 2}], idx)
    assert ids == [10, 20, 30, 99] and st == 2
    assert rec[:, 0].tolist() == [0, 1, 2] and rec[1, 2] == 0      # image 20 keeps rank 0's record


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        idx = {10: 0, 20: 1, 30: 2}
        ids = [[10, 20], [20, 30]][rank]
        rec = np.array([[idx[i], rank, 0, 0, 0, 0, 0, 0] for i in ids], np.int32)
        q.put((rank, E.all_gather_records(ids, rec, rank, idx)))
    finally:
        dist.destroy_process_group()


def test_gather_and_dedupe_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=120) for _ in procs), key=lambda x: x[0])
    for p in procs:
        p.join(timeout=60)
    for _, (ids, rec, st) in res:
        assert ids == [10, 20, 30] and st == 1
        assert rec[:, :2].tolist() == [[0, 0], [1, 0], [2, 1]]    # image 20 from rank 0, image 30 from rank 1
