"""COCO box evaluation on the device (yolort_b200.data.COCOEvaluator): COCOeval's precision / recall / scores arrays and
stats bit-identical to the numpy restatement (oracle/restate_cocoeval.py) on the known-answer cases and on seeded
corpora up to the COCO-val shape; the padded path, sync-free updates, deferred errors, and an end-to-end run."""
import collections
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from coco_corpus import ONE, cases, corpus
from oracle import restate_cocoeval as O
from yolort_b200.data import COCOEvaluator

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def feed(ev, calls, padded=False, device=DEV):
    for call in calls:
        ids = [i for i, _ in call]
        if padded:
            d = max(len(s) for _, (_, s, _) in call)
            n = len(call)
            boxes = torch.full((n, d, 4), 7.0)
            scores = torch.full((n, d), 0.5)
            labels = torch.full((n, d), 12345, dtype=torch.int64)     # padding is never read
            for r, (_, (b, s, l)) in enumerate(call):
                boxes[r, : len(s)] = torch.from_numpy(b)
                scores[r, : len(s)] = torch.from_numpy(s)
                labels[r, : len(s)] = torch.from_numpy(l)
            counts = torch.tensor([len(s) for _, (_, s, _) in call], dtype=torch.int32)
            ev.update_padded(boxes.to(device), scores.to(device), labels.to(device), counts.to(device), ids)
        else:
            preds = [{"boxes": torch.from_numpy(b).to(device), "scores": torch.from_numpy(s).to(device),
                      "labels": torch.from_numpy(l).to(device)} for _, (b, s, l) in call]
            ev.update(preds, [{"image_id": torch.tensor([i])} for i in ids])


def check(gt, calls, eval_type="yolov5", padded=False):
    want, want_stats = O.evaluate(gt, calls, eval_type)
    ev = COCOEvaluator(gt, eval_type=eval_type, device=DEV)
    feed(ev, calls, padded)
    res = ev.compute()
    for k in ("precision", "recall", "scores"):
        assert ev.eval[k].dtype == np.float64 and np.array_equal(ev.eval[k], want[k]), k
    assert np.array_equal(ev.stats, want_stats)
    return ev, res


@pytest.mark.parametrize("name", sorted(cases()))
def test_known_answers(name):
    gt, calls, eval_type = cases()[name]
    check(gt, calls, eval_type)
    check(gt, calls, eval_type, padded=True)


@pytest.mark.parametrize("seed,n_images,n_cats,batch", [(0, 3, 4, 2), (1, 60, 10, 7), (2, 500, 80, 32),
                                                        (7, 5000, 80, 32)])
def test_seeded_corpora(seed, n_images, n_cats, batch):
    gt, calls = corpus(seed, n_images, n_cats=n_cats, batch=batch)
    ev, res = check(gt, calls)
    assert res["AP"] == ev.stats[0] * 100 and 0 < res["AP"] < 100
    if n_images <= 500:
        check(gt, calls, padded=True)


def test_pair_with_600_gt():
    gt, calls = corpus(11, 20, n_cats=3, big_pair=600)
    check(gt, calls)


def test_category_list_larger_than_shared_memory():
    # 300 images x 100 detections of one category: 30 000 entries, streamed through the accumulation
    rng = np.random.default_rng(5)
    anns, calls, call = [], [], []
    for im in range(1, 301):
        xy = rng.uniform(0, 500, (100, 2))
        wh = rng.uniform(5, 120, (100, 2))
        for g in range(0, 100, 3):
            anns.append({"id": len(anns) + 1, "image_id": im, "category_id": 4, "bbox": [*xy[g], *wh[g]],
                         "area": float(wh[g, 0] * wh[g, 1]), "iscrowd": 0})
        jit = rng.normal(0, 3, (100, 4))
        boxes = np.concatenate([xy, xy + wh], 1) + jit
        call.append((im, (boxes.astype(np.float32), (rng.integers(1, 200, 100) / 200).astype(np.float32),
                          np.zeros(100, np.int64))))
        if len(call) == 64:
            calls.append(call)
            call = []
    calls.append(call)
    gt = {"images": [{"id": i} for i in range(1, 301)], "annotations": anns, "categories": [{"id": 4}]}
    check(gt, calls)


def test_torchvision_map_on_a_corpus():
    gt, calls = corpus(4, 40, n_cats=6)
    cat_ids = sorted(c["id"] for c in gt["categories"])
    # labels are category ids; label 0 is no category of the file, so those detections are not evaluated
    calls = [[(i, (b, s, np.array([cat_ids[x] if x % 3 else 0 for x in l], np.int64)))
              for i, (b, s, l) in call] for call in calls]
    check(gt, calls, "torchvision")


def test_updates_do_not_synchronise():
    gt, calls = corpus(3, 64, n_cats=8)
    ev = COCOEvaluator(gt, device=DEV)
    preds = [[{"boxes": torch.from_numpy(b).to(DEV), "scores": torch.from_numpy(s).to(DEV),
               "labels": torch.from_numpy(l).to(DEV)} for _, (b, s, l) in call] for call in calls]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for call, p in zip(calls, preds):
            ev.update(p, [i for i, _ in call])
        n, d = 4, 9
        ev.update_padded(torch.zeros((n, d, 4), device=DEV), torch.zeros((n, d), device=DEV),
                         torch.zeros((n, d), dtype=torch.int64, device=DEV),
                         torch.zeros((n,), dtype=torch.int32, device=DEV), [10 ** 6 + i for i in range(n)])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ev.compute()


def test_errors_surface_at_compute():
    gt, calls, _ = cases()["identical"]
    ev = COCOEvaluator(gt, device=DEV)
    b, s, l = calls[0][0][1]
    ev.update([{"boxes": torch.from_numpy(b).to(DEV), "scores": torch.from_numpy(s).to(DEV),
                "labels": torch.tensor([1], device=DEV)}], [1])
    with pytest.raises(ValueError, match="label"):
        ev.compute()
    ev.reset()
    ev.update([{"boxes": torch.from_numpy(b).to(DEV), "scores": torch.from_numpy(s).to(DEV),
                "labels": torch.from_numpy(l).to(DEV)}], [99])
    with pytest.raises(ValueError, match="image id"):
        ev.compute()
    ev.reset()
    ev.update([{"boxes": torch.zeros((0, 4), device=DEV), "scores": torch.zeros((0,), device=DEV),
                "labels": torch.zeros((0,), dtype=torch.int64, device=DEV)}], [99])
    ev.compute()     # an unknown image without detections is not an error


def test_cpu_device_is_refused():
    from yolort_b200._C import NativeLibraryError

    with pytest.raises(NativeLibraryError):
        COCOEvaluator(cases()["identical"][0], device="cpu")


def test_end_to_end_yolov5s_scores_its_own_detections():
    from bench import make_images, make_state_dict
    from yolort_b200.models import yolov5s

    model = yolov5s(score_thresh=0.25, size=(320, 320)).eval()
    model.load_state_dict(make_state_dict(model))
    model = model.to(DEV)
    ims = [im[:, :240 + 16 * i, :] for i, im in enumerate(make_images(6, 50, size=320))]
    out = model.predict([im.to(DEV) for im in ims])

    def usable(o):
        """The detections that can match themselves: a positive fp32 width and height, and among the first 100 of
        their (image, category) in the evaluator's stable score order (the NMS keeps up to 300 per image)."""
        o = {k: v.cpu() for k, v in o.items()}
        b = o["boxes"]
        keep = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
        rank = {}
        for p in np.argsort(-o["scores"].numpy(), kind="stable"):
            lab = int(o["labels"][p])
            rank[lab] = rank.get(lab, 0) + 1
            keep[p] &= rank[lab] <= 100
        return {k: v[keep] for k, v in o.items()}

    dets = [usable(o) for o in out]
    cat_ids = list(range(1, 81))
    anns = []
    for i, d in enumerate(dets):
        b = d["boxes"]
        wh = torch.stack([b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], 1)      # fp32, as the evaluator converts
        for p in range(len(b)):
            w, h = float(wh[p, 0]), float(wh[p, 1])
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": cat_ids[int(d["labels"][p])],
                         "bbox": [float(b[p, 0]), float(b[p, 1]), w, h], "area": w * h, "iscrowd": 0})
    gt = {"images": [{"id": i + 1} for i in range(len(dets))], "annotations": anns,
          "categories": [{"id": c} for c in cat_ids]}
    assert len(anns) > 50
    ev = COCOEvaluator(gt, device=DEV)
    ev.update([{k: v.to(DEV) for k, v in d.items()} for d in dets], list(range(1, len(dets) + 1)))
    ev.compute()
    calls = [[(i + 1, (d["boxes"].numpy(), d["scores"].numpy(), d["labels"].numpy())) for i, d in enumerate(dets)]]
    want, want_stats = O.evaluate(gt, calls)
    assert np.array_equal(ev.eval["precision"], want["precision"]) and np.array_equal(ev.stats, want_stats)
    # every detection matches its own GT at every threshold (IoU exactly 1), so a category with n detections has
    # pr = n / ((0 + n) + 2^-52) at every recall threshold (rule 7): 1 - 2^-52 for n = 1, rounded to 1.0 for n >= 2
    n_k = collections.Counter(a["category_id"] for a in anns)
    per_cat = np.array([ONE if n_k[c] == 1 else 1.0 for c in cat_ids if c in n_k])
    assert ev.stats[0] == np.mean(np.broadcast_to(per_cat, (10, 101, len(per_cat))).ravel())
    assert np.all(ev.eval["recall"][:, [cat_ids.index(c) for c in n_k], 0, 2] == 1.0)
    # the same detections as host tensors, and through predict_stream (one batch: the canvas, and so the
    # detections, depend on the batch's composition), which yields host tensors
    streamed = [o for batch in model.predict_stream([list(ims)]) for o in batch]
    for host in (dets, [usable(o) for o in streamed]):
        ev2 = COCOEvaluator(gt, device=DEV)
        ev2.update(host, list(range(1, len(dets) + 1)))
        ev2.compute()
        assert np.array_equal(ev2.stats, ev.stats) and np.array_equal(ev2.eval["precision"], ev.eval["precision"])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device(f"cuda:{rank}")
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        gt, calls = corpus(2, 300, n_cats=20, batch=16)
        ev = COCOEvaluator(gt, device=dev)
        feed(ev, calls[rank::world], device=dev)
        ev.compute()
        if rank == 0:
            q.put((ev.stats, ev.eval["precision"]))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two devices")
def test_two_ranks_give_the_single_process_result():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    stats, precision = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    gt, calls = corpus(2, 300, n_cats=20, batch=16)
    # the union the ranks evaluate: rank 0's calls, then rank 1's (an image keeps the first rank that had it)
    want, want_stats = O.evaluate(gt, calls[0::2] + calls[1::2])
    assert np.array_equal(stats, want_stats) and np.array_equal(precision, want["precision"])
