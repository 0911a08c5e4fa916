"""Every case of tests/postprocess_cases.py on the H100, in two stages so that a decode difference cannot hide inside
an NMS cascade.

Decode stage: `yb_nms_begin` + `yb_decode_candidates` (or the head convolutions' fused decode epilogue) on a zeroed
workspace, then a snapshot of the candidate arena (`yb_nms_layout`).  The (anchor, class) indices in the arena must be
exactly the pairs whose fp64 score (`postprocess_cases.reference`, on the same rounded logits) is over the threshold,
except pairs within a few fp32 ulps of it (GPU expf differs from the exact exponential by up to 2 ulp); the score in each
key and the box of each candidate anchor must match fp64 within rounding.

NMS stage: `yb_nms_finish` must equal, bit for bit, `oracle.restate.batched_nms` run on the snapshot's own candidates
in row-major index order, with the boxes put through numpy fp32 `(x - pad) / gain`; so must `yb_batched_nms` on the
same candidates (explicit mode) and `_C.decode_nms`.  The arena's slots past each image's count hold zero keys, which
would sort first: a kernel that read one would return a detection the oracle does not have.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

import conv_cases as CC
from oracle import restate as R
from postprocess_cases import CASES, DTYPES, FUSED_CASES, SCORE_BAND, candidate_masks, decode64, fused_desc, \
    head_tensors, membership, postprocess_paths, reference, rescale_params
from yolort_b200 import _C
from yolort_b200.engine import pack_bias, pack_weight

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SCORE_ATOL = 2e-6      # the tolerances of tests/test_gpu_postprocess.py
BOX_ATOL, BOX_RTOL = 2e-4, 2e-6


# ---- the arena ----------------------------------------------------------------------------------------------------------
def _snapshot(ws: torch.Tensor, lay: "_C.NmsLayout", n: int) -> dict:
    base = ws.data_ptr()

    def part(ptr, count, dtype):
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return ws[ptr - base:ptr - base + nbytes].view(dtype).cpu()

    cap, apm = int(lay.cap_per_image), int(lay.anchors_per_image)
    return {"cap": cap, "apm": apm,
            "counts": part(lay.img_count, n, torch.int32).numpy().astype(np.int64),
            "keys": part(lay.keys, n * cap, torch.int64).numpy().view(np.uint64).reshape(n, cap),
            "boxes": part(lay.boxes, n * apm * 4, torch.float32).numpy().reshape(n, apm, 4)}


def _key_scores(keys: np.ndarray) -> np.ndarray:
    """decode_common.cuh from_orderable_desc of the keys' high words."""
    u = ~(keys >> np.uint64(32)).astype(np.uint32)
    u = np.where(u & np.uint32(0x80000000), u & np.uint32(0x7FFFFFFF), ~u).astype(np.uint32)
    return u.view(np.float32)


def _outputs(n: int, D: int):
    return (torch.empty((n, D, 4), dtype=torch.float32, device=DEV), torch.empty((n, D), dtype=torch.float32, device=DEV),
            torch.empty((n, D), dtype=torch.int64, device=DEV), torch.empty((n,), dtype=torch.int32, device=DEV),
            torch.empty((4,), dtype=torch.int64, device=DEV))


def run_stages(case, heads, cap: int, rescale):
    """begin + decode, snapshot, finish on a zeroed workspace with `cap` candidates per image."""
    L = _C.lib()
    n = case.n_images
    levels = (_C.HeadLevel * len(heads))(*[
        _C._level_struct(t, case.layout, case.anchors, case.K, case.strides[i], case.anchors_px[i])
        for i, t in enumerate(heads)])
    p = _C.NmsParams(n, len(heads), case.anchors, case.nc, case.thr, case.iou, case.max_det, case.semantics, cap * n)
    need = L.yb_decode_nms_workspace_bytes(ctypes.byref(p), levels)
    ws = torch.zeros((need,), dtype=torch.uint8, device=DEV)
    lay = _C.NmsLayout()
    _C.check(L.yb_nms_layout(ctypes.byref(p), levels, ws.data_ptr(), ws.numel(), ctypes.byref(lay)), "yb_nms_layout")
    boxes, scores, labels, counts, status = _outputs(n, case.max_det)
    st = _C.current_stream_ptr(DEV)
    _C.check(L.yb_nms_begin(ctypes.byref(p), levels, status.data_ptr(), ws.data_ptr(), ws.numel(), st), "yb_nms_begin")
    _C.check(L.yb_decode_candidates(ctypes.byref(p), levels, ws.data_ptr(), ws.numel(), st), "yb_decode_candidates")
    snap = _snapshot(ws, lay, n)
    _C.check(L.yb_nms_finish(ctypes.byref(p), levels, rescale.data_ptr() if rescale is not None else None,
                             boxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), counts.data_ptr(), status.data_ptr(),
                             ws.data_ptr(), ws.numel(), st), "yb_nms_finish")
    torch.cuda.synchronize()
    return snap, (boxes.cpu(), scores.cpu(), labels.cpu(), counts.cpu(), status.cpu())


# ---- decode stage -------------------------------------------------------------------------------------------------------
def _where(anchor: int, levels, A: int) -> str:
    start = 0
    for l, (h, w) in enumerate(levels):
        if anchor < start + A * h * w:
            r = anchor - start
            return f"level {l} anchor {r // (h * w)} y {r % (h * w) // w} x {r % w}"
        start += A * h * w
    return f"anchor {anchor} past the levels"


def image_candidates(snap: dict, i: int, nc: int):
    """Image i's arena entries in row-major index order: (anchors, labels, fp32 scores)."""
    keys = snap["keys"][i, :snap["counts"][i]]
    cidx = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    order = np.argsort(cidx, kind="stable")
    cidx, scores = cidx[order], _key_scores(keys)[order]
    assert len(np.unique(cidx)) == len(cidx), "an (anchor, class) pair was appended twice"
    return cidx // nc, cidx % nc, scores


def check_decode(snap, i, nc, levels, A, scores64, boxes64, scale64, sure, amb, band, box_extra=0.0):
    """The arena of image i against the fp64 decode (see the module docstring); returns the number of candidates."""
    count = int(snap["counts"][i])
    assert count <= snap["cap"]
    anchors, labels, scores = image_candidates(snap, i, nc)
    assert np.all(anchors < snap["apm"]), "candidate index past the image's anchors"
    got = np.zeros_like(sure)
    got[anchors, labels] = True
    missing, extra = sure & ~got, got & ~(sure | amb)
    for what, m in (("missing", missing), ("extra", extra)):
        if m.any():
            a, k = (int(v) for v in np.argwhere(m)[0])
            pytest.fail(f"image {i}: {int(m.sum())} {what} candidates; first {_where(a, levels, A)} class {k}: "
                        f"fp64 score {scores64[a, k]!r}, got {count} candidates, reference {int(sure.sum())} + "
                        f"{int(amb.sum())} ambiguous")
    want = scores64[anchors, labels]
    err = np.abs(scores.astype(np.float64) - want)
    tol = SCORE_ATOL + band[anchors, labels]
    assert np.all(err <= tol), f"image {i}: score error {err.max():.3g} (worst of {count} at {_where(int(anchors[np.argmax(err / tol)]), levels, A)})"
    ua = np.unique(anchors)
    berr = np.abs(snap["boxes"][i, ua].astype(np.float64) - boxes64[ua]).max(1)
    btol = BOX_ATOL + BOX_RTOL * scale64[ua] + (box_extra[ua] if np.ndim(box_extra) else box_extra)
    if np.any(berr > btol):
        j = int(np.argmax(berr / btol))
        pytest.fail(f"image {i}: box of {_where(int(ua[j]), levels, A)} off by {berr[j]:.3g}: "
                    f"{snap['boxes'][i, ua[j]].tolist()} vs {boxes64[ua[j]].tolist()}")
    return count


# ---- NMS stage ----------------------------------------------------------------------------------------------------------
def expected_nms(snap, i, nc, iou, semantics, max_det, rescale):
    """The oracle's detections on image i's snapshotted candidates: (boxes, scores, labels, candidate boxes/scores/labels,
    keep)."""
    anchors, labels, scores = image_candidates(snap, i, nc)
    boxes = snap["boxes"][i, anchors]
    keep = R.batched_nms(boxes, scores, labels, iou, semantics)[:max_det]
    b = boxes[keep].copy()
    if rescale is not None:
        gain, padx, pady = (np.float32(v) for v in rescale[i])
        b[:, 0] = (b[:, 0] - padx) / gain
        b[:, 2] = (b[:, 2] - padx) / gain
        b[:, 1] = (b[:, 1] - pady) / gain
        b[:, 3] = (b[:, 3] - pady) / gain
    return b, scores[keep], labels[keep].astype(np.int64), (boxes, scores, labels), keep


def check_nms(snap, out, nc, iou, semantics, max_det, rescale, explicit=True):
    boxes, scores, labels, counts, status = out
    n = counts.numel()
    raw = snap["counts"]
    assert int(status[0]) == int(raw.sum()) and int(status[2]) == int(raw.max())
    assert int(status[1]) == int((raw > snap["cap"]).any())
    for i in range(n):
        if raw[i] > snap["cap"]:
            assert int(counts[i]) == 0
            continue
        wb, ws, wl, cand, keep = expected_nms(snap, i, nc, iou, semantics, max_det, rescale)
        c = int(counts[i])
        assert c == len(keep), f"image {i}: {c} detections, the oracle keeps {len(keep)} of {raw[i]} candidates"
        assert torch.equal(labels[i, :c], torch.from_numpy(wl)), f"image {i}: labels differ"
        assert torch.equal(scores[i, :c], torch.from_numpy(ws)), f"image {i}: scores differ"
        assert torch.equal(boxes[i, :c], torch.from_numpy(wb)), f"image {i}: boxes differ"
        if explicit:
            cb, cs, cl = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in cand)
            got = _C.batched_nms(cb, cs, cl, iou, semantics, max_keep=max_det).cpu().numpy()
            assert np.array_equal(got, keep), f"image {i}: explicit-mode keep differs"


# ---- the decode + NMS cases ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_postprocess_case(case):
    t0 = time.perf_counter()
    heads = head_tensors(case, DEV)
    ref = reference(case)
    masks = candidate_masks(case)
    rs = rescale_params(case)
    rescale = torch.from_numpy(rs).to(DEV) if rs is not None else None
    counts = [int((s | a).sum()) for s, a in masks]
    if max(counts) > case.cap:
        # one image overflows its share: it returns no detections and flags the status; the others are unaffected
        snap, out = run_stages(case, heads, case.cap, rescale)
        assert [bool(c > case.cap) for c in snap["counts"]] == [c > case.cap for c in counts]
        check_nms(snap, out, case.nc, case.iou, case.semantics, case.max_det, rs, explicit=False)
    big = max(case.cap, max(counts) + 64)
    snap, out = run_stages(case, heads, big, rescale)
    for i in range(case.n_images):
        sure, amb = masks[i]
        check_decode(snap, i, case.nc, case.levels, case.anchors, ref.scores[i], ref.boxes[i], ref.scale[i], sure, amb,
                     SCORE_BAND * np.maximum(np.float32(case.thr), ref.scores[i]))
    check_nms(snap, out, case.nc, case.iou, case.semantics, case.max_det, rs)
    # the public entry point: the same detections, growing its arena from the case's share when an image overflows
    arena = _C._arenas.setdefault(DEV, _C._NmsArena())
    saved = arena.cap_per_image
    try:
        arena.cap_per_image, arena.ws = case.cap, None
        dets = _C.decode_nms(heads, case.layout, case.strides, case.anchors_px, case.thr, case.iou, case.max_det,
                             case.semantics, rescale, num_classes=case.nc)
        if max(counts) > case.cap:
            assert arena.cap_per_image >= max(counts), "decode_nms did not grow its arena"
    finally:
        arena.cap_per_image, arena.ws = saved, None
    boxes, scores, labels, n_det, _ = out
    for i, d in enumerate(dets):
        c = int(n_det[i])
        assert torch.equal(d["boxes"].cpu(), boxes[i, :c]) and torch.equal(d["scores"].cpu(), scores[i, :c])
        assert torch.equal(d["labels"].cpu(), labels[i, :c])
    print(f"{case.name}: candidates {snap['counts'].tolist()} (ambiguous {[int(a.sum()) for _, a in masks]}), "
          f"detections {n_det.tolist()}, {time.perf_counter() - t0:.2f} s; {sorted(postprocess_paths(case))}")


# ---- the fused decode epilogue ------------------------------------------------------------------------------------------
def _fused_operands(fc, level):
    """x [N, H, W, Cin], w [width, Cin] (rounded to the dtype) and the fp32 bias, with the objectness and class columns
    shifted."""
    g = torch.Generator().manual_seed(5000 + 10 * fc.seed + level)
    dt = DTYPES[fc.dtype]
    x = torch.randn(fc.n_images, *fc.levels[level], fc.Cin, generator=g).to(dt)
    w = (torch.randn(fc.width, fc.Cin, generator=g) * (1.5 / fc.Cin) ** 0.5).to(dt)
    b = torch.randn(fc.width, generator=g) * 0.5
    K = fc.nc + 5
    for a in range(fc.anchors):
        b[a * K + 4] += fc.obj_shift
        b[a * K + 5:(a + 1) * K] += fc.cls_shift
    return x, w, b


@pytest.mark.parametrize("fc", FUSED_CASES, ids=[c.name for c in FUSED_CASES])
def test_fused_decode_case(fc):
    """Head convolutions with the decode epilogue (conv_sm90.cu decode_fragment) against the fp64 convolution followed
    by the fp64 decode; the ambiguity band and the box tolerance widen by conv_cases.tau(Cin) times the logits'
    magnitude."""
    t0 = time.perf_counter()
    n = fc.n_images
    fp = _C.FusedPost(n, fc.levels, fc.strides, fc.anchors_px, fc.nc, fc.thr, fc.iou, fc.max_det, R.TV_AUTO, DEV,
                      cap_per_image=1 << 15)
    keep_alive, descs, lv64, mag64 = [], [], [], []
    for level in range(len(fc.levels)):
        x, w, b = _fused_operands(fc, level)
        w_conv = torch.zeros(fc.Cout, fc.Cin, 1, 1, dtype=torch.float64)   # pad channels: zero weights and bias
        w_conv[:fc.width, :, 0, 0] = w.double()
        wp, _, co_pad = pack_weight(w_conv, x.dtype, DEV)
        t = {"x": x.to(DEV), "w": wp, "b": pack_bias(b.double(), co_pad, DEV),
             "out": torch.zeros((n + 1, *fc.levels[level], fc.Cout), dtype=x.dtype, device=DEV)}
        keep_alive.append(t)
        descs.append(fused_desc(fc, level, lambda name, t=t: t[name].data_ptr(), fp.head_decode[level]))
        h, wd = fc.levels[level]
        x64, w64, b64 = x.double(), w.double(), b.double()
        lg = (x64 @ w64.T + b64).view(n, h, wd, fc.anchors, fc.nc + 5).permute(0, 3, 1, 2, 4)
        mg = (x64.abs() @ w64.abs().T + b64.abs()).view(n, h, wd, fc.anchors, fc.nc + 5).permute(0, 3, 1, 2, 4)
        lv64.append(lg.numpy())
        mag64.append(mg.numpy())
    plan = _C.Plan(descs, DEV)
    fp.ws.zero_()
    fp.begin()
    plan.run()
    snap = _snapshot(fp.ws, fp.layout, n)
    out = tuple(v.cpu() for v in fp.finish(None))
    torch.cuda.synchronize()
    scores64, boxes64, scale64 = decode64(lv64, fc.strides, fc.anchors_px)
    # logit error bound, per anchor: objectness and class logits move the score by at most score * (e_obj + e_cls),
    # the box logits move a coordinate by at most (stride + 2 * anchor) * e_box
    e = [CC.tau(fc.Cin) * m for m in mag64]
    e_obj = np.concatenate([v[..., 4].reshape(n, -1) for v in e], 1)
    e_cls = np.concatenate([v[..., 5:].reshape(n, -1, fc.nc) for v in e], 1)
    e_box = np.concatenate([(v[..., :4].max(-1) * (s + 2 * max(a))).reshape(n, -1)
                            for v, s, a in zip(e, fc.strides, fc.anchors_px)], 1)
    total = []
    for i in range(n):
        band = scores64[i] * (e_obj[i][:, None] + e_cls[i]) + SCORE_BAND * np.maximum(np.float32(fc.thr), scores64[i])
        sure, amb = membership(scores64[i], fc.thr, band)
        total.append((check_decode(snap, i, fc.nc, fc.levels, fc.anchors, scores64[i], boxes64[i], scale64[i], sure,
                                   amb, band, e_box[i]), int(amb.sum())))
    check_nms(snap, out, fc.nc, fc.iou, R.TV_AUTO, fc.max_det, None)
    del plan, keep_alive
    print(f"{fc.name}: candidates (ambiguous) {total}, detections {out[3].tolist()}, {time.perf_counter() - t0:.2f} s")
