"""Shared helpers for the parity tests."""
import json
import os

import numpy as np
import torch

from oracle.make_golden import checksum, synth_image_u8, synth_state_dict  # noqa: F401  (pure functions, no reference import)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def layouts():
    out = {}
    for fn in ("state_dict_layouts.json", "state_dict_layouts_p6.json", "state_dict_layouts_v4.json"):
        with open(os.path.join(GOLDEN, fn)) as f:
            out.update(json.load(f))
    return out


P6_STRIDES = [8, 16, 32, 64]
P6_ANCHORS = [[19, 27, 44, 40, 38, 94], [96, 68, 86, 152, 180, 137], [140, 301, 303, 264, 238, 542],
              [436, 615, 739, 380, 925, 792]]
GAIN_N6 = 2.22   # oracle/make_golden_p6.py
GAINS_V4 = {"s_r40": 2.1, "s_r31": 2.05}   # oracle/make_golden_v4.py


def load_npz(name):
    return dict(np.load(os.path.join(GOLDEN, name)))


def dets_from_npz(z, n):
    return [{k: z[f"det{i}_{k}"] for k in ("scores", "labels", "boxes")} for i in range(n)]


def assert_dets_close(got, ref, box_atol, score_atol, allow_tie_swaps=False):
    """got/ref: dicts of numpy arrays. Labels and order exact unless equal scores swap places."""
    assert len(got["scores"]) == len(ref["scores"]), (len(got["scores"]), len(ref["scores"]))
    if len(ref["scores"]) == 0:
        return
    gl, rl = np.asarray(got["labels"]), np.asarray(ref["labels"])
    gb, rb = np.asarray(got["boxes"], dtype=np.float64), np.asarray(ref["boxes"], dtype=np.float64)
    gs, rs = np.asarray(got["scores"], dtype=np.float64), np.asarray(ref["scores"], dtype=np.float64)
    np.testing.assert_allclose(gs, rs, atol=score_atol, rtol=0)
    if allow_tie_swaps and not np.array_equal(gl, rl):
        # compare as multisets within groups of (nearly) equal score
        order_g = np.lexsort((gb[:, 0], gb[:, 1], gl, -np.round(gs, 6)))
        order_r = np.lexsort((rb[:, 0], rb[:, 1], rl, -np.round(rs, 6)))
        gl, rl, gb, rb = gl[order_g], rl[order_r], gb[order_g], rb[order_r]
    assert np.array_equal(gl, rl)
    np.testing.assert_allclose(gb, rb, atol=box_atol, rtol=0)


def rel_rms(got, ref):
    """Root mean square of got - ref over that of ref."""
    return float(np.sqrt(((got - ref) ** 2).mean()) / np.sqrt((ref ** 2).mean()))


def head_logits(plan, i, anchors=3, outputs=85):
    """Head buffer i of `plan` as the reference's [N, A, H, W, K] logits (numpy, fp32)."""
    h = plan.heads[i][..., :anchors * outputs].float().cpu()
    n, hh, ww, _ = h.shape
    return h.view(n, hh, ww, anchors, outputs).permute(0, 3, 1, 2, 4).numpy()


def assert_repeat_and_graph_replay_bit_identical(plan):
    """`plan` (input written) run twice eagerly, then twice as one CUDA graph with its heads zeroed before each replay:
    every run gives the first run's heads bit for bit."""
    plan.run()
    torch.cuda.synchronize()
    eager = [h.clone() for h in plan.heads]
    plan.run()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, plan.heads))
    plan.use_graph = True
    for _ in range(2):
        for h in plan.heads:
            h.zero_()
        plan.run()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(eager, plan.heads))


def to_np(d):
    return {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _iou_matrix(a, b):
    x1 = np.maximum(a[:, None, 0], b[None, :, 0]); y1 = np.maximum(a[:, None, 1], b[None, :, 1])
    x2 = np.minimum(a[:, None, 2], b[None, :, 2]); y2 = np.minimum(a[:, None, 3], b[None, :, 3])
    inter = np.clip(x2 - x1, 0, None) * np.clip(y2 - y1, 0, None)
    aa = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]); ab = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    return inter / (aa[:, None] + ab[None, :] - inter + 1e-12)


def match_fraction(got, ref, iou_thr=0.9, side=None, box_rel=None):
    """Fraction of reference detections that have a same-label detection with IoU > iou_thr (SURVEY.md 8c.2).
    With `side` (canvas / image side in pixels) the one-to-one matched pairs must also agree to `box_rel` x side in
    every coordinate (default BOX_REL_TOL = 1e-3, north_star's tolerance); labels of matched pairs are equal by
    construction."""
    if side is not None:
        st = pair_stats(got, ref, float(side), iou_thr)
        tol = BOX_REL_TOL if box_rel is None else box_rel
        assert st["max_box_rel"] <= tol, f"matched boxes differ by {st['max_box_rel']:.2e} x side (> {tol:.0e}): {st}"
        return st["matched"]
    if len(ref["scores"]) == 0:
        return 1.0 if len(got["scores"]) == 0 else 0.0
    if len(got["scores"]) == 0:
        return 0.0
    iou = _iou_matrix(np.asarray(ref["boxes"], dtype=np.float64), np.asarray(got["boxes"], dtype=np.float64))
    same = np.asarray(ref["labels"])[:, None] == np.asarray(got["labels"])[None, :]
    return float(((iou > iou_thr) & same).any(axis=1).mean())


# ---------------------------------------------------------------------------------------------------
# north_star tolerance (BASELINE.json): class indices bit-exact, boxes within 1e-3 relative (x canvas side) of the
# reference, on the detections both sides agree exist (SURVEY.md 8c.2: greedy match by label and IoU > 0.9)
# ---------------------------------------------------------------------------------------------------
BOX_REL_TOL = 1e-3


def pair_stats(got, ref, side: float, iou_thr: float = 0.9):
    """One-to-one greedy matching of reference detections (score-descending) to same-label detections of `got` with
    IoU > iou_thr.  Returns matched fraction of the reference, and over the matched pairs: the largest coordinate
    difference relative to the canvas side, the fraction within BOX_REL_TOL, and the largest score difference."""
    nr, ng = len(ref["scores"]), len(got["scores"])
    st = {"n_ref": nr, "n_got": ng, "matched": 1.0 if nr == 0 and ng == 0 else 0.0, "within": 1.0, "max_box_rel": 0.0,
          "max_score_err": 0.0, "labels_equal": True}
    if nr == 0 or ng == 0:
        return st
    rb, gb = np.asarray(ref["boxes"], dtype=np.float64), np.asarray(got["boxes"], dtype=np.float64)
    rl, gl = np.asarray(ref["labels"]), np.asarray(got["labels"])
    rs, gs = np.asarray(ref["scores"], dtype=np.float64), np.asarray(got["scores"], dtype=np.float64)
    iou = _iou_matrix(rb, gb)
    ok = (iou > iou_thr) & (rl[:, None] == gl[None, :])
    taken = np.zeros(ng, dtype=bool)
    errs, serrs = [], []
    for i in np.argsort(-rs, kind="stable"):
        cand = np.nonzero(ok[i] & ~taken)[0]
        if cand.size == 0:
            continue
        j = cand[np.argmax(iou[i, cand])]
        taken[j] = True
        errs.append(np.abs(rb[i] - gb[j]).max() / side)
        serrs.append(abs(rs[i] - gs[j]))
    st["matched"] = len(errs) / nr
    if errs:
        e = np.asarray(errs)
        st["within"] = float((e <= BOX_REL_TOL).mean())
        st["max_box_rel"] = float(e.max())
        st["max_score_err"] = float(max(serrs))
    return st


def assert_e2e_parity(name, got_list, ref_list, side, min_matched, min_within, max_box_rel, max_score_err, iou_thr=0.9):
    """Every image: labels of matched pairs are equal by construction of the matching (bit-exact class indices);
    matched fraction >= min_matched; >= min_within of the matched boxes within 1e-3 x side, none beyond max_box_rel."""
    tot = {"n_ref": 0, "n_pairs": 0.0, "within_w": 0.0}
    worst = {"matched": 1.0, "within": 1.0, "max_box_rel": 0.0, "max_score_err": 0.0}
    for k, (got, ref) in enumerate(zip(got_list, ref_list)):
        st = pair_stats(to_np(got), ref, side, iou_thr)
        tot["n_ref"] += st["n_ref"]
        tot["n_pairs"] += st["matched"] * st["n_ref"]
        tot["within_w"] += st["within"] * st["matched"] * st["n_ref"]
        worst["matched"] = min(worst["matched"], st["matched"])
        worst["within"] = min(worst["within"], st["within"])
        worst["max_box_rel"] = max(worst["max_box_rel"], st["max_box_rel"])
        worst["max_score_err"] = max(worst["max_score_err"], st["max_score_err"])
    matched = tot["n_pairs"] / max(tot["n_ref"], 1)
    within = tot["within_w"] / max(tot["n_pairs"], 1)
    print(f"PARITY {name}: ref dets {tot['n_ref']} matched {matched:.4f} (worst image {worst['matched']:.4f}) "
          f"within 1e-3*side {within:.4f} (worst {worst['within']:.4f}) max |dbox|/side {worst['max_box_rel']:.2e} "
          f"max |dscore| {worst['max_score_err']:.2e}")
    assert tot["n_ref"] > 0, "the oracle produced no detections: the test would be vacuous"
    assert matched >= min_matched, (matched, min_matched)
    assert within >= min_within, (within, min_within)
    assert worst["max_box_rel"] <= max_box_rel, worst
    assert worst["max_score_err"] <= max_score_err, worst
    return {"matched": matched, "within_1e-3": within, **worst}
