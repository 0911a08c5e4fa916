"""Test-time augmentation on the CPU: the host pass geometry and the oracle restatement (oracle/restate_tta.py)
against fixtures generated from the unmodified reference (oracle/make_golden_tta.py)."""
import json
import os

import numpy as np
import torch

import parity_util as util
from oracle import restate_tta as RT
from yolort_b200 import _C


def test_pass_geometry_matches_reference():
    with open(os.path.join(util.GOLDEN, "tta_geometry.json")) as f:
        entries = json.load(f)
    assert len(entries) > 100
    for e in entries:
        want = [tuple(p) for p in e["passes"]]
        assert _C.tta_pass_geometry(e["H"], e["W"], e["gs"]) == want, e
        assert RT.pass_geometry(e["H"], e["W"], e["gs"]) == want, e


def test_restated_canvases_bit_exact():
    z = util.load_npz("tta.npz")
    for c, (h, w, gs) in enumerate(z["canvas_shapes"].tolist()):
        x = z[f"c{c}_x"]
        for q, s in enumerate(RT.SCALES):
            if q == 0:
                continue
            for flip in (None, 3):
                want = z[f"c{c}_s{q}_f{flip or 0}"]
                got = RT.scale_img(x, s, flip, gs)
                assert got.shape == want.shape, (c, q, flip)
                np.testing.assert_array_equal(got, want, err_msg=f"canvas {h}x{w} scale {s} flip {flip}")


def test_restated_descale_and_clip_bit_exact():
    z = util.load_npz("tta.npz")
    for q, (s, f) in enumerate(zip(RT.SCALES, RT.FLIPS)):
        np.testing.assert_array_equal(RT.descale(z["pred"], f, s, (96, 160)), z[f"descale{q}"])
    out = RT.clip_augmented([z[f"clip_in{k}"] for k in range(3)], 3)
    for k in range(3):
        np.testing.assert_array_equal(out[k], z[f"clip_out{k}"])


def _e2e(name, gain, strides, anchors):
    z = util.load_npz(f"e2e_tta_{name}.npz")
    kw = {} if gain is None else {"gain": gain}
    sd = util.synth_state_dict(util.layouts()[name], knob_obj=7.0, knob_cls=4.5, seed=0, **kw)
    ims = [torch.from_numpy(z["img0"]), torch.from_numpy(z["img1"])]
    got = RT.detect(sd, ims, score_thresh=0.15, size=(128, 128), size_divisible=int(max(strides)), strides=strides,
                    anchor_grids=anchors)
    for g, r in zip(got, util.dets_from_npz(z, 2)):
        util.assert_dets_close(g, r, box_atol=2e-5 * 128, score_atol=2e-5, allow_tie_swaps=True)


def test_restated_end_to_end_n():
    _e2e("n", None, [8, 16, 32], [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]])


def test_restated_end_to_end_n6():
    _e2e("n6", util.GAIN_N6, util.P6_STRIDES, util.P6_ANCHORS)
