"""P6 variants (SURVEY.md section 8f row 2: 4 levels, stride 64, size_divisible 64). CPU: the oracle and the
host-side model containers against fixtures generated from the reference (oracle/make_golden_p6.py). GPU: the
native plan against the same fixtures."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200.models import yolov5m6, yolov5n6, yolov5s6

DEV = "cuda:0"
KW = dict(strides=util.P6_STRIDES, anchor_grids=util.P6_ANCHORS)


def _sd():
    return util.synth_state_dict(util.layouts()["n6"], knob_obj=7.0, knob_cls=4.5, seed=0, gain=util.GAIN_N6)


def test_oracle_network_p6(golden_dir):
    z = util.load_npz("network_n6.npz")
    sd = _sd()
    assert util.checksum(sd) == pytest.approx(float(z["checksum"]), rel=1e-12)
    net = R.Net(sd)
    with torch.no_grad():
        feats = net.backbone(torch.from_numpy(z["x"]))
        heads = net.head(feats)
    assert len(feats) == 4
    for i, got in enumerate(feats):
        np.testing.assert_allclose(got.numpy(), z[f"p{i + 3}"], atol=5e-5, rtol=2e-5)
    for i, got in enumerate(heads):
        np.testing.assert_allclose(got.numpy(), z[f"h{i}"], atol=5e-5, rtol=2e-5)
    dets = R.postprocess(heads, 0.15, 0.45, 300, **KW)
    util.assert_dets_close(dets[0], util.dets_from_npz(z, 1)[0], box_atol=2e-3, score_atol=1e-5, allow_tie_swaps=True)


def test_oracle_end_to_end_p6(golden_dir):
    z = util.load_npz("e2e_n6.npz")
    ims = [torch.from_numpy(z["img0"]), torch.from_numpy(z["img1"])]
    dets = R.detect(_sd(), ims, score_thresh=0.15, size=(192, 192), size_divisible=64, **KW)
    for got, ref in zip(dets, util.dets_from_npz(z, 2)):
        util.assert_dets_close(got, ref, box_atol=2e-2, score_atol=2e-5, allow_tie_swaps=True)


@pytest.mark.parametrize("name,ctor", [("n6", yolov5n6), ("s6", yolov5s6), ("m6", yolov5m6)])
def test_state_dict_layout_equals_reference_p6(name, ctor):
    ref = util.layouts()[name]
    m = ctor()
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    m.load_state_dict(util.synth_state_dict(ref))
    assert m.transform.size_divisible == 64                        # models/__init__.py:121
    assert m.model.anchor_generator.strides == util.P6_STRIDES     # yolo.py:641
    assert m.model.anchor_generator.anchor_grids == [list(map(float, a)) for a in util.P6_ANCHORS]
    assert len(m.model.head.head) == 4


def test_lowering_p6_topology():
    """72 launches for n6: 60 of the 3-level net + p6 conv/C3 (5) + one more C3 down (5) + lateral + upsample ...;
    checked structurally: every window of every concat buffer is written exactly once before it is read."""
    from yolort_b200.engine import lower_yolo

    m = yolov5n6().eval()
    L, x0, heads, feats = lower_yolo(m.model, torch.float16, torch.device("cpu"))
    assert [h.div for h in heads] == [8, 16, 32, 64] and list(feats) == ["p3", "p4", "p5", "p6"]
    written = {}
    for op in L.ops:
        for c in range(op.src.ch0, op.src.ch0 + op.src.C):
            assert (op.src.buf.name, c) in written or op.src.buf is x0, f"{op.name} reads an unwritten channel"
        for c in range(op.dst.ch0, op.dst.ch0 + op.dst.C):
            written[(op.dst.buf.name, c)] = op.name
    names = [op.name for op in L.ops]
    assert "pan.intermediate_blocks.p6.0" in names and "pan.layer_blocks.6.cv3" in " ".join(names)


# ---- GPU ----------------------------------------------------------------------------------------------
def _model():
    m = yolov5n6(size=(192, 192), score_thresh=0.15).eval()
    m.load_state_dict(_sd())
    return m.to(DEV)


@pytest.mark.gpu
def test_gpu_heads_vs_reference_fixture_p6():
    z = util.load_npz("network_n6.npz")
    m = _model()
    x = torch.from_numpy(z["x"]).to(DEV)
    dets = m.model(x)
    plan = m.model.get_plan(1, 128, 192)
    m.model.run_plan(plan)
    torch.cuda.synchronize()
    for i in range(4):
        got = plan.features[f"p{i + 3}"].float().permute(0, 3, 1, 2).cpu().numpy()
        ref = z[f"p{i + 3}"]
        rr = float(np.sqrt(((got - ref) ** 2).mean()) / np.sqrt((ref ** 2).mean()))
        print(f"p{i + 3} rel_rms {rr:.2e}")
        # this random net sits at the edge of chaos (oracle/make_golden_p6.py): rounding only the weights and the
        # input to fp16 inside the fp32 oracle already moves these maps by 4e-3; fp16 activations through ~75
        assert rr < 4e-2
        h = plan.heads[i][..., :255].float().cpu()
        got = h.view(*h.shape[:3], 3, 85).permute(0, 3, 1, 2, 4).numpy()
        ref = z[f"h{i}"]
        rr = float(np.sqrt(((got - ref) ** 2).mean()) / np.sqrt((ref ** 2).mean()))
        print(f"h{i} rel_rms {rr:.2e}")
        assert rr < 4e-2
    ref = util.dets_from_npz(z, 1)[0]
    frac = util.match_fraction(util.to_np(dets[0]), ref, iou_thr=0.9)
    # informational: on this input the top-300 of ~170 000 near-tied candidates of the edge-of-chaos net reorder
    # under fp16 (measured 0.4); detection parity of the P6 path is asserted on the e2e fixture below (0.97 / 1.0)
    print("p6 network dets matched:", frac)
    assert len(dets[0]["scores"]) == len(ref["scores"])


@pytest.mark.gpu
def test_gpu_end_to_end_vs_reference_fixture_p6():
    z = util.load_npz("e2e_n6.npz")
    m = _model()
    ims = [torch.from_numpy(z["img0"]).to(DEV), torch.from_numpy(z["img1"]).to(DEV)]
    out = m(ims)
    # (1) against the reference fixture.  This random net sits at the edge of chaos (see the heads test above) and its
    # boxes reach +-1300 px on a 192-px canvas ((2 sigmoid)^2 x 900-px anchors): a 1e-3 change of a head logit moves such a
    # box by pixels, so the coordinate tolerance of the matched pairs is relative to the BOX here, and loose; the strict
    # 1e-3-of-canvas check of the 4-level path is (2).
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.9)
        st = util.pair_stats(util.to_np(got), ref, 192.0)
        print("p6 e2e matched:", frac, len(got["scores"]), len(ref["scores"]), st)
        assert frac >= 0.95
        extent = float(np.abs(ref["boxes"]).max())
        assert st["max_box_rel"] * 192.0 <= 2e-2 * max(extent, 192.0)
    # (2) post-processing of the 4-level path, strictly: the oracle's decode + batched_nms + scale_coords applied to the
    # GPU's OWN head logits must reproduce the model's detections (labels exact, boxes within 1e-3 x canvas).
    geoms, (Hb, Wb) = m.transform.geometry(ims)
    plan = m.model.get_plan(2, Hb, Wb)
    heads = []
    for h in plan.heads:
        hh = h[..., :255].float().cpu()
        heads.append(hh.view(*hh.shape[:3], 3, 85).permute(0, 3, 1, 2, 4).contiguous())
    own = R.postprocess(heads, 0.15, 0.45, 300, R.TV_AUTO, util.P6_STRIDES, util.P6_ANCHORS)
    for got, ref, im in zip(out, own, ims):
        ref["boxes"] = R.scale_coords(ref["boxes"], Hb, Wb, int(im.shape[-2]), int(im.shape[-1]))
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.9, side=192)
        assert frac >= 0.999 and len(got["scores"]) == len(ref["scores"])


@pytest.mark.gpu
def test_gpu_s6_1280_canvas_runs():
    """The P6 models' native resolution (1280x1280, 4 levels = 102 000 anchors/image): plumbing + output contract."""
    m = yolov5s6(size=(1280, 1280), score_thresh=0.3).eval().to(DEV)
    out = m([torch.randint(0, 256, (3, 1000, 1280), dtype=torch.uint8, device=DEV)])
    assert len(out) == 1 and out[0]["boxes"].shape[1] == 4 and out[0]["boxes"].shape[0] <= 300
