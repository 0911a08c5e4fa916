"""r4.0 / r3.1 families (SURVEY.md section 8f row 4: Focus stem, BottleneckCSP + LeakyReLU, Hardswish, SPP inside
the body). CPU: oracle + host containers + weight transforms against fixtures generated from the reference
(oracle/make_golden_v4.py). GPU: the native plan against the same fixtures."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parity_util as util
from oracle import restate as R
from yolort_b200.models import yolov5l, yolov5m, yolov5n, yolov5s

DEV = "cuda:0"
TAGS = [("s_r40", "r4.0"), ("s_r31", "r3.1")]


def _sd(tag):
    return util.synth_state_dict(util.layouts()[tag], knob_obj=7.0, knob_cls=4.5, seed=0, gain=util.GAINS_V4[tag])


@pytest.mark.parametrize("tag,ver", TAGS)
def test_oracle_network_v4(tag, ver, golden_dir):
    z = util.load_npz(f"network_{tag}.npz")
    sd = _sd(tag)
    assert util.checksum(sd) == pytest.approx(float(z["checksum"]), rel=1e-12)
    net = R.Net(sd)
    assert net.focus and net.r31 == (ver == "r3.1")
    with torch.no_grad():
        feats = net.backbone(torch.from_numpy(z["x"]))
        heads = net.head(feats)
    for i, got in enumerate(feats):
        np.testing.assert_allclose(got.numpy(), z[f"p{i + 3}"], atol=2e-5, rtol=1e-5)
    for i, got in enumerate(heads):
        np.testing.assert_allclose(got.numpy(), z[f"h{i}"], atol=2e-5, rtol=1e-5)
    dets = R.postprocess(heads, 0.15, 0.45, 300)
    util.assert_dets_close(dets[0], util.dets_from_npz(z, 1)[0], box_atol=1e-3, score_atol=1e-5, allow_tie_swaps=True)


@pytest.mark.parametrize("tag,ver", TAGS)
def test_oracle_end_to_end_v4(tag, ver, golden_dir):
    z = util.load_npz(f"e2e_{tag}.npz")
    ims = [torch.from_numpy(z["img0"]), torch.from_numpy(z["img1"])]
    dets = R.detect(_sd(tag), ims, score_thresh=0.15, size=(128, 128))
    for got, ref in zip(dets, util.dets_from_npz(z, 2)):
        util.assert_dets_close(got, ref, box_atol=2e-2, score_atol=2e-5, allow_tie_swaps=True)


@pytest.mark.parametrize("size,ctor", [("s", yolov5s), ("m", yolov5m), ("l", yolov5l)])
@pytest.mark.parametrize("ver", ["r3.1", "r4.0"])
def test_state_dict_layout_equals_reference_v4(size, ctor, ver):
    ref = util.layouts()[f"{size}_{ver.replace('.', '')}"]
    m = ctor(upstream_version=ver)
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    m.load_state_dict(util.synth_state_dict(ref))


def test_version_surface():
    with pytest.raises(NotImplementedError):
        yolov5n(upstream_version="r4.0")           # models/__init__.py:32-35: n exists for r6.0 only
    with pytest.raises(NotImplementedError):
        yolov5s(upstream_version="r5.0")
    assert type(yolov5s(upstream_version="r3.1").model.backbone.body["2"]).__name__ == "BottleneckCSP"
    assert type(yolov5s(upstream_version="r4.0").model.backbone.body["0"]).__name__ == "Focus"


def test_focus_weight_permutation_is_exact():
    """Focus (common.py:230-240) == 3x3/s1/p1 conv over the plan's space-to-depth input with permuted weights."""
    from yolort_b200.engine import focus_to_s2d

    g = torch.Generator().manual_seed(0)
    x = torch.rand(2, 3, 16, 24, generator=g, dtype=torch.float64)
    w = torch.randn(8, 12, 3, 3, generator=g, dtype=torch.float64)
    want = F.conv2d(torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1), w, padding=1)
    s2d = torch.zeros(2, 16, 8, 12, dtype=torch.float64)         # channel (dy*2+dx)*4 + c, c == 3 zero
    for dy in range(2):
        for dx in range(2):
            s2d[:, (dy * 2 + dx) * 4:(dy * 2 + dx) * 4 + 3] = x[..., dy::2, dx::2]
    got = F.conv2d(s2d, focus_to_s2d(w), padding=1)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("ver,n_ops", [("r4.0", 57), ("r3.1", 73)])
def test_lowering_v4_topology(ver, n_ops):
    from yolort_b200 import _C
    from yolort_b200.engine import lower_yolo

    m = yolov5s(upstream_version=ver).eval()
    L, x0, heads, feats = lower_yolo(m.model, torch.float16, torch.device("cpu"))
    assert len(L.ops) == n_ops and [h.div for h in heads] == [8, 16, 32]
    written = set()
    for op in L.ops:
        for c in range(op.src.ch0, op.src.ch0 + op.src.C):
            assert (op.src.buf.name, c) in written or op.src.buf is x0, f"{op.name} reads an unwritten channel"
        written.update((op.dst.buf.name, c) for c in range(op.dst.ch0, op.dst.ch0 + op.dst.C))
    acts = {op.act for op in L.ops if op.kind == _C.YB_OP_CONV}
    want = {_C.YB_ACT_NONE, _C.YB_ACT_SILU} if ver == "r4.0" else {_C.YB_ACT_NONE, _C.YB_ACT_HARDSWISH, _C.YB_ACT_LEAKY01}
    assert acts == want


# ---- GPU ----------------------------------------------------------------------------------------------
def _model(tag, ver):
    m = yolov5s(upstream_version=ver, size=(128, 128), score_thresh=0.15).eval()
    m.load_state_dict(_sd(tag))
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("tag,ver", TAGS)
def test_gpu_heads_vs_reference_fixture_v4(tag, ver):
    z = util.load_npz(f"network_{tag}.npz")
    m = _model(tag, ver)
    x = torch.from_numpy(z["x"]).to(DEV)
    dets = m.model(x)
    plan = m.model.get_plan(1, 96, 128)
    m.model.run_plan(plan)
    torch.cuda.synchronize()
    for i in range(3):
        got = plan.features[f"p{i + 3}"].float().permute(0, 3, 1, 2).cpu().numpy()
        ref = z[f"p{i + 3}"]
        rr = float(np.sqrt(((got - ref) ** 2).mean()) / np.sqrt((ref ** 2).mean()))
        h = plan.heads[i][..., :255].float().cpu()
        goth = h.view(*h.shape[:3], 3, 85).permute(0, 3, 1, 2, 4).numpy()
        refh = z[f"h{i}"]
        rh = float(np.sqrt(((goth - refh) ** 2).mean()) / np.sqrt((refh ** 2).mean()))
        print(f"{tag} p{i + 3} rel_rms {rr:.2e}  h{i} rel_rms {rh:.2e}")
        assert rr < 2e-2 and rh < 2e-2
    ref = util.dets_from_npz(z, 1)[0]
    frac = util.match_fraction(util.to_np(dets[0]), ref, iou_thr=0.9)
    print(tag, "network dets matched:", frac)
    assert frac >= 0.97      # measured 0.993 / 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("tag,ver", TAGS)
def test_gpu_end_to_end_vs_reference_fixture_v4(tag, ver):
    z = util.load_npz(f"e2e_{tag}.npz")
    m = _model(tag, ver)
    ims = [torch.from_numpy(z["img0"]).to(DEV), torch.from_numpy(z["img1"]).to(DEV)]
    out = m(ims)
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.9)
        print(tag, "e2e matched:", frac, len(got["scores"]), len(ref["scores"]))
        assert frac >= 0.95      # measured 0.973 .. 1.0
