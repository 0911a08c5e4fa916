"""yolov5ts: r4.0 with the C3TR transformer block as the first block of the neck.  CPU: constructor surface, state-dict
layout, lowering topology, exactness of the weight folding, the CPU oracle against fixtures generated from the
reference (oracle/make_golden_ts.py) and the attention op's descriptor validation.  GPU: the native plan stage by
stage, against the fixtures, and under CUDA-graph replay."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

import parity_util as util
import stagewise as S
from oracle import restate_ts as RT
from oracle.make_golden_ts import SCORE_THRESH, SIZE, e2e_images, network_input, stored_part, synth_state_dict_ts
from oracle.restate import postprocess
from yolort_b200 import _C
from yolort_b200.models import yolov5ts

DEV = "cuda:0"
PREFIX = "model.backbone.pan.inner_blocks.0"


def _layout():
    with open(os.path.join(util.GOLDEN, "state_dict_layouts_ts.json")) as f:
        return json.load(f)["ts"]


def _sd():
    return synth_state_dict_ts(_layout())


# ---- CPU -------------------------------------------------------------------------------------------------------
def test_state_dict_layout_equals_reference_ts():
    ref = _layout()
    m = yolov5ts()
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    assert list(sd[f"{PREFIX}.m.tr.0.ma.in_proj_weight"].shape) == [768, 256]
    assert not any(k.startswith(f"{PREFIX}.m.0.") for k in sd)
    m.load_state_dict(_sd(), strict=True)


def test_constructor_surface_ts():
    from yolort_b200.models import yolo

    m = yolov5ts(upstream_version="r4.0", export_friendly=False)
    assert m.arch == "yolov5_darknet_tan_s_r40" and "yolov5_darknet_tan_s_r40" in yolo.__all__
    assert type(m.model.backbone.pan.inner_blocks[0]).__name__ == "C3TR"
    assert type(m.model.backbone.pan).__name__ == "TransformerAttentionNetwork"
    assert type(m.model.backbone.body["8"]).__name__ == "SPP"
    for ver in ("r6.0", "r3.1"):
        with pytest.raises(NotImplementedError):
            yolov5ts(upstream_version=ver)
    from yolort_b200.models.transformer import darknet_tan_backbone

    with pytest.raises(NotImplementedError):
        darknet_tan_backbone("darknet_s_r6_0", 0.33, 0.5, version="r6.0")
    with pytest.raises(NotImplementedError):
        darknet_tan_backbone("darknet_s_r4_0", 0.33, 0.5, use_p6=True)


def test_lowering_ts_topology():
    from yolort_b200.engine import lower_yolo

    m = yolov5ts().eval()
    L, x0, heads, feats = lower_yolo(m.model, torch.float16, torch.device("cpu"))
    kinds = [op.kind for op in L.ops]
    assert len(L.ops) == 60 and kinds.count(_C.YB_OP_ATTENTION) == 1
    assert kinds.count(_C.YB_OP_SPP_POOL) == 1 and kinds.count(_C.YB_OP_UPSAMPLE2X) == 2
    written = set()
    for op in L.ops:
        for v in (op.src, op.residual):
            if v is None:
                continue
            for c in range(v.ch0, v.ch0 + v.C):
                assert (v.buf.name, c) in written or v.buf is x0, f"{op.name} reads an unwritten channel"
        written.update((op.dst.buf.name, c) for c in range(op.dst.ch0, op.dst.ch0 + op.dst.C))
    names = [op.name for op in L.ops if op.name.startswith("pan.inner_blocks.0")]
    assert names == ["pan.inner_blocks.0.cv1+cv2", "pan.inner_blocks.0.m.linear(pos)",
                     "pan.inner_blocks.0.m.tr.0.q|k|v+in_proj", "pan.inner_blocks.0.m.tr.0.ma(attention)",
                     "pan.inner_blocks.0.m.tr.0.ma.out_proj", "pan.inner_blocks.0.m.tr.0.fc2*fc1", "pan.inner_blocks.0.cv3"]
    ops = {op.name: op for op in L.ops}
    att = ops["pan.inner_blocks.0.m.tr.0.ma(attention)"]
    assert att.ksize == 4 and att.src.C == 768 and att.src.ch0 == 0 and att.dst.C == 256 and att.dst.buf.div == 32
    assert att.weight is None and att.bias is None and att.residual is None and att.act == _C.YB_ACT_NONE
    qkv = ops["pan.inner_blocks.0.m.tr.0.q|k|v+in_proj"]
    assert qkv.dst.buf is att.src.buf and qkv.act == _C.YB_ACT_NONE
    out = ops["pan.inner_blocks.0.m.tr.0.ma.out_proj"]
    pos = ops["pan.inner_blocks.0.m.linear(pos)"]
    assert out.src.buf is att.dst.buf and out.residual.buf is pos.dst.buf
    fc = ops["pan.inner_blocks.0.m.tr.0.fc2*fc1"]
    assert fc.residual.buf is out.dst.buf and fc.src.buf is out.dst.buf
    assert fc.dst.buf.name == "pan.inner_blocks.0.cat" and fc.dst.ch0 == 0 and fc.dst.C == 256
    assert pos.src.buf is fc.dst.buf and pos.src.ch0 == 0
    E = 256
    assert [pos.flops_per_pixel, qkv.flops_per_pixel, out.flops_per_pixel, fc.flops_per_pixel] == \
        [2 * E * E, 12 * E * E, 2 * E * E, 4 * E * E]
    # no pointwise chain is marked inside the block
    assert all(op.chain_own == 0 for op in L.ops if op.name.startswith("pan.inner_blocks.0"))


def test_fold_exactness_transformer_layer():
    """pos / qkv / out / fc as folded by the lowering reproduce TransformerBlock (common.py:328-357) computed module by
    module in float64 with torch's own nn.MultiheadAttention, given the same attention core."""
    from yolort_b200.engine import _Lowering, _Buf, _View
    from yolort_b200.models.common import TransformerBlock

    torch.manual_seed(0)
    E, Lt, N = 256, 37, 3
    tb = TransformerBlock(E, E, 4, 1).double().eval()
    with torch.no_grad():
        for p in tb.parameters():    # fp32-representable: the plan keeps its biases in fp32
            p.copy_(torch.randn(p.shape, dtype=torch.float32).mul_(0.1).double())
    low = _Lowering(torch.float64, torch.device("cpu"))
    src = _View(_Buf("in", 32, 2 * E), 0, E)
    low.transformer("t", tb, src, _View(src.buf, 0, E))
    ops = low.ops
    x = torch.randn(Lt, N, E, dtype=torch.float64)

    def conv(op, t, res=None):
        w = op.weight[:op.dst.C, 0, :op.src.C]
        y = t @ w.T + op.bias[:op.dst.C].double()
        return y if res is None else y + res

    p = conv(ops[0], x)
    qkv = conv(ops[1], p)
    assert ops[2].kind == _C.YB_OP_ATTENTION
    q, k, v = (qkv[..., i * E:(i + 1) * E].reshape(Lt, N, 4, 64).permute(1, 2, 0, 3) for i in range(3))
    a = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ v
    a = a.permute(2, 0, 1, 3).reshape(Lt, N, E)
    x1 = conv(ops[3], a, p)
    got = conv(ops[4], x1, x1)
    layer = tb.tr[0]
    with torch.no_grad():
        want_p = x + tb.linear(x)
        want_x1 = layer.ma(layer.q(want_p), layer.k(want_p), layer.v(want_p), need_weights=False)[0] + want_p
        want = layer.fc2(layer.fc1(want_x1)) + want_x1
    torch.testing.assert_close(p, want_p, rtol=0, atol=1e-10)
    torch.testing.assert_close(x1, want_x1, rtol=0, atol=1e-10)
    torch.testing.assert_close(got, want, rtol=0, atol=1e-10)


def test_oracle_network_ts():
    z = util.load_npz("network_ts.npz")
    sd = _sd()
    assert util.checksum(sd) == pytest.approx(float(z["checksum"]), rel=1e-12)
    x = network_input()
    assert float(x.double().sum()) == pytest.approx(float(z["x_checksum"]), rel=1e-12)
    net = RT.NetTS(sd)
    with torch.no_grad():
        feats = net.backbone(x)
        heads = net.head(feats)
    for i, got in enumerate(feats):
        np.testing.assert_allclose(stored_part(f"p{i + 3}", got), z[f"p{i + 3}"], atol=2e-5, rtol=1e-5)
    for i, got in enumerate(heads):
        np.testing.assert_allclose(stored_part(f"h{i}", got), z[f"h{i}"], atol=2e-5, rtol=1e-5)
    dets = postprocess(heads, SCORE_THRESH, 0.45, 300)
    ref = util.dets_from_npz(z, 1)[0]
    assert 0 < len(ref["scores"]) < 300
    # near-equal scores of neighbouring candidates may swap rank order between two fp32 CPU runs: matched by box
    assert util.match_fraction(util.to_np(dets[0]), ref, iou_thr=0.99) >= 0.97
    # non-vacuity: the fixture's attention is far from uniform (the oracle's probabilities match the reference's)
    a = net.attention[0]
    L = a.shape[-1]
    ent = float(-(a * a.clamp_min(1e-30).log()).sum(-1).mean())
    assert L == 100 and ent < 0.8 * math.log(L)
    assert ent == pytest.approx(float(z["attn_entropy"]), rel=1e-4)


def test_oracle_end_to_end_ts():
    z = util.load_npz("e2e_ts.npz")
    ims = e2e_images()
    assert sum(int(im.sum()) for im in ims) == int(z["img_checksum"])
    dets = RT.detect(_sd(), ims, score_thresh=SCORE_THRESH, size=SIZE)
    for got, ref in zip(dets, util.dets_from_npz(z, 2)):
        util.assert_dets_close(got, ref, box_atol=2e-2, score_atol=2e-5, allow_tie_swaps=True)


def _attn_desc(**kw):
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_ATTENTION, _C.dtype_code(torch.float16)
    d.N, d.H, d.W, d.Ho, d.Wo = 2, 20, 20, 20, 20
    d.Cin, d.in_cstride, d.in_ = 768, 768, 4096
    d.Cout, d.out_cstride, d.out = 256, 256, 8192
    d.ksize = 4
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("field,value,msg", [
    ("dtype", _C.YB_F32, "dtype"),
    ("ksize", 3, "multiple of the 3 heads"),
    ("ksize", 2, "head_dim must be 64"),
    ("Cin", 760, "Cin must be 3E"),
    ("in_cstride", 772, "multiples of 8"),
    ("out_cstride", 260, "multiples of 8"),
    ("in_", 4096 + 8, "16-byte aligned"),
    ("out", 8192 + 4, "16-byte aligned"),
    ("H", 0, "empty sequence"),
    ("act", _C.YB_ACT_SILU, "act and reserved"),
    ("reserved", 8, "act and reserved"),
    ("weight", 4096, "must be NULL"),
    ("residual", 4096, "must be NULL"),
])
def test_attention_descriptor_rejections(field, value, msg):
    """yb_plan_create validates an attention op before any driver call: no GPU is needed to be refused."""
    d = _attn_desc(**{field: value})
    if field == "H":
        d.Ho = 0
    arr = (_C.OpDesc * 1)(d)
    h = ctypes.c_void_p()
    lib = _C.lib()
    rc = lib.yb_plan_create(arr, 1, ctypes.byref(h))
    assert rc == -1 and not h.value
    err = lib.yb_last_error().decode()
    assert "attention" in err and msg in err, err


# ---- GPU -------------------------------------------------------------------------------------------------------
def _model():
    m = yolov5ts(size=SIZE, score_thresh=SCORE_THRESH).eval()
    m.load_state_dict(_sd())
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("N,hw,dtype", [(32, 640, torch.float16), (4, 1280, torch.bfloat16)])
def test_gpu_stagewise_ts(N, hw, dtype):
    """Every launch of the yolov5ts plan against fp32 PyTorch on its own rounded input (attention: fp32 SDPA)."""
    from yolort_b200.engine import Engine

    m = yolov5ts().eval()
    m.load_state_dict(_sd())
    m = m.to(DEV)
    eng = Engine(m.model, dtype, torch.device(DEV))
    plan = eng.plan(N, hw, hw, keep_intermediates=True)
    g = torch.Generator(device=DEV).manual_seed(3)
    plan.input.copy_(torch.rand(plan.input.shape, generator=g, device=DEV).to(dtype))
    plan.input[..., 3::4] = 0
    res = S.check_plan_stagewise(plan, m.model.backbone.body["0"])
    assert len(res) == len(plan._low.L.ops)
    att = [r for r in res if "attention" in r.name]
    assert len(att) == 1
    bad = [r for r in res if r.violations]
    assert not bad, bad


@pytest.mark.gpu
def test_gpu_heads_vs_reference_fixture_ts():
    z = util.load_npz("network_ts.npz")
    m = _model()
    x = network_input().to(DEV)
    dets = m.model(x)
    plan = m.model.get_plan(1, *SIZE)
    m.model.run_plan(plan)
    torch.cuda.synchronize()
    for i in range(3):
        got = plan.features[f"p{i + 3}"].float().permute(0, 3, 1, 2).cpu().numpy()
        rr = util.rel_rms(stored_part(f"p{i + 3}", got), z[f"p{i + 3}"])
        rh = util.rel_rms(stored_part(f"h{i}", util.head_logits(plan, i)), z[f"h{i}"])
        print(f"ts p{i + 3} rel_rms {rr:.2e}  h{i} rel_rms {rh:.2e}")
        assert rr < 2e-2 and rh < 2e-2
    frac = util.match_fraction(util.to_np(dets[0]), util.dets_from_npz(z, 1)[0], iou_thr=0.9)
    print("ts network dets matched:", frac)
    assert frac >= 0.97


@pytest.mark.gpu
def test_gpu_end_to_end_vs_reference_fixture_ts():
    z = util.load_npz("e2e_ts.npz")
    m = _model()
    out = m([im.to(DEV) for im in e2e_images()])
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        print("ts e2e:", len(got["scores"]), len(ref["scores"]))
        if len(ref["scores"]) == 0:
            assert len(got["scores"]) <= 2
            continue
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.9)
        print("ts e2e matched:", frac)
        assert frac >= 0.95


@pytest.mark.gpu
def test_gpu_graph_replay_and_repeat_are_bit_identical_ts():
    from yolort_b200.engine import Engine

    m = yolov5ts().eval()
    m.load_state_dict(_sd())
    m = m.to(DEV)
    eng = Engine(m.model, torch.float16, torch.device(DEV))
    plan = eng.plan(8, 640, 480)
    g = torch.Generator(device=DEV).manual_seed(4)
    plan.input.copy_(torch.rand(plan.input.shape, generator=g, device=DEV).half())
    plan.input[..., 3::4] = 0
    util.assert_repeat_and_graph_replay_bit_identical(plan)
