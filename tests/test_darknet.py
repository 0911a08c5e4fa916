"""DarkNetV4 / DarkNetV6 image classifiers (CPU): constructor surface and state-dict layout against the reference,
lowering topology, weight identity with the detection body, the CPU oracle against fixtures generated from the
reference (oracle/make_golden_darknet.py) and the descriptor validation of YB_OP_AVGPOOL."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from torch import nn

import parity_util as util
from oracle.make_golden_darknet import INPUTS, NC10, NETWORK_ARCHS, network_input, stored_features, \
    synth_state_dict_darknet
from oracle.restate_darknet import NetDarknet
from yolort_b200 import _C
from yolort_b200.models import darknet as D
from yolort_b200.models import darknetv4, darknetv6


def _fixture():
    with open(os.path.join(util.GOLDEN, "state_dict_layouts_darknet.json")) as f:
        return json.load(f)


def _sd(arch, seed=0):
    return synth_state_dict_darknet(_fixture()["layouts"][arch], seed)


@pytest.mark.parametrize("arch", list(_fixture()["layouts"]))
def test_state_dict_layout_equals_reference_darknet(arch):
    ref = _fixture()["layouts"][arch]
    m = D.darknet_s_r6_0(num_classes=10) if arch == NC10 else getattr(D, arch)()
    sd = m.state_dict()
    assert list(sd) == list(ref)
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    m.load_state_dict(_sd(arch), strict=True)
    bns = [mod for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    assert bns and all(b.eps == 1e-3 and b.momentum == 0.03 for b in bns)


def test_star_import_and_constructor_surface():
    ns = {}
    exec("from yolort_b200.models.darknet import *", ns)
    assert list(D.__all__) == _fixture()["all"]
    assert {k for k in ns if not k.startswith("__")} == set(D.__all__)
    assert darknetv6.model_urls == {f"darknet_{s}_r6.0": None for s in "nsmlx"}
    assert darknetv4.model_urls == {f"darknet_{s}_r{v}": None for v in ("3.1", "4.0") for s in "sml"}
    with pytest.raises(NotImplementedError, match=r"^pretrained darknet_s_r6\.0 is not supported as of now$"):
        D.darknet_s_r6_0(pretrained=True)
    with pytest.raises(NotImplementedError, match=r"pretrained darknet_m_r3\.1 is not"):
        D.darknet_m_r3_1(pretrained=True)
    with pytest.raises(AssertionError):
        D.DarkNetV6(0.33, 0.5, version="r3.1")
    with pytest.raises(AssertionError):
        D.DarkNetV4(0.33, 0.5, version="r6.0")
    assert isinstance(D.darknet_s_r3_1().features[2], darknetv4.BottleneckCSP)
    m = D.DarkNetV6(0.33, 0.25, num_classes=7, stages_repeats=[1, 1, 1], stages_out_channels=[64, 128, 256],
                    last_channel=512)
    assert m.classifier[3].out_features == 7 and m.classifier[0].in_features == 128
    assert isinstance(m.avgpool, nn.AdaptiveAvgPool2d)


def test_forward_errors_before_any_launch():
    m = D.darknet_n_r6_0().eval()
    with pytest.raises(ValueError, match="multiple of 32"):
        m(torch.zeros(1, 3, 100, 96))
    with pytest.raises(ValueError, match=r"\[N,3,H,W\]"):
        m(torch.zeros(1, 4, 64, 64))
    with pytest.raises(NotImplementedError, match="training"):
        m.train()(torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError, match="plan"):
        D.darknet_n_r6_0().features[1](torch.zeros(1, 16, 8, 8))


def _lower(model, dtype=torch.float16):
    from yolort_b200.engine import lower_darknet

    return lower_darknet(model, dtype, torch.device("cpu"))


@pytest.mark.parametrize("arch,nc", [("darknet_n_r6_0", 1000), ("darknet_s_r4_0", 10), ("darknet_s_r3_1", 1003)])
def test_lowering_darknet_topology(arch, nc):
    from yolort_b200.engine import GLOBAL

    m = getattr(D, arch)(num_classes=nc).eval()
    L, x0, heads, feats = _lower(m)
    C = m.classifier[0].in_features
    tail = L.ops[-3:]
    assert [op.name for op in tail] == ["avgpool", "classifier.0", "classifier.3"]
    assert [op.kind for op in tail] == [_C.YB_OP_AVGPOOL, _C.YB_OP_CONV, _C.YB_OP_CONV]
    assert [op.act for op in tail] == [_C.YB_ACT_NONE, _C.YB_ACT_HARDSWISH, _C.YB_ACT_NONE]
    pool, fc1, fc2 = tail
    assert pool.src.buf is feats["features"].buf and pool.src.buf.div == 32 and pool.src.C == C
    assert pool.dst.buf is feats["avgpool"].buf and pool.weight is None
    assert all(op.dst.buf.div == GLOBAL for op in tail) and fc1.src.buf is pool.dst.buf and fc2.src.buf is fc1.dst.buf
    assert heads == [fc2.dst.buf] and fc2.dst.C == -(-nc // 8) * 8
    assert (fc1.ksize, fc2.ksize) == (1, 1) and fc2.weight.shape[0] == -(-nc // 16) * 16
    assert not fc2.weight[nc:].any() and not fc2.bias[nc:].any()
    assert fc1.flops_per_pixel == 2 * C * C and fc2.flops_per_pixel == 2 * C * nc
    assert max(b.div for b in L.bufs) == 32       # the global buffers do not widen the canvas rule
    assert all(op.kind != _C.YB_OP_AVGPOOL for op in L.ops[:-3])
    assert all(op.name.startswith("features.") for op in L.ops[:-3])


@pytest.mark.parametrize("arch,upstream", [("darknet_s_r6_0", "r6.0"), ("darknet_s_r4_0", "r4.0"),
                                           ("darknet_s_r3_1", "r3.1")])
def test_features_lower_to_the_detection_body_bit_for_bit(arch, upstream):
    """A classifier's `features` loaded into yolov5s's body lowers to the same ops with the same packed weights."""
    from yolort_b200.engine import lower_yolo
    from yolort_b200.models import yolov5s

    cls = getattr(D, arch)().eval()
    cls.load_state_dict(_sd(arch))
    det = yolov5s(upstream_version=upstream).model.eval()
    det.backbone.body.load_state_dict(cls.features.state_dict())
    for dtype in (torch.float16, torch.bfloat16):
        Ld = lower_yolo(det, dtype, torch.device("cpu"))[0]
        Lc = _lower(cls, dtype)[0]
        body = [op for op in Ld.ops if op.name.startswith("body.")]
        feats = Lc.ops[:-3]
        assert len(body) == len(feats) > 20
        for a, b in zip(body, feats):
            assert a.name == "body." + b.name[len("features."):]
            assert (a.kind, a.ksize, a.stride, a.pad, a.act, a.pack, a.band) == \
                (b.kind, b.ksize, b.stride, b.pad, b.act, b.pack, b.band), a.name
            for t, u in ((a.weight, b.weight), (a.bias, b.bias)):
                assert (t is None) == (u is None)
                if t is not None:
                    assert t.dtype == u.dtype and torch.equal(t.view(torch.int16) if t.element_size() == 2 else t,
                                                              u.view(torch.int16) if u.element_size() == 2 else u), a.name


def test_custom_block_constructs_but_does_not_lower():
    class MyBlock(nn.Module):
        def __init__(self, c1, c2, n=1):
            super().__init__()
            self.conv = nn.Conv2d(c1, c2, 1)

    m = D.DarkNetV6(0.33, 0.25, block=MyBlock).eval()
    assert isinstance(m.features[2], MyBlock)
    with pytest.raises(NotImplementedError, match="features.2: no lowering for MyBlock"):
        _lower(m)


@pytest.mark.parametrize("arch", NETWORK_ARCHS)
def test_oracle_network_darknet(arch):
    z = util.load_npz("network_darknet.npz")
    sd = _sd(arch, int(z[f"{arch}_seed"]))
    assert util.checksum(sd) == pytest.approx(float(z[f"{arch}_checksum"]), rel=1e-12)
    net = NetDarknet(sd)
    for i in range(len(INPUTS)):
        x = network_input(i)
        assert float(x.double().sum()) == pytest.approx(float(z[f"{arch}_{i}_x_checksum"]), rel=1e-12)
        with torch.no_grad():
            f, logits = net.forward(x)
        np.testing.assert_allclose(stored_features(f), z[f"{arch}_{i}_features"], atol=1e-4, rtol=1e-5)
        np.testing.assert_allclose(logits.numpy(), z[f"{arch}_{i}_logits"], atol=1e-4, rtol=1e-5)
        # the fixture's margins: top-1 clearly above the fp16 tolerance 1e-2 * max(1, |ref|)
        assert z[f"{arch}_{i}_top1_margin"].min() >= 0.05


def _desc(**kw):
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_AVGPOOL, _C.dtype_code(torch.float16)
    d.N, d.H, d.W, d.Ho, d.Wo = 4, 7, 7, 1, 1
    d.Cin, d.in_cstride, d.in_ = 512, 512, 4096
    d.Cout, d.out_cstride, d.out = 512, 512, 8192
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_avgpool_descriptor_accepted():
    """The descriptor the rejections below start from is valid (creating an AVGPOOL op makes no driver call)."""
    arr = (_C.OpDesc * 1)(_desc())
    h = ctypes.c_void_p()
    lib = _C.lib()
    assert lib.yb_plan_create(arr, 1, ctypes.byref(h)) == 0, lib.yb_last_error().decode()
    lib.yb_plan_destroy(h)


@pytest.mark.parametrize("field,value,msg", [
    ("Ho", 7, "1x1"),
    ("Wo", 2, "1x1"),
    ("Cout", 504, "must equal Cout"),
    ("Cin", 508, "must equal Cout"),
    ("in_cstride", 516, "multiples of 8"),
    ("out_cstride", 508, "multiples of 8"),
    ("in_", 4096 + 8, "16-byte aligned"),
    ("out", 8192 + 2, "16-byte aligned"),
    ("weight", 1 << 20, "must be NULL"),
    ("bias", 1 << 20, "must be NULL"),
    ("residual", 4096, "must be NULL"),
    ("chain", 4096, "must be NULL"),
    ("decode", 4096, "must be NULL"),
    ("act", _C.YB_ACT_SILU, "act must be 0"),
    ("reserved", 1, "reserved"),
    ("N", 0, "empty"),
    ("N", 70000, "too large"),
    ("dtype", _C.YB_F32, "dtype"),
])
def test_avgpool_descriptor_rejections(field, value, msg):
    """yb_plan_create validates an AVGPOOL op before any driver call: no GPU is needed to be refused."""
    d = _desc(**{field: value})
    if field == "Cin":
        d.Cout = 512
    arr = (_C.OpDesc * 1)(d)
    h = ctypes.c_void_p()
    lib = _C.lib()
    assert lib.yb_plan_create(arr, 1, ctypes.byref(h)) == -1 and not h.value
    err = lib.yb_last_error().decode()
    assert "avgpool" in err and msg in err, err
