"""yolov5_mobilenet_v3_small_fpn: MobileNetV3-Small + FPN on the native plan.  CPU: constructor surface, state-dict
layout and trainable flags, offline pretrained-backbone loading, lowering topology, the stem rewrite, the CPU oracle
against fixtures generated from the reference (oracle/make_golden_lite.py), the decode levels and the descriptor
validation of the depthwise and squeeze-excitation ops.  GPU: the plan launch by launch, against the fixtures, through
the callable sub-modules and under CUDA-graph replay."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parity_util as util
import stagewise as S
from oracle import restate_lite as RL
from oracle.make_golden_lite import (NUM_CLASSES, SCORE_THRESH, SIZE, e2e_input, network_input, stored_part,
                                     synth_state_dict_lite)
from yolort_b200 import _C
from yolort_b200.models.yolo_lite import (BackboneWithFPN, mobilenet_backbone, model_urls,
                                          yolov5_mobilenet_v3_small_fpn)

DEV = "cuda:0"
WEIGHTS_FILE = "mobilenet_v3_small-047dcff4.pth"


def _fixture():
    with open(os.path.join(util.GOLDEN, "state_dict_layouts_lite.json")) as f:
        return json.load(f)


def _sd():
    return synth_state_dict_lite(_fixture()["lite"])


def _new(**kw):
    return yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False, num_classes=NUM_CLASSES, **kw)


# ---- CPU -------------------------------------------------------------------------------------------------------
def test_state_dict_layout_equals_reference_lite():
    ref = _fixture()["lite"]
    sd = _new().state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    m = _new()
    m.load_state_dict(_sd(), strict=True)
    assert isinstance(m.backbone, BackboneWithFPN) and m.backbone.out_channels == 256


def test_requires_grad_sets_match_reference():
    ref = _fixture()["requires_grad"]
    for t in range(7):
        got = [n for n, p in mobilenet_backbone("mobilenet_v3_small", False, trainable_layers=t).named_parameters()
               if p.requires_grad]
        assert got == ref[str(t)], t
    assert len(ref["0"]) == 12 and len(ref["6"]) > len(ref["2"]) > len(ref["0"])   # only the FPN stays trainable at 0
    # without pretrained weights every stage stays trainable, whatever is asked (reference behaviour)
    with pytest.warns(UserWarning):
        m = _new(trainable_backbone_layers=1)
    assert all(p.requires_grad for p in m.parameters())


def test_constructor_errors_lite():
    from yolort_b200.models import yolo_lite

    assert yolo_lite.__all__ == ["yolov5_mobilenet_v3_small_fpn"]
    assert model_urls == {"yolov5_mobilenet_v3_small_fpn_coco": None}
    with pytest.raises(ValueError, match="No checkpoint is available"):
        yolov5_mobilenet_v3_small_fpn(pretrained=True)
    with pytest.raises(ValueError):
        mobilenet_backbone("mobilenet_v3_small", False, trainable_layers=7)
    with pytest.raises(ValueError):
        mobilenet_backbone("mobilenet_v3_small", False, returned_layers=[4, 6])
    with pytest.raises(RuntimeError, match="plan"):
        mobilenet_backbone("mobilenet_v3_small", False)(torch.zeros(1, 3, 64, 64))


def test_pretrained_backbone_reads_the_hub_cache_only(tmp_path, monkeypatch):
    import torchvision

    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    path = os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)
    assert path.startswith(str(tmp_path))
    with pytest.raises(ValueError, match=WEIGHTS_FILE) as e:
        yolov5_mobilenet_v3_small_fpn()
    assert "pretrained_backbone=False" in str(e.value)
    # a seeded fake of torchvision's ImageNet file (BatchNorm2d statistics included) loads exactly
    net = torchvision.models.mobilenet_v3_small(weights=None)
    g = torch.Generator().manual_seed(5)
    fake = {k: (torch.rand(v.shape, generator=g) + 0.5 if v.is_floating_point() else v)
            for k, v in net.state_dict().items()}
    os.makedirs(os.path.dirname(path))
    torch.save(fake, path)
    m = yolov5_mobilenet_v3_small_fpn(num_classes=NUM_CLASSES)
    got = m.backbone.body.state_dict()
    n = 0
    for k, v in got.items():
        assert torch.equal(v, fake[f"features.{k}"]), k
        n += 1
    assert n > 100
    # default trainable_backbone_layers = 3 with pretrained weights: layers 0..3 frozen
    frozen = {k.split(".")[2] for k, p in m.named_parameters() if not p.requires_grad}
    assert frozen == {"0", "1", "2", "3"}


def _lower(model=None, dtype=torch.float16):
    from yolort_b200.engine import lower_lite

    model = model or _new().eval()
    return lower_lite(model, dtype, torch.device("cpu"))


def test_lowering_lite_topology():
    L, x0, heads, feats = _lower()
    kinds = [op.kind for op in L.ops]
    assert len(L.ops) == 55
    assert kinds.count(_C.YB_OP_DWCONV) == 12 and kinds.count(_C.YB_OP_SE) == 9
    assert kinds.count(_C.YB_OP_UPSAMPLE2X) == 1 and kinds.count(_C.YB_OP_CONV) == 33
    res = [op for op in L.ops if op.residual is not None]
    assert len(res) == 8 and all(op.kind == _C.YB_OP_CONV for op in res)
    written = set()
    for op in L.ops:
        for v in (op.src, op.residual):
            if v is None:
                continue
            for c in range(v.ch0, v.ch0 + v.C):
                assert (v.buf.name, c) in written or v.buf is x0, f"{op.name} reads an unwritten channel"
        written.update((op.dst.buf.name, c) for c in range(op.dst.ch0, op.dst.ch0 + op.dst.C))
    ops = {op.name: op for op in L.ops}
    # residual projections read the block input: blocks 3, 5, 6, 8, 10, 11 (InvertedResidual.use_res_connect)
    proj = {op.name.split(".")[1]: op for op in res if op.name.startswith("body.")}
    assert sorted(proj, key=int) == ["3", "5", "6", "8", "10", "11"]
    for i, op in proj.items():
        assert op.residual.buf.name == f"body.{int(i) - 1}" and op.dst.buf.name == f"body.{i}" and op.act == 0
    assert ops["fpn.inner_blocks.1"].residual.buf is ops["fpn.inner_blocks.2"].dst.buf
    up = ops["fpn.interpolate0"]
    assert up.src.buf is ops["fpn.inner_blocks.1"].dst.buf and ops["fpn.inner_blocks.0"].residual.buf is up.dst.buf
    pool = ops["fpn.extra_blocks(max_pool2d k1 s2)"]
    assert (pool.kind, pool.ksize, pool.stride, pool.pad) == (_C.YB_OP_DWCONV, 1, 2, 0)
    assert pool.src.buf is feats["2"].buf and pool.dst.buf is feats["pool"].buf
    assert torch.equal(pool.weight.float(), torch.ones(1, 256)) and not pool.bias.any()
    # every fact read from the modules: SE squeeze widths, depthwise kernels and strides, activations
    se = [op.ksize for op in L.ops if op.kind == _C.YB_OP_SE]
    assert se == [8, 24, 64, 64, 32, 40, 72, 144, 144]
    dw = [(op.ksize, op.stride, op.act) for op in L.ops if op.kind == _C.YB_OP_DWCONV][:11]
    R, H = _C.YB_ACT_RELU, _C.YB_ACT_HARDSWISH
    assert dw == [(3, 2, R), (3, 2, R), (3, 1, R)] + [(5, 2, H)] + [(5, 1, H)] * 4 + [(5, 2, H)] + [(5, 1, H)] * 2
    assert [feats[k].buf.div for k in ("0", "1", "2", "pool")] == [16, 32, 32, 64]
    assert all(op.flops_per_pixel == 2 * op.ksize ** 2 * op.src.C for op in L.ops if op.kind == _C.YB_OP_DWCONV)
    assert max(b.div for b in L.bufs) == 64      # the canvas must be a multiple of 64


def test_stem_rewrite_exact_fp64():
    from yolort_b200.engine import stem_s2_to_s2d

    g = torch.Generator().manual_seed(3)
    w = torch.randn(16, 3, 3, 3, generator=g, dtype=torch.float64)
    x = torch.randn(2, 3, 24, 40, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, None, 2, 1)
    n, _, h, wd = x.shape
    s2d = torch.zeros(n, 16, h // 2, wd // 2, dtype=torch.float64)
    for dy in range(2):
        for dx in range(2):
            q = (dy * 2 + dx) * 4
            s2d[:, q:q + 3] = x[:, :, dy::2, dx::2]
    got = F.conv2d(s2d, stem_s2_to_s2d(w), None, 1, 1)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-12)


def test_oracle_network_lite():
    z = util.load_npz("network_lite.npz")
    sd = _sd()
    assert util.checksum(sd) == pytest.approx(float(z["checksum"]), rel=1e-12)
    x = network_input()
    assert float(x.double().sum()) == pytest.approx(float(z["x_checksum"]), rel=1e-12)
    net = RL.NetLite(sd)
    with torch.no_grad():
        feats = net.backbone(x)
        heads = net.head(feats)
    for i, got in enumerate(feats):
        np.testing.assert_allclose(stored_part(f"f{i}", got), z[f"f{i}"], atol=1e-4, rtol=1e-5)
    for i, got in enumerate(heads):
        np.testing.assert_allclose(stored_part(f"h{i}", got), z[f"h{i}"], atol=1e-4, rtol=1e-5)
    dets = RL.postprocess(heads, SCORE_THRESH)
    ref = util.dets_from_npz(z, 1)[0]
    assert 20 <= len(ref["scores"]) < 300
    assert util.match_fraction(util.to_np(dets[0]), ref, iou_thr=0.99) >= 0.97
    # non-vacuity: the SE gates are neither constant nor saturated
    g = torch.cat([t.reshape(-1) for t in net.se_gates])
    inside = float(((g > 0.05) & (g < 0.95)).double().mean())
    assert inside == pytest.approx(float(z["se_inside"]), abs=1e-3) and 0.5 < inside < 0.95


def test_oracle_end_to_end_lite():
    z = util.load_npz("e2e_lite.npz")
    x = e2e_input()
    assert float(x.double().sum()) == pytest.approx(float(z["x_checksum"]), rel=1e-12)
    dets = RL.detect(_sd(), x, SCORE_THRESH)
    for got, ref in zip(dets, util.dets_from_npz(z, 2)):
        assert len(ref["scores"]) > 20
        assert util.match_fraction(util.to_np(got), ref, iou_thr=0.99) >= 0.97


def test_decode_levels_at_320():
    """The heads sit at strides 16, 32, 32, 64 and are decoded with 8, 16, 32, 64 (reference behaviour)."""
    m = _new().eval()
    _, _, head_bufs, _ = _lower(m)
    got = [(320 // b.div, 320 // b.div, s) for b, s in zip(head_bufs, m.post_config()["strides"])]
    assert got == [(20, 20, 8), (10, 10, 16), (10, 10, 32), (5, 5, 64)]
    with torch.no_grad():
        heads = RL.NetLite(_sd()).head(RL.NetLite(_sd()).backbone(network_input()))
    assert RL.level_shapes(heads) == got


def _desc(kind, **kw):
    d = _C.OpDesc()
    d.kind, d.dtype = kind, _C.dtype_code(torch.float16)
    d.N, d.H, d.W, d.Ho, d.Wo = 2, 20, 20, 10, 10
    d.Cin, d.in_cstride, d.in_ = 96, 96, 4096
    d.Cout, d.out_cstride, d.out = 96, 96, 8192
    d.ksize, d.stride, d.pad, d.act = 5, 2, 2, _C.YB_ACT_HARDSWISH
    d.weight, d.bias = 1 << 20, 1 << 21
    if kind == _C.YB_OP_SE:
        d.Ho, d.Wo, d.out, d.ksize, d.stride, d.pad, d.act = 20, 20, 4096, 24, 1, 0, 0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _reject(d, who, msg):
    arr = (_C.OpDesc * 1)(d)
    h = ctypes.c_void_p()
    lib = _C.lib()
    rc = lib.yb_plan_create(arr, 1, ctypes.byref(h))
    assert rc == -1 and not h.value
    err = lib.yb_last_error().decode()
    assert who in err and msg in err, err


@pytest.mark.parametrize("field,value,msg", [
    ("ksize", 7, "ksize must be 1, 3 or 5"),
    ("ksize", 3, "pad must be ksize/2"),
    ("stride", 3, "stride must be 1 or 2"),
    ("pad", 1, "pad must be ksize/2"),
    ("act", _C.YB_ACT_SILU, "act must be"),
    ("Cout", 88, "must equal Cout"),
    ("Cin", 92, "must equal Cout"),
    ("in_cstride", 100, "multiples of 8"),
    ("Ho", 20, "output extent"),
    ("in_", 4096 + 8, "16-byte aligned"),
    ("weight", (1 << 20) + 2, "16-byte aligned"),
    ("weight", 0, "null weight"),
    ("bias", 0, "null weight"),
    ("reserved", 2, "reserved"),
    ("residual", 4096, "must be NULL"),
    ("chain", 4096, "must be NULL"),
    ("decode", 4096, "must be NULL"),
    ("dtype", _C.YB_F32, "dtype"),
])
def test_dwconv_descriptor_rejections(field, value, msg):
    """yb_plan_create validates a depthwise op before any driver call: no GPU is needed to be refused."""
    d = _desc(_C.YB_OP_DWCONV, **{field: value})
    if field == "Cin":
        d.Cout = 96
    _reject(d, "dwconv", msg)


@pytest.mark.parametrize("field,value,msg", [
    ("out", 8192, "in place"),
    ("out_cstride", 104, "in place"),
    ("Cout", 88, "must equal Cout"),
    ("Cin", 92, "must equal Cout"),
    ("Cin", 2056, "multiple of 8 up to"),
    ("ksize", 0, "squeeze width"),
    ("ksize", 1025, "squeeze width"),
    ("Ho", 10, "output extent"),
    ("in_", 4096 + 8, "16-byte aligned"),
    ("weight", 0, "null weight"),
    ("bias", (1 << 21) + 4, "16-byte aligned"),
    ("reserved", 1, "reserved"),
    ("residual", 4096, "must be NULL"),
    ("chain", 4096, "must be NULL"),
    ("decode", 4096, "must be NULL"),
])
def test_se_descriptor_rejections(field, value, msg):
    d = _desc(_C.YB_OP_SE, **{field: value})
    if field == "in_":
        d.out = d.in_
    if field == "Cin":
        d.Cout = value if value == 2056 else 96
    _reject(d, "se", msg)


# ---- GPU -------------------------------------------------------------------------------------------------------
def _model():
    m = yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False, num_classes=NUM_CLASSES,
                                      score_thresh=SCORE_THRESH).eval()
    m.load_state_dict(_sd())
    return m.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("N,hw,dtype", [(32, 640, torch.float16), (8, 1280, torch.bfloat16)])
def test_gpu_stagewise_lite(N, hw, dtype):
    from yolort_b200.engine import Engine

    m = _model()
    eng = Engine(m, dtype, torch.device(DEV))
    plan = eng.plan(N, hw, hw, keep_intermediates=True)
    g = torch.Generator(device=DEV).manual_seed(3)
    plan.input.copy_(torch.rand(plan.input.shape, generator=g, device=DEV).to(dtype))
    plan.input[..., 3::4] = 0
    res = S.check_plan_stagewise(plan, m.backbone.body["0"])
    assert len(res) == len(plan._low.L.ops) == 55
    bad = [r for r in res if r.violations]
    assert not bad, bad


@pytest.mark.gpu
def test_gpu_heads_vs_reference_fixture_lite():
    z = util.load_npz("network_lite.npz")
    m = _model()
    x = network_input().to(DEV)
    dets = m(x)
    plan = m.get_plan(1, *SIZE)
    m.run_plan(plan)
    torch.cuda.synchronize()
    for i, key in enumerate(("0", "1", "2", "pool")):
        got = plan.features[key].float().permute(0, 3, 1, 2).cpu().numpy()
        rr = util.rel_rms(stored_part(f"f{i}", got), z[f"f{i}"])
        rh = util.rel_rms(stored_part(f"h{i}", util.head_logits(plan, i)), z[f"h{i}"])
        print(f"lite f{i} rel_rms {rr:.2e}  h{i} rel_rms {rh:.2e}")
        assert rr < 2e-2 and rh < 2e-2
    frac = util.match_fraction(util.to_np(dets[0]), util.dets_from_npz(z, 1)[0], iou_thr=0.9)
    print("lite network dets matched:", frac)
    assert frac >= 0.97


@pytest.mark.gpu
def test_gpu_end_to_end_vs_reference_fixture_lite():
    z = util.load_npz("e2e_lite.npz")
    m = _model()
    out = m(e2e_input().to(DEV))
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.9)
        print("lite e2e:", len(got["scores"]), len(ref["scores"]), "matched:", frac)
        assert frac >= 0.95


@pytest.mark.gpu
def test_gpu_submodules_with_hooks_match_the_plan_lite():
    m = _model()
    x = e2e_input().to(DEV)
    plain = m(x)
    seen = []
    hooks = [m.backbone.register_forward_hook(lambda mod, i, o: seen.append([t.shape for t in o])),
             m.head.register_forward_hook(lambda mod, i, o: seen.append([t.shape for t in o]))]
    hooked = m(x)
    for h in hooks:
        h.remove()
    assert seen[0] == [torch.Size([2, 256, 16, 24]), torch.Size([2, 256, 8, 12]), torch.Size([2, 256, 8, 12]),
                       torch.Size([2, 256, 4, 6])]
    assert seen[1][0] == torch.Size([2, 3, 16, 24, 85]) and seen[1][3] == torch.Size([2, 3, 4, 6, 85])
    feats = m.backbone(x)
    heads = m.head(feats)
    plan = m.get_plan(2, 256, 384)
    for i, hb in enumerate(plan.heads):
        n, h, w, _ = hb.shape
        assert torch.equal(heads[i], hb[..., :255].view(n, h, w, 3, 85).permute(0, 3, 1, 2, 4))
    for a, b in zip(plain, hooked):
        for k in ("scores", "labels", "boxes"):
            assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
def test_gpu_graph_replay_and_repeat_are_bit_identical_lite():
    from yolort_b200.engine import Engine

    m = _model()
    eng = Engine(m, torch.float16, torch.device(DEV))
    plan = eng.plan(8, 640, 448)
    g = torch.Generator(device=DEV).manual_seed(4)
    plan.input.copy_(torch.rand(plan.input.shape, generator=g, device=DEV).half())
    plan.input[..., 3::4] = 0
    util.assert_repeat_and_graph_replay_bit_identical(plan)
