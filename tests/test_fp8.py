"""FP8 (e4m3) lowering, calibration objects and descriptor validation, without a GPU."""
import ctypes
import hashlib
import os
import sys

import pytest
import torch

from yolort_b200 import _C, engine
from yolort_b200.engine import lower_fp8, lower_yolo, scale_groups

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CPU = torch.device("cpu")


def _model(ctor, version="r6.0"):
    import bench
    from yolort_b200 import models

    m = getattr(models, ctor)(upstream_version=version).eval()
    m.load_state_dict(bench.make_state_dict(m))
    return m


def _amax(L):
    """A synthetic calibration: a different max|x| for every buffer."""
    return {b.name: 0.75 + 0.37 * i for i, b in enumerate(L.bufs)}


FP8_MODELS = [("yolov5s", "r6.0"), ("yolov5n6", "r6.0"), ("yolov5s", "r4.0"), ("yolov5s", "r3.1")]


@pytest.mark.parametrize("ctor,version", FP8_MODELS)
def test_scale_groups_merge_exactly_the_copies(ctor, version):
    """Every SPP and upsample shares its source's scale group (concat windows are one buffer, hence one group), and no
    other buffers are merged: the groups are the connected components of the SPP / upsample edges."""
    L = lower_yolo(_model(ctor, version).model, torch.float16, CPU, fp8=True)[0]
    groups = scale_groups(L)
    group_of = {id(b): i for i, g in enumerate(groups) for b in g}
    assert sorted(id(b) for g in groups for b in g) == sorted(id(b) for b in L.bufs)
    edges = [(op.src.buf, op.dst.buf) for op in L.ops if op.kind in (_C.YB_OP_SPP_POOL, _C.YB_OP_UPSAMPLE2X)]
    assert len(edges) >= 3
    for a, b in edges:
        assert group_of[id(a)] == group_of[id(b)]
    comp = {id(b): id(b) for b in L.bufs}

    def find(k):
        while comp[k] != k:
            k = comp[k]
        return k

    for a, b in edges:
        comp[find(id(a))] = find(id(b))
    for g in groups:
        assert len({find(id(b)) for b in g}) == 1
    assert len(groups) == len({find(id(b)) for b in L.bufs})
    merged = [g for g in groups if len(g) > 1]
    assert merged and all(b.name.startswith("pan.") for g in merged for b in g), [[b.name for b in g] for g in merged]


def _view(v):
    return None if v is None else (v.buf.name, v.ch0, v.C)


@pytest.mark.parametrize("ctor,version", FP8_MODELS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fp8_op_list_is_the_fp16_list_plus_one_quantize(ctor, version, dtype):
    m = _model(ctor, version).model
    L16, x0_16, heads16, feats16 = lower_yolo(m, dtype, CPU)
    L8, x0, heads, feats, scale = lower_fp8(m, dtype, CPU, _amax(L16))
    qi = [i for i, op in enumerate(L8.ops) if op.kind == _C.YB_OP_QUANTIZE]
    assert qi == [1], qi
    q = L8.ops[1]
    stem_out = L16.ops[0].dst
    assert _view(q.src) == _view(stem_out) and q.dst.C == stem_out.C and q.dst.buf.esz == 1
    assert q.dtype is None and q.bias.dtype == torch.float32 and float(q.bias[0]) == 1.0 / scale[id(q.dst.buf)]
    ops8 = [L8.ops[0]] + L8.ops[2:]
    assert len(ops8) == len(L16.ops)

    def remap(v):      # the fp16 list reads the stem output where the FP8 list reads its e4m3 copy
        return _view(q.src) if v is not None and _view(v) == _view(q.dst) else _view(v)

    head_names = {b.name for b in heads}
    for a, b in zip(L16.ops, ops8):
        assert (a.name, a.kind, a.ksize, a.stride, a.pad, a.act, a.pack) == (b.name, b.kind, b.ksize, b.stride, b.pad,
                                                                              b.act, b.pack)
        assert (_view(a.src), _view(a.dst), _view(a.residual)) == (remap(b.src), remap(b.dst), remap(b.residual)), a.name
        if b is L8.ops[0]:
            assert b.dtype is None and torch.equal(a.weight, b.weight) and torch.equal(a.bias, b.bias)   # the stem
            continue
        assert b.dtype == _C.YB_F8E4M3, b.name
        if b.kind != _C.YB_OP_CONV:
            continue
        co = a.dst.C if a.dst.buf.name not in head_names else None
        co_pad, taps, ci_pad = b.weight.shape
        assert b.weight.dtype == torch.float8_e4m3fn and co_pad == a.weight.shape[0] and taps == a.weight.shape[1]
        assert ci_pad % 32 == 0 and (ci_pad % 128 == 0 or ci_pad <= 64) and ci_pad >= a.src.C
        assert b.bias.dtype == torch.float32 and b.bias.shape == (2 * co_pad + 2,)
        n = a.bias.shape[0]
        assert torch.equal(b.bias[:n], a.bias), b.name                                    # the same fp32 bias
        mul = b.bias[co_pad:2 * co_pad]
        live = mul[mul != 0]
        assert torch.equal(torch.exp2(torch.round(torch.log2(live))), live)               # powers of two
        head = b.dst.buf.name in head_names
        assert b.reserved == ((32 if dtype == torch.bfloat16 else 16) if head else 0)
        s_in = scale[id(b.src.buf)]
        s_out = 1.0 if head else scale[id(b.dst.buf)]
        assert float(b.bias[2 * co_pad + 1]) == 1.0 / s_out
        assert float(b.bias[2 * co_pad]) == (scale[id(b.residual.buf)] if b.residual is not None else 0.0)
        assert torch.all((mul / s_in)[: co or n].ne(0)) or head
        # the multipliers are s_w * s_in for the s_w the weights were divided by: dequantised with m / s_in, the e4m3
        # weights are one rounding of the folded weights (here their fp16 / bf16 packing), and s_w is the smallest
        # power of two that brings each channel's max|w| within 448
        co_w = int(torch.count_nonzero(mul))
        s_w = (mul[:co_w] / s_in).double()
        wq = b.weight[:co_w].double()
        ref = a.weight[:co_w].double()
        deq = wq * s_w.view(-1, 1, 1)
        ci = a.src.C
        ulp = torch.exp2(torch.clamp(torch.frexp((ref / s_w.view(-1, 1, 1)).abs())[1] - 4, min=-9).double())
        tol16 = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
        err = (deq[..., :ci] - ref[..., :ci]).abs()
        assert torch.all(err <= (0.5 * ulp[..., :ci] * (1 + tol16) + tol16 * ref[..., :ci].abs()) * s_w.view(-1, 1, 1)
                         * (1 + 1e-12) + 1e-30), b.name
        assert torch.count_nonzero(wq[..., ci:]) == 0
        amax_q = wq.abs().flatten(1).amax(1)
        assert torch.all(amax_q <= 448) and torch.all(amax_q >= 224 * (1 - 4 * tol16)), b.name
    esz = {b.name: b.esz for b in L8.bufs}
    assert esz[x0.name] == 2 and esz[stem_out.buf.name] == 2 and all(esz[b.name] == 2 for b in heads)
    assert sum(1 for v in esz.values() if v == 1) == len(L8.bufs) - 2 - len(heads)


def test_e4m3_weights_are_one_rounding_of_the_folded_weights():
    w = torch.tensor([[[[0.0, 1.0 / 1024, -300.0, 449.0]]], [[[2.0 ** -12, 17.0, 0.1, -0.2]]]], dtype=torch.float64)
    s_w = torch.tensor([1.0, 2.0 ** -4], dtype=torch.float64)
    q = engine.pack_weight_e4m3(w, s_w, CPU)
    assert q.shape == (16, 4, 32)
    got = q[:2, :, 0].double()
    exact = (w / s_w.view(-1, 1, 1, 1)).view(2, 4)
    assert float(got[0, 3]) == 448.0 and float(got[0, 2]) == -288.0     # saturation; spacing 32 above 256
    fin = exact.abs() <= 448
    assert torch.equal(got[fin], torch.tensor(torch.clamp(exact, -448, 448)[fin].tolist()).double().to(torch.float32)
                       .to(torch.float8_e4m3fn).double())
    assert torch.count_nonzero(q[2:].float()) == 0 and torch.count_nonzero(q[:, :, 1:].float()) == 0


def test_pack_weight_e4m3_keeps_the_tap_order_of_an_asymmetric_kernel():
    g = torch.Generator().manual_seed(5)
    w = torch.randn(24, 40, 3, 3, generator=g, dtype=torch.float64)
    w[:, :, 0, 2] *= 8.0                       # an asymmetric kernel: a transposed kh / kw would move these taps
    s_w = engine.e4m3_scales(w.abs().amax(dim=(1, 2, 3)))
    q = engine.pack_weight_e4m3(w, s_w, CPU)
    assert q.shape == (32, 9, 64)
    for co in (0, 7, 23):
        for kh in range(3):
            for kw in range(3):
                for ci in (0, 13, 39):
                    exact = float(w[co, ci, kh, kw] / s_w[co])
                    got = float(q[co, kh * 3 + kw, ci].float())
                    ulp = 2.0 ** max(__import__("math").frexp(abs(exact))[1] - 4, -9)
                    assert abs(got - exact) <= 0.5 * ulp, (co, kh, kw, ci)


def test_e4m3_scales_match_e4m3_scale():
    a = torch.cat([torch.tensor([0.0, 448.0, 448.0 * 2 ** -5, 1e-30, 7e4]),
                   torch.rand(200, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 1e3])
    assert engine.e4m3_scales(a).tolist() == [engine.e4m3_scale(v) for v in a.tolist()]


def test_e4m3_scale_is_the_smallest_power_of_two():
    for a in (448.0, 448.0001, 1.0, 3e-5, 7e4, 0.0):
        s = engine.e4m3_scale(a)
        assert s > 0 and 2.0 ** round(__import__("math").log2(s)) == s
        assert a / s <= 448.0 and (a == 0.0 or a / (s / 2) > 448.0)


# the parent commit's fp16 / bf16 lowerings (buffers, ops, packed weights and biases) of the bench-seeded weights
PARENT_DIGESTS = {
    ("yolov5n", "r6.0", "float16"): "9fb2f95364e5d604c4ebd17622d4ccfc14acb17b4ba10981388f4cb892c7bf62",
    ("yolov5s", "r6.0", "float16"): "9440abb91366be2d1de3313b74b4ebc5265d1e872c0863cf4a80f63852389b94",
    ("yolov5m", "r6.0", "float16"): "e2a35e1ca714a02e515bf05bd290f408ef88cafda12cafe7958b92443204214f",
    ("yolov5l", "r6.0", "float16"): "4e23d5ae28d723d0a99a8eb75a075dcd0bbe06cdd7750b48a04a2a48e992ca6c",
    ("yolov5x", "r6.0", "float16"): "b0a321b523c398b58911cf20701b20fbd79d710a3a41ee2d1a0e367543fc5088",
    ("yolov5n6", "r6.0", "float16"): "f6e1c9a79feff078c8c9be6c522e616b626b5061db3dc1b79c9d2b6255a1b6c5",
    ("yolov5s6", "r6.0", "float16"): "164ed1b80b6bd283f0e685f9572afaddc242e00c3299d43af452c996f87fb906",
    ("yolov5m6", "r6.0", "float16"): "4dc6c38ac8ecb03edb5d2336a5dc690524e27ebb8bbf6582facdca1083316b8d",
    ("yolov5s", "r4.0", "float16"): "1d3c0b7382fb2e3b7bd8dc94ee98ef2b7d147603c484ce1de2e2efd5e3f8bfa1",
    ("yolov5m", "r4.0", "float16"): "9530d4cb0d52c0f86395b2913d0c620b1e84664b5063847c0cd64e39da6e80cb",
    ("yolov5l", "r4.0", "float16"): "17f112b1316fc550045039b08fcd143c8ca2489a62fcb7c3d8d559876c461404",
    ("yolov5s", "r3.1", "float16"): "bcea88bb7108e596bccd01157be14bea07477787247467b067ba462626107058",
    ("yolov5m", "r3.1", "float16"): "e9a1c2a541035727bf71e8df05fd08f351fed6b20e7cc0e7c5eb616d87209243",
    ("yolov5l", "r3.1", "float16"): "a2be51df94737c2cc5fa70c6ed50e03681690398285a763db3e32b7623854eb2",
    ("yolov5n", "r6.0", "bfloat16"): "6d8669d45956373e6b87ac65bb5e98b82f1969932237152d4c24f3adfa2285a5",
    ("yolov5s", "r6.0", "bfloat16"): "f085110f066a18302fbb8a70377167fa3972d9f40e3eca9fea805c379d95a362",
    ("yolov5m", "r6.0", "bfloat16"): "e1e3ae946f925ddf6aa00be343d1907fbf9d4d00a4a43eaab7ffa9cff84c45fc",
    ("yolov5l", "r6.0", "bfloat16"): "f239de611718ae3bc01b79d78a47fc1965e5d9c3ece99c9cfee0cbe26f4f05c7",
    ("yolov5x", "r6.0", "bfloat16"): "b9a718f0173e4c6e533ec4a861ddffb31a89e088d89ed6af7f7dd7e070546fe2",
    ("yolov5n6", "r6.0", "bfloat16"): "411b71bee7499199700f20e85771489a87d7fb29f185c227930027503f89fd4e",
    ("yolov5s6", "r6.0", "bfloat16"): "e9ebecea534988ae750df0722a648b640453b4c9353522e75133497f262ba52b",
    ("yolov5m6", "r6.0", "bfloat16"): "35308689622323d7ef13affd8fab013b323bedad2dc584b9876bd8dd964d1b0b",
    ("yolov5s", "r4.0", "bfloat16"): "ccd2311b4fbaab70b14ffed513f9f60cbd91d45746197164909f9f46f9c426a0",
    ("yolov5m", "r4.0", "bfloat16"): "1b3624af0c2573d7a50b341d4524c23dd1c4f2f2d59ab0ec02f20af24ead54a6",
    ("yolov5l", "r4.0", "bfloat16"): "514f15c11c7119627d38b35d4a17025749e6642528af81ae2ed9e5e03ef69d86",
    ("yolov5s", "r3.1", "bfloat16"): "7338011ccece5f9950d090cbe037aedf2a65fc8bbec1c90e38a2ab5f8841f05b",
    ("yolov5m", "r3.1", "bfloat16"): "1c1d6423ab560d7660cb29754da8fa7f60d630b587347abd42adf789050fe02a",
    ("yolov5l", "r3.1", "bfloat16"): "2bbe1a5c9478ea261af5c3ebe46d28952e29ee4f71a76cfc24d6a46f5d49f471",
}


def _digest(L, x0, heads, feats):
    h = hashlib.sha256()
    for b in L.bufs:
        h.update(repr((b.name, b.div, b.C)).encode())
    for op in L.ops:
        h.update(repr((op.name, op.kind, _view(op.src), _view(op.dst), op.ksize, op.stride, op.pad, op.act,
                       _view(op.residual), op.flops_per_pixel, op.pack, op.force_im2col, op.band, op.chain_own,
                       _view(op.chain_extra), op.chain_store)).encode())
        for t in (op.weight, op.bias):
            if t is not None:
                h.update(repr((tuple(t.shape), str(t.dtype))).encode())
                h.update(t.contiguous().view(torch.uint8).numpy().tobytes())
    h.update(repr((x0.name, [b.name for b in heads], sorted((k, f.buf.name) for k, f in feats.items()))).encode())
    return h.hexdigest()


@pytest.mark.parametrize("key", sorted(PARENT_DIGESTS))
def test_fp16_lowering_unchanged(key):
    ctor, version, dt = key
    m = _model(ctor, version)
    assert _digest(*lower_yolo(m.model, getattr(torch, dt), CPU)) == PARENT_DIGESTS[key]


def test_calibration_state_dict_round_trip_and_model_state_dict_unchanged():
    from yolort_b200.quantization import Fp8Calibration, arch_fingerprint

    m = _model("yolov5n")
    keys = list(m.state_dict())
    c = Fp8Calibration({"a": 1.5, "b": 0.0}, arch_fingerprint(m.model))
    c2 = Fp8Calibration({}, "")
    c2.load_state_dict(c.state_dict())
    assert c2.amax == c.amax and c2.fingerprint == c.fingerprint
    import io

    buf = io.BytesIO()
    torch.save(c.state_dict(), buf)
    buf.seek(0)
    c3 = Fp8Calibration({}, "")
    c3.load_state_dict(torch.load(buf))
    assert c3.state_dict() == c.state_dict()
    m.set_fp8(c)
    assert m.precision == "fp8" and list(m.state_dict()) == keys
    m.set_fp8(None)
    assert m.precision == "fp16"
    with pytest.raises(ValueError):
        _model("yolov5s").set_fp8(c)      # another architecture


def test_models_without_fp8_plans_raise():
    from yolort_b200 import models
    from yolort_b200.models import darknetv6, yolo_lite
    from yolort_b200.quantization import Fp8Calibration, calibrate_fp8

    c = Fp8Calibration({}, "")
    ts = models.yolov5ts()
    with pytest.raises(NotImplementedError, match="yolov5ts"):
        ts.set_fp8(c)
    lite = yolo_lite.yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False)
    with pytest.raises(NotImplementedError, match="mobilenet"):
        lite.set_fp8(c)
    with pytest.raises(NotImplementedError, match="DarkNet"):
        calibrate_fp8(darknetv6.darknet_s_r6_0(), [torch.zeros(1, 3, 64, 64)])
    with pytest.raises(NotImplementedError):
        calibrate_fp8(ts, [[torch.zeros(3, 64, 64)]])


# ---------------------------------------------------------------------------------------------------------------------
# yb_plan_create refuses bad e4m3 descriptors before any driver call
# ---------------------------------------------------------------------------------------------------------------------
def _conv_desc(**kw):
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_CONV, _C.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = 2, 20, 20, 64, 128, 4096
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = 20, 20, 64, 64, 8192
    d.ksize, d.stride, d.pad, d.act = 3, 1, 1, _C.YB_ACT_SILU
    d.weight, d.Cin_pad, d.Cout_pad, d.bias = 16384, 64, 64, 32768
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _refuse(d, msg):
    arr = (_C.OpDesc * 1)(d)
    h = ctypes.c_void_p()
    lib = _C.lib()
    assert lib.yb_plan_create(arr, 1, ctypes.byref(h)) == -1 and not h.value
    err = lib.yb_last_error().decode()
    assert msg in err, err


def test_valid_e4m3_conv_config():
    cfg = _C.conv_config(_conv_desc())
    assert cfg["e4m3_kernel"] == 1 and cfg["patch_kernel"] == 0 and cfg["block_n"] == 64
    assert not _C.conv_chain_supported(_conv_desc())


@pytest.mark.parametrize("field,value,msg", [
    ("in_", 4096 + 8, "16-byte aligned"),
    ("out", 8192 + 4, "16-byte aligned"),
    ("Cin", 56, "multiples of 16"),
    ("in_cstride", 120, "multiples of 16"),
    ("out_cstride", 72, "multiples of 16"),
    ("Cin_pad", 48, "Cin_pad"),
    ("ksize", 5, "3x3/s1/p1"),
    ("pad", 0, "3x3/s1/p1"),
    ("act", 9, "activation"),
    ("reserved", 1, "reserved"),
    ("reserved", 2, "reserved"),
    ("reserved", 48, "reserved"),
    ("decode", 4096, "fused decode"),
    ("chain", 4096, "chained tail"),
    ("Ho", 19, "extent"),
])
def test_plan_create_rejects_bad_e4m3_conv(field, value, msg):
    _refuse(_conv_desc(**{field: value}), msg)


def test_plan_create_rejects_residual_with_wide_output():
    _refuse(_conv_desc(reserved=16, residual=12288, res_cstride=64), "residual")
    _refuse(_conv_desc(residual=12288 + 8, res_cstride=64), "residual")


def _q_desc(**kw):
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_QUANTIZE, _C.YB_F16
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = 2, 20, 20, 32, 32, 4096
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = 20, 20, 32, 32, 8192
    d.bias = 32768
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("field,value,msg", [
    ("dtype", _C.YB_F8E4M3, "source type"),
    ("Cout", 48, "Cin == Cout"),
    ("Cin", 24, "Cin == Cout"),
    ("out_cstride", 40, "multiple of 8, out_cstride of 16"),
    ("in_", 4096 + 2, "16-byte aligned"),
    ("bias", 0, "bias"),
    ("weight", 4096, "NULL"),
    ("act", 1, "NULL"),
    ("Ho", 10, "extent"),
])
def test_plan_create_rejects_bad_quantize(field, value, msg):
    d = _q_desc(**{field: value})
    if field == "Cin":
        d.Cout = 24
    _refuse(d, msg)


def test_plan_create_rejects_bad_e4m3_pool_views():
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_UPSAMPLE2X, _C.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = 2, 10, 10, 24, 32, 4096
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = 20, 20, 24, 32, 8192
    _refuse(d, "multiples of 16")


# ---------------------------------------------------------------------------------------------------------------------
# the fake-quant restatement (oracle/restate_fp8.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctor,version", FP8_MODELS)
def test_restate_fp8_without_quantisation_equals_restate_net(ctor, version):
    from oracle import restate as R
    from oracle import restate_fp8 as R8

    sd = _model(ctor, version).model.state_dict()
    x = torch.rand(2, 3, 128, 192, generator=torch.Generator().manual_seed(3))
    ref = R.Net(sd)
    net = R8.NetFP8(sd, None)
    with torch.no_grad():
        a = ref.head(ref.backbone(x))
        b = net.head(net.backbone(x))
    assert all(torch.equal(u, v) for u, v in zip(a, b)) and len(a) == len(b)


@pytest.mark.parametrize("ctor,version", FP8_MODELS)
def test_restate_fp8_rounds_every_module_output_into_its_plan_buffer(ctor, version):
    """With a calibration, every scale the walk asks for names a buffer of the FP8 plan, and the walk's rounding and
    scales agree with the engine's (e4m3_round, e4m3_scale, the scale groups)."""
    from oracle import restate_fp8 as R8

    m = _model(ctor, version).model
    L8, x0, heads, feats, scale = lower_fp8(m, torch.float16, CPU, _amax(lower_yolo(m, torch.float16, CPU)[0]))
    amax = _amax(lower_yolo(m, torch.float16, CPU)[0])
    net = R8.NetFP8(m.state_dict(), amax)
    asked = []
    q0 = net.q
    net.q = lambda t, buf: (asked.append(buf), q0(t, buf))[1]
    with torch.no_grad():
        out = net.head(net.backbone(torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))))
    assert all(torch.isfinite(o).all() for o in out)
    by_name = {b.name: b for b in L8.bufs}
    for buf in set(asked):
        b = by_name["body.0(e4m3)" if buf == "body.0" else buf]
        assert net.scale(buf) == scale[id(b)], buf
    x = torch.randn(4096, dtype=torch.float64) * 300
    assert torch.equal(R8.e4m3_round(x), engine.e4m3_round(x))


def _run_op_list(L, stem_out, fp8, scale=None):
    """A plain fp32 interpreter of a lowering's op list after the stem (test infrastructure).  An e4m3 buffer holds
    its e4m3 codes times the buffer's own scale (`scale`), and every op reads codes and applies the factors its
    descriptor carries, as the kernels do: act(conv(codes, Wq) * m + bias) [+ res codes * s_res], rounded with 1/s_out;
    QUANTIZE with its 1/s; SPP and upsample copy codes.  A factor that disagrees with a buffer's scale therefore shows
    in the values.  Returns {buffer name: NCHW tensor}."""
    import torch.nn.functional as F

    acts = {_C.YB_ACT_SILU: F.silu, _C.YB_ACT_HARDSWISH: F.hardswish, _C.YB_ACT_RELU: F.relu,
            _C.YB_ACT_LEAKY01: lambda t: F.leaky_relu(t, 0.1)}
    bufs = {}

    def get(v):
        return bufs[v.buf.name][:, v.ch0:v.ch0 + v.C]

    def put(v, t):
        b = bufs.setdefault(v.buf.name, torch.zeros(t.shape[0], v.buf.C, t.shape[2], t.shape[3]))
        b[:, v.ch0:v.ch0 + v.C] = t

    def codes(v):      # e4m3 codes of a view (fp8) or its values
        return get(v) / scale[id(v.buf)] if fp8 and v.buf.esz == 1 else get(v)

    def put_codes(v, c):
        put(v, c * scale[id(v.buf)] if fp8 and v.buf.esz == 1 else c)

    put(L.ops[0].dst, stem_out)
    for op in L.ops[1:]:
        if op.kind == _C.YB_OP_QUANTIZE:
            put_codes(op.dst, engine.e4m3_round(get(op.src).double() * float(op.bias[0])).float())
            continue
        src = codes(op.src)
        if op.kind == _C.YB_OP_SPP_POOL:
            put_codes(op.dst, torch.cat([F.max_pool2d(src, k, 1, k // 2) for k in (5, 9, 13)], 1))
            continue
        if op.kind == _C.YB_OP_UPSAMPLE2X:
            put_codes(op.dst, F.interpolate(src, scale_factor=2.0, mode="nearest"))
            continue
        co, ci, k = op.dst.C, op.src.C, op.ksize
        w = op.weight[:co, :, :ci].float().view(co, k, k, ci).permute(0, 3, 1, 2)
        act = acts.get(op.act, lambda t: t)
        if fp8:
            cp, t = op.weight.shape[0], op.bias
            y = act(F.conv2d(src, w, None, op.stride, op.pad) * t[cp:cp + co].view(1, -1, 1, 1) + t[:co].view(1, -1, 1, 1))
            if op.residual is not None:
                y = y + codes(op.residual) * float(t[2 * cp])
            if op.reserved:
                put(op.dst, y)
            else:
                put_codes(op.dst, engine.e4m3_round((y * float(t[2 * cp + 1])).double()).float())
            continue
        else:
            y = act(F.conv2d(src, w, op.bias[:co], op.stride, op.pad))
            if op.residual is not None:
                y = y + get(op.residual)
        put(op.dst, y)
    return bufs


@pytest.mark.parametrize("ctor,version", FP8_MODELS)
def test_fp8_op_list_agrees_with_restate_fp8_buffer_by_buffer(ctor, version):
    """The FP8 lowering against the module walk of oracle/restate_fp8.py, both in fp32 on the CPU with one
    calibration: every module output the walk rounds into a plan buffer equals that buffer of the op list up to the
    rounding flips that fp32 summation order causes.  A flip is one e4m3 step (at most 32 s in the top binade) and the
    next layers carry it, so deep buffers differ by a few steps at most: the bound is 4 top-binade steps (128 s, a
    quarter of the range) and a mean below 10 % of the mean |value|.  A wrong multiplier, weight, scale group or amax
    shows as saturation (up to 448 s and more) or a difference of the size of the values."""
    from oracle import restate_fp8 as R8

    m = _model(ctor, version).model.half().float()
    sd = m.state_dict()
    x = torch.rand(1, 3, 128, 192, generator=torch.Generator().manual_seed(6))
    rec = []
    net = R8.NetFP8(sd, None)
    net.q = lambda t, buf: (rec.append((buf, t)), t)[1]
    with torch.no_grad():
        net.backbone(x)
    stem_out = next(t for buf, t in rec if buf == "body.0")
    L16 = lower_yolo(m, torch.float16, CPU)[0]
    with torch.no_grad():
        b16 = _run_op_list(L16, stem_out, False)
    amax = {k: float(v.abs().max()) for k, v in b16.items()}
    L8, x0, heads, feats, scale = lower_fp8(m, torch.float16, CPU, amax)
    with torch.no_grad():
        b8 = _run_op_list(L8, stem_out, True, scale)
    rec.clear()
    net = R8.NetFP8(sd, amax)
    q0 = net.q
    net.q = lambda t, buf: (lambda r: (rec.append((buf, r)), r)[1])(q0(t, buf))
    with torch.no_grad():
        net.backbone(x)
    checked = 0
    for buf, t in rec:
        got = b8["body.0(e4m3)" if buf == "body.0" else buf]
        if got.shape[1] != t.shape[1]:       # a window of a concat buffer: the windows are checked through the blocks
            continue
        s = net.scale(buf)
        d = (got - t).abs()
        assert float(d.max()) <= 128 * s, (buf, float(d.max()), s)
        assert float(d.mean()) <= 0.1 * float(t.abs().mean()) + 1e-12, buf
        checked += 1
    assert checked >= 15
