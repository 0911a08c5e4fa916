"""FP8 (e4m3) inference on the H100: the e4m3 convolution, QUANTIZE, SPP and upsample kernels against fp32 PyTorch on
the dequantised operands, every launch of FP8 plans at real shapes, and the model-level behaviour (calibration,
precision switching, hooks, graph replay, stale calibrations).  The bounds of e4m3 and of 16-bit outputs are
tests/stagewise.py's (e4m3_bound, bound16); measured worst cases are printed."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from stagewise import act_ref, bound16, check_plan_stagewise, compare, e4m3_bound, to_e4m3
from yolort_b200 import _C
from yolort_b200.engine import e4m3_scale, pack_weight_e4m3

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F8 = torch.float8_e4m3fn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

A = _C


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


# ---------------------------------------------------------------------------------------------------------------------
# the e4m3 convolution op
# ---------------------------------------------------------------------------------------------------------------------
S, H, L, R, NONE = A.YB_ACT_SILU, A.YB_ACT_HARDSWISH, A.YB_ACT_LEAKY01, A.YB_ACT_RELU, A.YB_ACT_NONE
# (k, s, Cin, Cout, output, residual, act, (N, H, W))
CASES = [
    (1, 1, 16, 16, "e4m3", False, S, (2, 20, 20)),
    (3, 1, 16, 32, "e4m3", True, S, (2, 20, 20)),
    (3, 2, 16, 48, "e4m3", False, H, (2, 20, 20)),
    (1, 1, 48, 48, "e4m3", True, L, (2, 20, 20)),
    (3, 1, 48, 80, "e4m3", False, R, (2, 20, 20)),
    (3, 2, 80, 128, "e4m3", False, NONE, (2, 20, 20)),
    (1, 1, 80, 80, "e4m3", True, S, (2, 20, 20)),
    (3, 1, 128, 128, "e4m3", True, S, (2, 20, 20)),
    (3, 2, 128, 640, "e4m3", False, S, (2, 20, 20)),
    (1, 1, 640, 640, "e4m3", True, H, (2, 20, 20)),
    (3, 1, 640, 48, "e4m3", False, L, (2, 12, 12)),
    (1, 1, 128, 256, "e4m3", True, S, (4, 96, 96)),      # M >= 2 x SMs x 128: one 256-wide N tile
    (3, 1, 80, 256, "e4m3", False, R, (4, 96, 96)),
    (1, 1, 128, 256, "f16", False, NONE, (4, 96, 96)),   # a head: fp16 logits
    (1, 1, 640, 256, "bf16", False, NONE, (2, 20, 20)),
    (1, 1, 80, 48, "f16", False, S, (2, 20, 20)),
    (3, 1, 48, 16, "bf16", False, R, (2, 20, 20)),
    (3, 2, 16, 640, "f16", False, H, (2, 20, 20)),
]
PAD = 16      # channel offset of every window inside its (wider) buffer; the other channels are sentinels


def conv_case(k, s, cin, cout, out, residual, act_code, shape, seed=0):
    N, Hh, Ww = shape
    p = k // 2
    Ho, Wo = (Hh + 2 * p - k) // s + 1, (Ww + 2 * p - k) // s + 1
    g = torch.Generator().manual_seed(seed + 7 * cin + cout)
    xbuf = to_e4m3(torch.randn(N, Hh, Ww, cin + 2 * PAD, generator=g) * 3.0).to(DEV)
    s_in = 2.0 ** -2
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) * (2.0 / (cin * k * k)) ** 0.5
    s_w = torch.tensor([e4m3_scale(a) for a in w.abs().amax(dim=(1, 2, 3)).tolist()], dtype=torch.float64)
    wq = pack_weight_e4m3(w, s_w, DEV)
    co_pad = wq.shape[0]
    bias = torch.randn(cout, generator=g, dtype=torch.float64) * 0.5
    m = (s_w * s_in).float().to(DEV)
    xs = xbuf[..., PAD:PAD + cin].float().permute(0, 3, 1, 2)
    ws = wq[:cout, :, :cin].float().view(cout, k, k, cin).permute(0, 3, 1, 2)
    v = act_ref(F.conv2d(xs, ws, None, s, p) * m.view(1, -1, 1, 1) + bias.float().to(DEV).view(1, -1, 1, 1), act_code)
    mag = F.conv2d(xs.abs(), ws.abs(), None, s, p) * m.view(1, -1, 1, 1)
    s_res, rbuf = 0.0, None
    if residual:
        s_res = 2.0 ** -1
        rbuf = to_e4m3(torch.randn(N, Ho, Wo, cout + 2 * PAD, generator=g) * 4.0).to(DEV)
        v = v + rbuf[..., PAD:PAD + cout].float().permute(0, 3, 1, 2) * s_res
    if out == "e4m3":
        s_out = e4m3_scale(float(torch.quantile(v.abs().flatten()[:1 << 20].cpu(), 0.98)))   # ~2 % saturate
        obuf = torch.full((N, Ho, Wo, cout + 2 * PAD), 1.75, device=DEV).to(F8)
    else:
        s_out = 1.0
        obuf = torch.full((N, Ho, Wo, cout + 2 * PAD), 7.0, device=DEV,
                          dtype=torch.float16 if out == "f16" else torch.bfloat16)
    tail = torch.zeros(2 * co_pad + 2, dtype=torch.float64)
    tail[:cout] = bias
    tail[co_pad:co_pad + cout] = s_w * s_in
    tail[2 * co_pad], tail[2 * co_pad + 1] = s_res, 1.0 / s_out
    tail = tail.float().to(DEV)
    esz = 1 if out == "e4m3" else 2
    d = _C.OpDesc()
    d.kind, d.dtype = A.YB_OP_CONV, A.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, Hh, Ww, cin, cin + 2 * PAD, xbuf.data_ptr() + PAD
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = Ho, Wo, cout, cout + 2 * PAD, obuf.data_ptr() + PAD * esz
    d.ksize, d.stride, d.pad, d.act = k, s, p, act_code
    d.weight, d.Cout_pad, d.Cin_pad = wq.data_ptr(), co_pad, wq.shape[2]
    d.bias = tail.data_ptr()
    if rbuf is not None:
        d.residual, d.res_cstride = rbuf.data_ptr() + PAD, cout + 2 * PAD
    d.reserved = {"e4m3": 0, "f16": 16, "bf16": 32}[out]
    keep = (xbuf, wq, tail, rbuf, obuf, mag)
    return d, keep, v, s_out, obuf


@pytest.mark.parametrize("case", CASES, ids=[f"k{c[0]}s{c[1]}_{c[2]}to{c[3]}_{c[4]}{'_res' if c[5] else ''}_act{c[6]}"
                                             for c in CASES])
def test_e4m3_conv_matches_fp32_on_dequantised_operands(case):
    k, s, cin, cout, out, residual, act_code, shape = case
    d, keep, v, s_out, obuf = conv_case(*case)
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    got = obuf[..., PAD:PAD + cout].permute(0, 3, 1, 2).float()
    if out == "e4m3":
        ref, bound = e4m3_bound(v / s_out, keep[-1] / s_out)
    else:
        ref, bound = v, bound16(v, obuf.dtype, keep[-1])
    bad, mx, worst = compare(got, ref, bound)
    print(f"{case}: worst {worst:.3f} of the bound")
    assert bad == 0, f"{case}: {bad}/{got.numel()} outside the bound, max err {mx:.3e}"
    full = obuf.float()
    assert torch.all(full[..., :PAD] == full[0, 0, 0, 0]) and torch.all(full[..., PAD + cout:] == full[0, 0, 0, 0])
    assert float(full[0, 0, 0, 0]) == (1.75 if out == "e4m3" else 7.0), "sentinels overwritten"


def test_e4m3_conv_cases_cover_every_n_tile():
    widths = {_C.conv_config(conv_case(*c)[0])["block_n"] for c in CASES}
    assert widths >= {16, 32, 64, 128, 256}, widths


# ---------------------------------------------------------------------------------------------------------------------
# QUANTIZE, SPP and upsample at e4m3
# ---------------------------------------------------------------------------------------------------------------------
def _bits(q):
    b = q.contiguous().view(torch.uint8)
    return torch.where(b == 0x80, torch.zeros_like(b), b)     # -0 and +0 compare equal


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_quantize_bit_exact_against_clamp_and_cast(dtype):
    N, Hh, Ww, C = 2, 17, 9, 48
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(N, Hh, Ww, C + 16, generator=g) * 150.0).to(dtype).to(DEV)   # some values saturate
    x[0, 0, 0, :8] = torch.tensor([0.0, -0.0, 1e-4, -1e-4, 300.0, -5000.0, 2.0 ** -10, 0.4375], dtype=dtype)
    s = 2.0 ** -1
    inv = torch.tensor([1.0 / s], device=DEV)
    out = torch.full((N, Hh, Ww, C + 32), 3.0, device=DEV).to(F8)
    d = _C.OpDesc()
    d.kind, d.dtype = A.YB_OP_QUANTIZE, _C.dtype_code(dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, Hh, Ww, C, C + 16, x.data_ptr() + 8 * 2
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = Hh, Ww, C, C + 32, out.data_ptr() + 16
    d.bias = inv.data_ptr()
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    ref = to_e4m3(x[..., 8:8 + C].float() / s)
    assert torch.equal(_bits(out[..., 16:16 + C]), _bits(ref))
    assert torch.all(out[..., :16].float() == 3.0) and torch.all(out[..., 16 + C:].float() == 3.0)


@pytest.mark.parametrize("hw", [(20, 20), (13, 20), (40, 40), (7, 5), (120, 120)])
def test_spp_pool_e4m3_exact(hw):
    N, C = 2, 64
    Hh, Ww = hw
    g = torch.Generator().manual_seed(1)
    cat = to_e4m3(torch.randn(N, Hh, Ww, 4 * C, generator=g) * 20.0).to(DEV)
    x = cat[..., :C].float().permute(0, 3, 1, 2)
    d = _C.OpDesc()
    d.kind, d.dtype = A.YB_OP_SPP_POOL, A.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, Hh, Ww, C, 4 * C, cat.data_ptr()
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = Hh, Ww, 3 * C, 4 * C, cat.data_ptr() + C
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    for i, k in enumerate((5, 9, 13)):
        ref = F.max_pool2d(x, k, 1, k // 2)
        assert torch.equal(cat[..., (i + 1) * C:(i + 2) * C].float().permute(0, 3, 1, 2), ref), (k, hw)


def test_upsample2x_e4m3_exact():
    N, Hh, Ww, C = 2, 10, 6, 32
    g = torch.Generator().manual_seed(2)
    src = to_e4m3(torch.randn(N, Hh, Ww, 2 * C, generator=g) * 30.0).to(DEV)
    dst = torch.full((N, 2 * Hh, 2 * Ww, 3 * C), 5.0, device=DEV).to(F8)
    d = _C.OpDesc()
    d.kind, d.dtype = A.YB_OP_UPSAMPLE2X, A.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, Hh, Ww, C, 2 * C, src.data_ptr() + C
    d.Ho, d.Wo, d.Cout, d.out_cstride, d.out = 2 * Hh, 2 * Ww, C, 3 * C, dst.data_ptr() + C
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    ref = src[..., C:].view(torch.uint8).repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(dst[..., C:2 * C].view(torch.uint8), ref)
    assert torch.all(dst[..., :C].float() == 5.0) and torch.all(dst[..., 2 * C:].float() == 5.0)


# ---------------------------------------------------------------------------------------------------------------------
# every launch of FP8 plans at real shapes
# ---------------------------------------------------------------------------------------------------------------------
def _fp8_model(ctor_name, gain=None, dtype=torch.float16, **kw):
    import bench
    from yolort_b200 import models

    m = getattr(models, ctor_name)(**kw).eval()
    sd = bench.make_state_dict(m) if gain is None else bench.zoo_state_dict(m, gain)
    m.load_state_dict(sd)
    return m.to(DEV).to(dtype)


@pytest.mark.parametrize("ctor,version,gain,batch,size", [
    ("yolov5s", "r6.0", None, 32, 640),
    ("yolov5x", "r6.0", 1.3, 8, 1280),
    ("yolov5n6", "r6.0", 1.4, 4, 1280),
    ("yolov5s", "r4.0", 1.4, 8, 640),
    ("yolov5s", "r3.1", 1.4, 8, 640),
])
def test_every_launch_of_fp8_plans(ctor, version, gain, batch, size):
    import bench
    from yolort_b200.quantization import calibrate_fp8

    m = _fp8_model(ctor, gain, upstream_version=version, size=(size, size))
    ims = [im.to(DEV) for im in bench.make_images(batch, 4321, size)]
    calib = calibrate_fp8(m, [ims])
    m.set_fp8(calib)
    yolo = m.model
    eng = yolo.engine()
    plan = eng.plan(batch, size, size, keep_intermediates=True)
    assert plan._low.fp8
    geoms, (Hb, Wb) = m.transform.geometry(ims, None)
    m.transform.letterbox_into(ims, geoms, Hb, Wb, plan.input, _C.YB_LAYOUT_S2D16)
    res = check_plan_stagewise(plan, m.model.backbone.body["0"])
    assert len(res) == len(plan._low.L.ops)
    bad = [r for r in res if r.violations]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def s320():
    import bench
    from yolort_b200.quantization import calibrate_fp8

    m = _fp8_model("yolov5s", size=(320, 320), score_thresh=bench.SCORE_THRESH)
    calib = calibrate_fp8(m, [[im.to(DEV) for im in bench.make_images(4, 777, 320)]])
    ims = [im.to(DEV) for im in bench.make_images(2, 1234, 320)]
    return m, calib, ims


def _same(a, b):
    return all(torch.equal(x[k], y[k]) for x, y in zip(a, b) for k in ("scores", "labels", "boxes")) and len(a) == len(b)


def test_fp8_end_to_end_matches_restate_fp8(s320):
    """The FP8 plan against the CPU fake-quant restatement (oracle/restate_fp8.py: a walk over the modules with the
    same calibration), under the north-star matching rule (same label, IoU > 0.9)."""
    import bench
    import parity_util as util
    from oracle import restate_fp8 as R8

    m, calib, _ = s320
    host = bench.make_images(2, 1234, 320)
    m.set_fp8(calib)
    try:
        got = [util.to_np(d) for d in m([im.to(DEV) for im in host])]
    finally:
        m.set_fp8(None)
    sd = {k: v.detach().cpu() for k, v in m.model.state_dict().items()}
    ref = [util.to_np(d) for d in R8.detect(sd, calib.amax, host, score_thresh=bench.SCORE_THRESH, size=(320, 320))]
    st = [util.pair_stats(g, r, 320.0) for g, r in zip(got, ref)]
    n_ref = sum(x["n_ref"] for x in st)
    frac = sum(x["matched"] * x["n_ref"] for x in st) / max(n_ref, 1)
    print(f"FP8 plan vs restate_fp8 yolov5s 2 x 320^2: matched {frac:.4f} of {n_ref} detections, "
          f"{[round(x['within'], 4) for x in st]} of the pairs within 1e-3 x side, "
          f"max |dbox|/side {max(x['max_box_rel'] for x in st):.2e}, max |dscore| {max(x['max_score_err'] for x in st):.2e}")
    assert n_ref > 100
    # measured 0.085 on an H100 (482 detections): an e4m3 network amplifies rounding-order differences (see the logits
    # test below), and the synthetic weights put many scores within that noise of each other, so the NMS reorders them
    assert frac >= 0.05


def test_fp8_logits_match_restate_fp8_within_the_quantisation_noise(s320):
    """The plan's head logits against restate_fp8 on the plan's own input canvas.  An 8-bit network amplifies
    rounding-order differences (a flipped e4m3 rounding is a 6 % change that the next layers carry), so the plan and the
    restatement agree to a fraction of the quantisation error itself, not bit for bit; a lowering mistake (a wrong
    scale, multiplier, weight or scale group) shows as a difference of the size of that error or more."""
    import bench
    from oracle import restate_fp8 as R8

    m, calib, _ = s320
    m.set_fp8(calib)
    try:
        m([im.to(DEV) for im in bench.make_images(2, 1234, 320)])      # letterboxes into the cached plan's canvas
        plan = m.model.get_plan(2, 320, 320)
        plan.run()
        torch.cuda.synchronize()
        heads = [h[..., :255].float().cpu() for h in plan.heads]
        canvas = plan.input.float().cpu()
    finally:
        m.set_fp8(None)
    n, h2, w2, _ = canvas.shape
    x = canvas.view(n, h2, w2, 2, 2, 4)[..., :3].permute(0, 5, 1, 3, 2, 4).reshape(n, 3, 2 * h2, 2 * w2)
    sd = {k: v.detach().cpu() for k, v in m.model.state_dict().items()}
    q, f = R8.NetFP8(sd, calib.amax), R8.NetFP8(sd, None)
    with torch.no_grad():
        hq, hf = q.head(q.backbone(x)), f.head(f.backbone(x))
    ratios = []
    for i, (g, a, b) in enumerate(zip(heads, hq, hf)):
        nn_, hh, ww, _ = g.shape
        g = g.view(nn_, hh, ww, 3, 85).permute(0, 3, 1, 2, 4)
        d_plan = float((g - a).abs().mean())
        d_quant = float((a - b).abs().mean())
        ratios.append(d_plan / d_quant)
        print(f"head {i}: mean |plan - restate_fp8| {d_plan:.4f}, mean |restate_fp8 - restate (fp32)| {d_quant:.4f}, "
              f"ratio {d_plan / d_quant:.3f}, max |plan - restate_fp8| {float((g - a).abs().max()):.3f}")
    assert max(ratios) <= 1.25      # measured 0.94-0.98 on an H100


def test_fp8_end_to_end_matches_fp16_detections(s320):
    import parity_util as util

    m, calib, ims = s320
    m.set_fp8(None)
    ref = [util.to_np(d) for d in m(ims)]
    m.set_fp8(calib)
    assert m.precision == "fp8"
    got = [util.to_np(d) for d in m(ims)]
    m.set_fp8(None)
    n_ref = sum(len(r["scores"]) for r in ref)
    frac = sum(util.match_fraction(g, r) * len(r["scores"]) for g, r in zip(got, ref)) / max(n_ref, 1)
    print(f"FP8 vs fp16 yolov5s 2 x 320^2: matched {frac:.4f} of {n_ref} detections (same label, IoU > 0.9)")
    assert n_ref > 100
    assert frac >= 0.1      # measured 0.128 on an H100 (383 fp16 detections)


def test_fp8_off_restores_fp16_bits_and_graph_replay(s320):
    m, calib, ims = s320
    m.set_fp8(None)
    before = m(ims)
    m.set_fp8(calib)
    a = m(ims)
    yolo = m.model
    yolo.engine().graphs = True
    try:
        b = m(ims)
        c = m(ims)
    finally:
        yolo.engine().graphs = False
        for p in yolo.engine()._plans.values():
            p.use_graph = False
    assert _same(a, b) and _same(b, c), "graph replay of the FP8 plan"
    m.set_fp8(None)
    assert m.precision == "fp16"
    assert _same(before, m(ims)), "fp16 detections after switching FP8 off"


def test_fp8_hook_path_equals_fused_path(s320):
    m, calib, ims = s320
    m.set_fp8(calib)
    try:
        fused = m(ims)
        seen = []
        h = m.model.backbone.register_forward_hook(lambda mod, i, o: seen.append([t.dtype for t in o]))
        try:
            hooked = m(ims)
        finally:
            h.remove()
        assert seen and all(dt == torch.float16 for dt in seen[0])
        assert _same(fused, hooked)
    finally:
        m.set_fp8(None)


def test_fp8_predict_paths(s320):
    """predict on host images (the chunked front), predict_stream and forward_padded give forward's detections."""
    import bench

    m, calib, _ = s320
    m.set_fp8(calib)
    try:
        host = bench.make_images(16, 99, 320)
        dev = [im.to(DEV) for im in host]
        ref = m(dev)
        assert _same(ref, m.predict(host))
        streamed = next(iter(m.predict_stream([host])))
        assert _same([{k: v.to(DEV) for k, v in d.items()} for d in streamed], ref)
        boxes, scores, labels, counts, status = m.forward_padded(dev)
        assert int(status[1]) == 0 and [int(c) for c in counts] == [len(d["scores"]) for d in ref]
    finally:
        m.set_fp8(None)


def test_stale_calibration_raises_and_moves_keep_it():
    import bench
    from yolort_b200.quantization import calibrate_fp8

    m = _fp8_model("yolov5n", size=(128, 128))
    ims = [im.to(DEV) for im in bench.make_images(2, 5, 128)]
    calib = calibrate_fp8(m, [ims])
    m.set_fp8(calib)
    m(ims)
    m.to(DEV).half()                     # moves keep the calibration
    m(ims)
    with torch.no_grad():
        next(m.parameters()).mul_(1.0)   # an in-place edit
    with pytest.raises(RuntimeError, match="stale"):
        m(ims)
    m.set_fp8(calib)
    m(ims)
    m.model.load_state_dict(m.model.state_dict())
    with pytest.raises(RuntimeError, match="stale"):
        m(ims)
    m.set_fp8(None)
    m(ims)


def test_fused_decode_has_no_fp8_variant(s320, monkeypatch):
    m, calib, ims = s320
    m.set_fp8(calib)
    monkeypatch.setenv("YB_FUSED_DECODE", "1")
    try:
        with pytest.raises(NotImplementedError):
            m(ims)
    finally:
        m.set_fp8(None)
