"""Whole-graph parity: backbone+PAN+head on the native plan vs reference fixtures / oracle, and end to end (H100)."""
import numpy as np
import pytest
import torch

import parity_util as util
from oracle import restate as R
from yolort_b200.models import yolov5n, yolov5s

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _stats(name, got, ref):
    err = np.abs(got - ref)
    rel_rms = util.rel_rms(got, ref)
    print(f"{name}: max_abs={err.max():.4f} rel_rms={rel_rms:.2e} ref_rms={np.sqrt((ref ** 2).mean()):.3f}")
    return float(err.max()), rel_rms


def _model_n():
    sd = util.synth_state_dict(util.layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0)
    m = yolov5n(size=(128, 128), score_thresh=0.15).eval()
    m.load_state_dict(sd)
    return m.to(DEV), sd


def test_features_and_heads_vs_reference_fixture():
    z = util.load_npz("network_n.npz")
    m, sd = _model_n()
    x = torch.from_numpy(z["x"]).to(DEV)
    dets = m.model(x)   # YOLO.forward on a pre-letterboxed NCHW batch
    plan = m.model.get_plan(1, 96, 128)
    m.model.run_plan(plan)   # (re)store the head logits
    torch.cuda.synchronize()
    for key, name in (("p3", "p3"), ("p4", "p4"), ("p5", "p5")):
        got = plan.features[name].float().permute(0, 3, 1, 2).cpu().numpy()
        mx, rr = _stats(key, got, z[key])
        assert rr < 1.5e-2      # fp16 activations through 20-30 layers vs the fp32 reference
    for i in range(3):
        mx, rr = _stats(f"head{i}", util.head_logits(plan, i), z[f"h{i}"])
        assert rr < 1.5e-2
    ref = util.dets_from_npz(z, 1)[0]
    frac = util.match_fraction(util.to_np(dets[0]), ref, iou_thr=0.9, side=128)
    print("network dets matched:", frac, len(dets[0]["scores"]), len(ref["scores"]))
    assert frac >= 0.97      # measured 0.993; matched boxes within 1e-3 x canvas (asserted inside)


def test_per_layer_stagewise_parity_yolov5n():
    """Each launch of the plan vs the fp32 oracle applied to the SAME (fp16) input of that stage: feed the
    oracle our previous activations by comparing only final taps with tight per-stage growth."""
    m, sd = _model_n()
    g = torch.Generator().manual_seed(3)
    x = torch.rand(2, 3, 64, 96, generator=g)
    plan = m.model.get_plan(2, 64, 96, keep_intermediates=True)   # default arenas reuse the bytes of dead activations
    m.model._write_samples(plan, x.to(DEV))
    plan.run()
    torch.cuda.synchronize()
    net = R.Net(sd)
    with torch.no_grad():
        xr = x.half().float()
        stem = net.conv(xr, "backbone.body.0")
        b1 = net.conv(stem, "backbone.body.1")
    got_stem = plan.buffers["body.0"].float().permute(0, 3, 1, 2).cpu().numpy()
    mx, rr = _stats("stem", got_stem, stem.numpy())
    assert rr < 2e-3
    got_b1 = plan.buffers["body.1"].float().permute(0, 3, 1, 2).cpu().numpy()
    mx, rr = _stats("body.1", got_b1, b1.numpy())
    assert rr < 3e-3


def test_end_to_end_vs_reference_fixture():
    z = util.load_npz("e2e_n.npz")
    m, sd = _model_n()
    ims = [torch.from_numpy(z["img0"]).to(DEV), torch.from_numpy(z["img1"]).to(DEV)]
    out = m(ims)
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        got = util.to_np(got)
        frac = util.match_fraction(got, ref, iou_thr=0.9, side=128)
        print("e2e matched fraction:", frac, "n_got", len(got["scores"]), "n_ref", len(ref["scores"]))
        assert frac >= 0.97      # measured 1.0 / 0.997
    # float inputs in [0,1] (the reference's own input contract) give the same detections as uint8 inputs
    # (the CUDA `/255` may differ from the CPU LUT by 1 ulp, so near-tied scores may swap places)
    out_f = m([im.float() / 255.0 for im in ims])
    for a, b in zip(out, out_f):
        assert util.match_fraction(util.to_np(b), util.to_np(a), iou_thr=0.95) >= 0.99


def test_predict_and_shapes_yolov5s_default_weights():
    m = yolov5s().eval().to(DEV)
    ims = [torch.randint(0, 256, (3, 480, 640), dtype=torch.uint8), torch.randint(0, 256, (3, 375, 500), dtype=torch.uint8)]
    out = m.predict(ims)
    assert isinstance(out, list) and len(out) == 2
    for d in out:
        assert d["boxes"].shape[1:] == (4,) and d["labels"].dtype == torch.int64 and d["scores"].dtype == torch.float32
        assert d["boxes"].shape[0] == d["scores"].shape[0] == d["labels"].shape[0] <= 300


def test_mixed_size_batch_vs_oracle():
    """Dynamic-shape batch (BASELINE.json configs[3] in miniature): different aspect ratios in one batch, the
    canvas is the batch maximum rounded up to 32; boxes come back in each image's own pixel frame."""
    m, sd = _model_n()
    ims = [util.synth_image_u8(h, w, 40 + i) for i, (h, w) in enumerate([(97, 128), (128, 64), (75, 75), (50, 117), (128, 128)])]
    ref = R.detect(sd, ims, score_thresh=0.15, size=(128, 128))
    out = m([im.to(DEV) for im in ims])
    for got, want, im in zip(out, ref, ims):
        got = util.to_np(got)
        frac = util.match_fraction(got, want, iou_thr=0.9, side=128)
        print("mixed batch", tuple(im.shape[1:]), "matched", frac, len(got["scores"]), len(want["scores"]))
        assert frac >= 0.95      # measured 0.977 .. 1.0 (300 detections cut out of a dense, near-tied candidate set)


def test_bf16_model_end_to_end():
    m, sd = _model_n()
    m = m.to(torch.bfloat16)
    z = util.load_npz("e2e_n.npz")
    ims = [torch.from_numpy(z["img0"]).to(DEV), torch.from_numpy(z["img1"]).to(DEV)]
    out = m(ims)
    for got, ref in zip(out, util.dets_from_npz(z, 2)):
        frac = util.match_fraction(util.to_np(got), ref, iou_thr=0.8)
        print("bf16 e2e matched fraction:", frac)
        assert frac >= 0.93     # measured 0.963 / 0.99; bf16 activations: 8 mantissa bits through ~25 layers


def test_fused_head_decode_equals_unfused(monkeypatch):
    """Heads with the decode epilogue (fp32 accumulators -> candidates) vs stored fp16 logits + stand-alone decode."""
    m, sd = _model_n()
    z = util.load_npz("e2e_n.npz")
    ims = [torch.from_numpy(z["img0"]).to(DEV), torch.from_numpy(z["img1"]).to(DEV)]
    plain = m(ims)
    monkeypatch.setenv("YB_FUSED_DECODE", "1")
    fused = m(ims)
    assert m.model.get_plan(2, 128, 128).fused_post is not None
    for a, b in zip(fused, plain):
        assert abs(len(a["scores"]) - len(b["scores"])) <= 3
        frac = util.match_fraction(util.to_np(a), util.to_np(b), iou_thr=0.95)
        print("fused vs unfused matched:", frac)
        assert frac >= 0.97      # logits rounded to fp16 in the unfused path move scores by <= 1e-3


def test_pipelined_host_predict_equals_device_forward():
    """predict() on >= 16 host images (a multiple of 4) copies them in four chunks and runs letterbox + the front of
    the plan per chunk while later chunks are still in flight; results must equal the device-resident call bit for
    bit (mixed sizes: every chunk is letterboxed to the whole batch's canvas)."""
    m, sd = _model_n()
    ims = [util.synth_image_u8(64 + 8 * (i % 5), 128 - 8 * (i % 3), 70 + i) for i in range(20)]
    ref = m([im.to(DEV) for im in ims])
    pinned = [im.pin_memory() for im in ims]
    assert m._predict_pipelined(pinned) is not None          # the chunked path is the one predict() takes here
    Hb, Wb = m.transform.geometry(ims)[1]
    plan = m.model.get_plan(20, Hb, Wb, chunked=True)
    assert plan.front_chunks == 4 and plan._front_op_count == 13 and plan.front_ops <= 13   # 13 ops, fewer launches when tails are chained
    for _ in range(2):                                        # twice: staging / arena reuse across calls
        got = m.predict(pinned)
        assert len(got) == len(ref) == 20
        for a, b in zip(got, ref):
            assert torch.equal(a["labels"], b["labels"]) and torch.equal(a["scores"], b["scores"])
            assert torch.equal(a["boxes"], b["boxes"])
    assert m._predict_pipelined(pinned[:18]) is None          # 18 images: not a multiple of 4 -> plain path
    got = m.predict(pinned[:18])
    for a, b in zip(got, m([im.to(DEV) for im in ims[:18]])):
        assert torch.equal(a["boxes"], b["boxes"])


def test_predict_stream_equals_predict():
    """The throughput API (copy of batch i+1 overlapping batch i, async result block) returns exactly predict()'s
    detections, batch after batch, for mixed sizes, changing batch sizes and more batches than ring slots."""
    m, sd = _model_n()
    batches = []
    for b in range(7):
        n = 1 + (b * 3) % 5
        ims = [util.synth_image_u8(64 + 8 * ((b + j) % 5), 96 + 16 * ((b * j) % 3), 500 + 10 * b + j) for j in range(n)]
        pinned = torch.cat([im.reshape(-1) for im in ims]).pin_memory()
        off, views = 0, []
        for im in ims:
            views.append(pinned[off: off + im.numel()].view(im.shape))
            off += im.numel()
        batches.append(views)
    want = [m.predict(b) for b in batches]
    got = list(m.predict_stream(iter(batches)))
    assert len(got) == len(want) == 7
    for gb, wb in zip(got, want):
        assert len(gb) == len(wb)
        for g, w in zip(gb, wb):
            assert not g["boxes"].is_cuda and g["labels"].dtype == torch.int64
            assert torch.equal(g["labels"], w["labels"].cpu())
            assert torch.equal(g["scores"], w["scores"].cpu()) and torch.equal(g["boxes"], w["boxes"].cpu())
    assert list(m.predict_stream(iter([]))) == []
