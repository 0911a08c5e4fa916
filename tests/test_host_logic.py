"""CPU-only checks of the host side: C-ABI loads and exports every declared symbol, host geometry
functions agree with the reference fixtures, module layout/state-dict keys equal the reference's, graph
lowering emits the reference's algorithmic work.  No kernel is launched."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

import parity_util as util
from yolort_b200 import _C
from yolort_b200.models import yolov5l, yolov5m, yolov5n, yolov5s, yolov5x, YOLOv5
from yolort_b200.models._utils import depth_gain, make_divisible
from yolort_b200.models.anchor_utils import AnchorGenerator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = _C.lib()
    header = open(os.path.join(ROOT, "include", "yolort_b200.h")).read()
    declared = set(re.findall(r"\b(yb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_C.EXPORTED_SYMBOLS), declared ^ set(_C.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.yb_abi_version() == 2


def test_ctypes_structs_match_header_sizes(tmp_path):
    """The ctypes mirrors must have the C layout of include/yolort_b200.h (checked with the C compiler)."""
    import subprocess

    src = tmp_path / "sz.c"
    src.write_text(
        '#include <stdio.h>\n#include "yolort_b200.h"\n'
        'int main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(yb_letterbox_geom), sizeof(yb_op_desc), '
        'sizeof(yb_head_level), sizeof(yb_nms_params), sizeof(yb_conv_chain));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert sizes == [ctypes.sizeof(_C.LetterboxGeom), ctypes.sizeof(_C.OpDesc), ctypes.sizeof(_C.HeadLevel),
                     ctypes.sizeof(_C.NmsParams), ctypes.sizeof(_C.ConvChain)]


def test_letterbox_geometry_matches_reference(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "letterbox_geometry.json")))
    sizes = [(h, w) for h, w, _, _ in g["sizes"]]
    geoms, _ = _C.letterbox_geometry(sizes, 640.0, 640.0, 32, None)
    for (h, w, nh, nw), gg in zip(g["sizes"], geoms):
        assert (gg.new_h, gg.new_w) == (nh, nw), (h, w)
        assert gg.ratio_h == np.float32(h) / np.float32(nh) and gg.ratio_w == np.float32(w) / np.float32(nw)
    for b in g["batches"]:
        sz = [sizes[i] for i in b["idx"]]
        geoms, (Hb, Wb) = _C.letterbox_geometry(sz, 640.0, 640.0, 32, None)
        assert (Hb, Wb) == (b["Hb"], b["Wb"])
        assert [(gg.top, gg.left) for gg in geoms] == [tuple(o) for o in b["offsets"]]
        probe = np.array([[10.0, 20.0, 300.5, 400.25], [0.0, 0.0, Wb, Hb]], dtype=np.float32)
        for (h, w), ref in zip(sz, b["scaled"]):
            gain, px, py = (np.float32(v) for v in _C.scale_coords_params(Hb, Wb, h, w))
            got = probe.copy()
            got[:, 0::2] = (got[:, 0::2] - px) / gain
            got[:, 1::2] = (got[:, 1::2] - py) / gain
            assert np.array_equal(got, np.array(ref, dtype=np.float32))


def test_letterbox_geometry_fixed_shape_and_errors():
    geoms, hw = _C.letterbox_geometry([(480, 640)], 640.0, 640.0, 32, (672, 672))
    assert hw == (672, 672) and (geoms[0].new_h, geoms[0].new_w) == (480, 640)
    assert (geoms[0].top, geoms[0].left) == (96, 16)
    with pytest.raises(_C.NativeLibraryError):
        _C.letterbox_geometry([(480, 640)], 640.0, 640.0, 32, (320, 320))


def test_make_divisible_known_answers():
    # yolort test/test_models_utils.py:16-37
    assert make_divisible(16.0, 8) == 16
    assert make_divisible(17.0, 8) == 16
    assert make_divisible(1.0, 8, min_value=8) == 8
    assert make_divisible(1.0, 8, min_value=16) == 16
    assert make_divisible(20.0, 16) >= 0.9 * 20.0
    assert make_divisible(256.0, 8) == 256
    assert [depth_gain(n, 0.33) for n in (3, 6, 9)] == [1, 2, 3]
    assert [depth_gain(n, 1.33) for n in (3, 6, 9)] == [4, 8, 12]


def test_anchor_generator_golden():
    # yolort test/test_models_anchor_utils.py:14-30
    grids, shifts = AnchorGenerator([4], [[6, 14]])([torch.rand(2, 8, 2, 2)])
    assert tuple(grids[0].shape) == (1, 1, 2, 2, 2)
    torch.testing.assert_close(grids[0], torch.tensor([[[[[0.0, 0.0], [1.0, 0.0]], [[0.0, 1.0], [1.0, 1.0]]]]]))
    torch.testing.assert_close(shifts[0], torch.tensor([[[[[6.0, 14.0], [6.0, 14.0]], [[6.0, 14.0], [6.0, 14.0]]]]]))


@pytest.mark.parametrize("name,ctor", [("n", yolov5n), ("s", yolov5s), ("m", yolov5m), ("l", yolov5l), ("x", yolov5x)])
def test_state_dict_layout_equals_reference(name, ctor):
    ref = util.layouts()[name]
    sd = ctor().state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: list(v.shape) for k, v in sd.items()} == ref
    m = ctor()
    m.load_state_dict(util.synth_state_dict(ref))  # a reference-layout state dict loads unchanged


def test_constructor_surface_and_errors():
    m = YOLOv5(arch="yolov5_darknet_pan_s_r60", score_thresh=0.3, nms_thresh=0.5, detections_per_img=100,
               size=(320, 416), size_divisible=64, fill_color=0)
    pp = m.model.post_process
    assert (pp.score_thresh, pp.nms_thresh, pp.detections_per_img) == (0.3, 0.5, 100)
    assert (m.transform.min_size, m.transform.max_size, m.transform.size_divisible, m.transform.fill_color) == (320, 416, 64, 0.0)
    assert yolov5s().model.post_process.score_thresh == 0.005  # yolo.py:77-79 defaults
    with pytest.raises(NotImplementedError):
        yolov5s(upstream_version="r5.0")
    with pytest.raises(ValueError):
        YOLOv5(arch="nope")
    with pytest.raises(NotImplementedError):
        m.collate_images(123, None)


def test_no_cpu_fallback():
    m = yolov5n().eval()
    with pytest.raises(_C.NativeLibraryError):
        m([torch.rand(3, 64, 64)])            # CPU tensors: must fail loudly, never compute on the host
    with pytest.raises(RuntimeError):
        m.model.backbone.body["0"](torch.rand(1, 3, 64, 64))
    assert m.training is False
    with pytest.raises((NotImplementedError, _C.NativeLibraryError)):
        yolov5n().train()([torch.rand(3, 64, 64)])


@pytest.mark.parametrize("name,ctor,gflop,n_convs", [("n", yolov5n, 4.468, 60), ("s", yolov5s, 16.434, 60), ("m", yolov5m, 48.872, 82)])
def test_lowering_carries_the_reference_work(name, ctor, gflop, n_convs):
    """SURVEY.md section 8d: conv counts and GFLOP/image at 640x640 measured on the reference modules."""
    from yolort_b200.engine import lower_yolo

    L, x0, heads, _ = lower_yolo(ctor().model, torch.float16, torch.device("cpu"))
    convs = [op for op in L.ops if op.kind == _C.YB_OP_CONV]
    n_c3 = sum(1 for op in convs if op.name.endswith("cv1+cv2"))
    assert len(convs) + n_c3 == n_convs          # each fused cv1||cv2 launch covers two reference convs
    total = sum(op.flops_per_pixel * (640 // op.dst.buf.div) ** 2 // op.pack for op in convs)
    assert total / 1e9 == pytest.approx(gflop, rel=2e-3)
    assert sum(1 for op in L.ops if op.kind == _C.YB_OP_UPSAMPLE2X) == 2
    assert sum(1 for op in L.ops if op.kind == _C.YB_OP_SPP_POOL) == 1


def test_stem_band_weights_reproduce_the_stem_conv():
    """engine.stem_band (kBand kernel variant, the default stem): emulate the kernel's addressing on the CPU -- per output
    super-pixel and filter row, the 6 pixels x 16 channels that are contiguous in the patch (96 B into the left
    neighbour) times the banded weights -- and compare with the plain 3x3/s1/p1 conv over the space-to-depth input."""
    import torch.nn.functional as F

    from yolort_b200.engine import stem_band, stem_superpixel

    g = torch.Generator().manual_seed(0)
    co, H, W = 8, 6, 16
    x = torch.randn(2, 16, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(co, 16, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(co, generator=g, dtype=torch.float64)
    want = F.conv2d(x, w, b, padding=1)                                   # [2, co, H, W]
    wb, bb = stem_band(w, b)
    assert tuple(wb.shape) == (4 * co, 3, 128) and torch.all(wb[:, :, 96:] == 0)
    # patch memory order: NHWC rows of super-pixels (4 pixels x 16 channels = 64 values), zero halo all around
    xs = x.permute(0, 2, 3, 1).reshape(2, H, W // 4, 64)
    padded = torch.zeros(2, H + 2, W // 4 + 2, 64, dtype=torch.float64)
    padded[:, 1:-1, 1:-1] = xs
    flat = padded.reshape(2, H + 2, -1)                                    # one patch row = consecutive super-pixels
    got = torch.zeros(2, H, W // 4, 4 * co, dtype=torch.float64)
    for h in range(H):
        for X in range(W // 4):
            acc = bb.clone()
            for ky in range(3):
                start = X * 64 + 48                                        # 96 bytes (48 fp16) into the LEFT neighbour
                span = flat[:, h + ky, start:start + 96]                   # 6 pixels x 16 channels, contiguous
                acc = acc + span @ wb[:, ky, :96].T
            got[:, h, X] = acc
    got = got.reshape(2, H, W // 4, 4, co).reshape(2, H, W, co).permute(0, 3, 1, 2)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # and it is the same linear map as the dense super-pixel matrix the default path uses
    w_sp, b_sp = stem_superpixel(w, b, 4)
    dense = F.conv2d(xs.permute(0, 3, 1, 2), w_sp, b_sp, padding=1)        # [2, 4co, H, W/4]
    torch.testing.assert_close(dense.permute(0, 2, 3, 1).reshape(2, H, W // 4, 4, co).reshape(2, H, W, co).permute(0, 3, 1, 2),
                               want, rtol=1e-12, atol=1e-12)


def test_stem_variants_of_the_lowering():
    """The banded stem is the default when the band fits in shared memory (4*Cout <= 128: n / s); m / l / x keep the
    dense super-pixel matrix.  No environment variable takes part in the lowering."""
    from yolort_b200.engine import lower_yolo
    from yolort_b200.models import yolov5x

    m = yolov5s().eval()
    L, *_ = lower_yolo(m.model, torch.float16, torch.device("cpu"))
    assert L.ops[0].band and tuple(L.ops[0].weight.shape) == (128, 3, 128) and L.ops[0].pack == 4
    L, *_ = lower_yolo(m.model, torch.float16, torch.device("cpu"), stem_variant="superpixel")
    assert not L.ops[0].band and tuple(L.ops[0].weight.shape) == (128, 9, 64)
    L, *_ = lower_yolo(yolov5x().eval().model, torch.float16, torch.device("cpu"))
    assert not L.ops[0].band and L.ops[0].pack == 4


def test_arena_liveness_reuse_never_overlaps_live_buffers():
    """engine.assign_offsets: with reuse, two buffers whose [first writer, last reader] intervals intersect never
    share bytes; the arena shrinks several-fold (SURVEY.md 7.2.6: 56 GB -> single digits for x batch 64 1280^2)."""
    from yolort_b200.engine import assign_offsets, lower_yolo

    for ctor, N, S in ((yolov5n, 3, 128), (yolov5s, 32, 640), (yolov5m, 16, 1280)):
        L, x0, heads, feats = lower_yolo(ctor().model, torch.float16, torch.device("cpu"))
        keep = list(heads) + [v.buf for v in feats.values()]
        o0, tot0 = assign_offsets(L, x0, keep, N, S, S, reuse=False)
        o1, tot1 = assign_offsets(L, x0, keep, N, S, S, reuse=True)
        n_ops = len(L.ops)
        size = {id(b): (N * (S // b.div) ** 2 * b.C * 2 + 1023) // 1024 * 1024 for b in L.bufs}
        first = {id(b): n_ops for b in L.bufs}
        last = {id(b): -1 for b in L.bufs}
        first[id(x0)] = -1
        for i, op in enumerate(L.ops):
            for v in (op.dst, op.src, op.residual):
                if v is not None:
                    first[id(v.buf)] = min(first[id(v.buf)], i)
                    last[id(v.buf)] = max(last[id(v.buf)], i)
        for b in keep:
            last[id(b)] = n_ops
        for i, a in enumerate(L.bufs):
            assert o1[id(a)] % 1024 == 0 and o1[id(a)] + size[id(a)] <= tot1
            for b in L.bufs[i + 1:]:
                if first[id(a)] <= last[id(b)] and first[id(b)] <= last[id(a)]:
                    assert o1[id(a)] + size[id(a)] <= o1[id(b)] or o1[id(b)] + size[id(b)] <= o1[id(a)], (a.name, b.name)
        assert tot0 == sum(size.values()) and tot1 < 0.35 * tot0, (ctor.__name__, tot0, tot1)


def test_engine_is_dropped_by_parent_load_state_dict_and_to():
    """ADVICE r1: nn.Module.load_state_dict on the YOLOv5 wrapper never calls YOLO.load_state_dict; the prepared
    weights must still be invalidated (post hook), and so must `.to()` / `.half()`."""
    m = yolov5n().eval()
    sentinel = object()
    m.model._engine = sentinel
    m.load_state_dict(m.state_dict())              # through the PARENT
    assert m.model._engine is None
    m.model._engine = sentinel
    m.model.load_state_dict(m.model.state_dict())
    assert m.model._engine is None
    m.model._engine = sentinel
    m.half()
    assert m.model._engine is None


def test_callable_submodules_are_wired_to_their_owner():
    """model.model.backbone / .head execute plan ranges of the owning YOLO (no eager fallback: on the CPU they raise
    the library error, not the 'plan only' error); deepcopy keeps the wiring inside the copy."""
    import copy

    m = yolov5n().eval()
    assert m.model.backbone._yb_owner[0] is m.model and m.model.head._yb_owner[0] is m.model
    m2 = copy.deepcopy(m)
    assert m2.model.backbone._yb_owner[0] is m2.model and m2.model is not m.model
    assert [k for k, _ in m.named_modules()] == [k for k, _ in m2.named_modules()]
    assert not any("_yb_owner" in k for k in m.state_dict())
    with pytest.raises(_C.NativeLibraryError):
        m.model.backbone(torch.rand(1, 3, 64, 64))
    assert m.model.has_hooks() is False
    h = m.model.backbone.register_forward_hook(lambda mod, inp, out: None)
    assert m.model.has_hooks() is True
    h.remove()
    assert m.model.has_hooks() is False


def test_training_mode_contract():
    """Training mode: the head outputs go to a caller-supplied criterion (yolo.py:168-171); without one the call says
    that SetCriterion is out of scope.  On the CPU both stop at the no-fallback error first."""
    m = yolov5n().train()
    with pytest.raises((NotImplementedError, _C.NativeLibraryError)):
        m.model(torch.rand(1, 3, 64, 64), None)


def test_u8_scaling_by_reciprocal_equals_division_after_16bit_rounding():
    """csrc/letterbox.cu copy fast path: fp16 / bf16 of `byte * (1/255)` equals fp16 / bf16 of torch's own
    `byte / 255.0` (yolov5.py:228) for every byte value (the fp32 values differ for 126 of the 256)."""
    v = torch.arange(256, dtype=torch.uint8)
    div = v / 255.0
    mul = v.float() * torch.tensor(1.0 / 255.0, dtype=torch.float32)
    assert torch.equal(div.half(), mul.half()) and torch.equal(div.bfloat16(), mul.bfloat16())
    assert not torch.equal(div, mul)


def _conv_desc(N, H, W, Cin, Cout, k, s, p, res=False):
    import torch

    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_CONV, _C.dtype_code(torch.float16)
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, H, W, Cin, Cin, 4096
    d.Ho, d.Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    d.Cout, d.out_cstride, d.out = Cout, Cout, 4096
    d.ksize, d.stride, d.pad, d.act = k, s, p, _C.YB_ACT_SILU
    d.weight, d.bias = 4096, 4096
    d.Cin_pad = (Cin + 63) // 64 * 64 if Cin > 32 else (Cin + 15) // 16 * 16
    d.Cout_pad = (Cout + 15) // 16 * 16
    if res:
        d.residual, d.res_cstride = 4096, Cout
    return d


def test_conv_config_and_chain_support_are_host_logic():
    """Launch configuration and chained-tail eligibility are decided without a GPU (yb_conv_config,
    yb_conv_chain_supported): the yolov5s batch-32 640x640 layers land where DESIGN.md says."""
    c = _C.conv_config(_conv_desc(32, 80, 80, 64, 64, 3, 1, 1))
    assert c["patch_kernel"] == 1 and c["weights_resident"] == 1 and c["n_tiles"] == 1
    c = _C.conv_config(_conv_desc(32, 40, 40, 128, 128, 3, 1, 1))           # 295 KB of weights: streamed, two tiles per pass
    assert c["patch_kernel"] == 1 and c["weights_resident"] == 0 and c["tiles_per_pass"] == 2 and c["slots"] >= 3
    c = _C.conv_config(_conv_desc(32, 160, 160, 64, 64, 1, 1, 0))
    assert c["patch_kernel"] == 0 and c["weights_resident"] == 1 and c["smem_bytes"] <= 222 * 1024

    def chain(d, cout, k, own, extra=0):
        ch = _C.ConvChain()
        ch.weight, ch.bias, ch.out = 4096, 4096, 4096
        ch.Cout, ch.Cout_pad, ch.K_pad, ch.act, ch.out_cstride, ch.own_C = cout, (cout + 15) // 16 * 16, k, _C.YB_ACT_SILU, cout, own
        if extra:
            ch.extra, ch.extra_C, ch.extra_cstride = 4096, extra, 2 * extra
        ch.store_first = 0 if extra else 1
        d.chain = ctypes.addressof(ch)
        ok = _C.conv_chain_supported(d)
        cfg = _C.conv_config(d) if ok else None
        return ok, cfg

    ok, cfg = chain(_conv_desc(32, 160, 160, 64, 64, 1, 1, 0), 32, 32, 32)                 # cv1||cv2 -> m.0.cv1, c = 32
    assert ok and cfg["chained"] == 1
    ok, cfg = chain(_conv_desc(32, 80, 80, 64, 64, 3, 1, 1, res=True), 128, 128, 64, extra=64)   # m.cv2 -> cv3, c = 64
    assert ok and cfg["chained"] == 1 and cfg["slots"] >= 2
    ok, _ = chain(_conv_desc(32, 40, 40, 128, 128, 3, 1, 1, res=True), 256, 256, 128, extra=128)  # 128 KB of tail weights
    assert not ok
    ok, _ = chain(_conv_desc(32, 20, 20, 512, 512, 1, 1, 0), 256, 256, 256)                # several N tiles
    assert not ok


def _cpu_plan(monkeypatch, ctor, N, H, W, **kw):
    import torch

    from yolort_b200 import engine

    class _NoPlan:                       # the native plan needs a GPU; everything before it is host logic
        def __init__(self, descs, device):
            self.n_ops = len(descs)

    monkeypatch.setattr(_C, "Plan", _NoPlan)
    m = ctor(**kw).eval()
    low = engine.Lowered(m.model, torch.float16, torch.device("cpu"))
    return low, engine.PlanInstance(low, N, H, W)


def _assert_arena_liveness(low, inst):
    """Two different buffers that are live during the same launch never share a byte of the arena (a fused launch keeps
    everything both of its convolutions touch live for its whole duration)."""
    L = low.L
    assert len({b.name for b in L.bufs}) == len(L.bufs)          # `PlanInstance.buffers` is keyed by name
    base = inst.arena.data_ptr()
    rng = {}
    for b in L.bufs:
        t = inst.buffers[b.name]
        lo = t.data_ptr() - base
        rng[b.name] = (lo, lo + t.numel() * t.element_size())
        assert 0 <= lo and rng[b.name][1] <= inst.arena.numel()
    first, last = {}, {}
    for t, grp in enumerate(inst.launch_ops):
        for i in grp:
            op = L.ops[i]
            for v in (op.src, op.dst, op.residual, op.chain_extra if len(grp) == 2 and i == grp[0] else None):
                if v is not None:
                    first.setdefault(v.buf.name, t)
                    last[v.buf.name] = t
    for k in {low.x0.name} | {b.name for b in low.head_bufs} | {v.buf.name for v in low.feats.values()}:
        last[k] = len(inst.launch_ops)
    first[low.x0.name] = -1
    names = [n for n in rng if n in first]
    for a in range(len(names)):
        for b2 in range(a + 1, len(names)):
            na, nb = names[a], names[b2]
            if first[na] <= last[nb] and first[nb] <= last[na]:
                assert not (rng[na][0] < rng[nb][1] and rng[nb][0] < rng[na][1]), (na, first[na], last[na], rng[na], nb, first[nb], last[nb], rng[nb])


@pytest.mark.parametrize("name", ["yolov5n", "yolov5m", "yolov5l", "yolov5x", "yolov5n6", "yolov5s_r40"])
def test_arena_liveness_with_fused_launches_across_the_zoo(monkeypatch, name):
    """The same invariant for the other topologies and widths (different fusion decisions per model: 16 / 48 / 80-channel
    levels are never chained, yolov5l's 64-channel level is), small canvas."""
    import yolort_b200.models as M

    if name == "yolov5s_r40":
        ctor, kw = M.yolov5s, {"upstream_version": "r4.0"}
    else:
        ctor, kw = getattr(M, name), {}
    low, inst = _cpu_plan(monkeypatch, ctor, 2, 256, 256, **kw)
    assert sum(len(g) for g in inst.launch_ops) == len(low.L.ops)
    assert [i for g in inst.launch_ops for i in g] == list(range(len(low.L.ops)))      # every op exactly once, in order
    _assert_arena_liveness(low, inst)
    if name == "yolov5l":
        assert any(len(g) == 2 for g in inst.launch_ops)
    if name in ("yolov5m", "yolov5x"):
        assert all(len(g) == 1 for g in inst.launch_ops)


def test_fused_launch_list_and_arena_liveness_on_cpu(monkeypatch):
    """Host logic of the plan, without a GPU: which convolutions ride as chained tails (yolov5s: the pointwise chains of
    the 32 / 64-channel C3 blocks), and the arena invariant that makes liveness reuse safe with fused launches -- every
    buffer a launch touches (source, destination, shortcut, the tail's second operand and output) is live for the whole
    launch, and two different buffers that are live at the same time never share a byte."""
    import torch

    from yolort_b200 import engine
    from yolort_b200.models import yolov5s

    class _NoPlan:                       # the native plan needs a GPU; everything before it is host logic
        def __init__(self, descs, device):
            self.n_ops = len(descs)

    monkeypatch.setattr(_C, "Plan", _NoPlan)
    m = yolov5s().eval()
    low = engine.Lowered(m.model, torch.float16, torch.device("cpu"))
    N, H, W = 4, 640, 640
    inst = engine.PlanInstance(low, N, H, W)
    L = low.L
    fused = [(L.ops[g[0]].name, L.ops[g[1]].name) for g in inst.launch_ops if len(g) == 2]
    assert len(L.ops) == 55 and len(inst.launch_ops) == 48
    assert fused == [("body.2.cv1+cv2", "body.2.m.0.cv1"), ("body.2.m.0.cv2", "body.2.cv3"),
                     ("body.4.cv1+cv2", "body.4.m.0.cv1"), ("body.4.m.0.cv2", "body.4.m.1.cv1"),
                     ("body.4.m.1.cv2", "body.4.cv3"),
                     ("pan.layer_blocks.0.cv1+cv2", "pan.layer_blocks.0.m.0.cv1"),
                     ("pan.layer_blocks.0.m.0.cv2", "pan.layer_blocks.0.cv3")]
    # byte range of every buffer inside the arena
    base = inst.arena.data_ptr()
    rng = {}
    for b in L.bufs:
        t = inst.buffers[b.name]
        lo = t.data_ptr() - base
        rng[b.name] = (lo, lo + t.numel() * t.element_size())
        assert 0 <= lo and rng[b.name][1] <= inst.arena.numel()
    # live interval of every buffer in launch steps: first writer .. last reader (inputs / results stay live)
    first, last = {}, {}
    for t, grp in enumerate(inst.launch_ops):
        for i in grp:
            op = L.ops[i]
            for v in (op.src, op.dst, op.residual, op.chain_extra if len(grp) == 2 and i == grp[0] else None):
                if v is not None:
                    first.setdefault(v.buf.name, t)
                    last[v.buf.name] = t
    keep = {low.x0.name} | {b.name for b in low.head_bufs} | {v.buf.name for v in low.feats.values()}
    n_steps = len(inst.launch_ops)
    for k in keep:
        last[k] = n_steps
    first[low.x0.name] = -1
    names = [n for n in rng if n in first]
    clashes = 0
    for a in range(len(names)):
        for b2 in range(a + 1, len(names)):
            na, nb = names[a], names[b2]
            overlap_time = first[na] <= last[nb] and first[nb] <= last[na]
            overlap_bytes = rng[na][0] < rng[nb][1] and rng[nb][0] < rng[na][1]
            if overlap_time and overlap_bytes:
                clashes += 1
                print("CLASH", na, first[na], last[na], rng[na], "|", nb, first[nb], last[nb], rng[nb])
    assert clashes == 0
    assert inst.arena_bytes < 0.5 * inst.unshared_bytes        # and the reuse still pays
