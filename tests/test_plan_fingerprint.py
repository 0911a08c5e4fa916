"""Descriptor fingerprints of the plans, without a GPU: the exact bytes every plan hands to the native library.

Each case builds one family's plans on the CPU with `_C.Plan` replaced by a recorder, serializes every `yb_op_desc`
field by field (with the `yb_conv_chain` and `yb_head_decode` it points to), and compares a digest with the one stored
in tests/golden/plan_fingerprints.json.  Pointers are replaced by what they point at: arena offsets, the owning op and
field of a weight or bias plus a sha256 of its bytes, offsets in the NMS workspace, or the role of a caller's tensor.
Identical fingerprints mean identical launches, so a change to how plans are built that keeps them cannot change what
the GPU computes or how fast.

Besides the digest, the golden keeps one short digest per serialized item (a launch, or the plan's metadata) and one
per field across all items, so that a mismatch names the first differing launch and the fields that differ.

`python tests/test_plan_fingerprint.py` rewrites the golden."""
import ctypes
import contextlib
import hashlib
import json
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from yolort_b200 import _C, engine  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "plan_fingerprints.json")
CPU = torch.device("cpu")

_DESC_PTRS = ("in_", "out", "weight", "bias", "residual")
_CHAIN_PTRS = ("weight", "bias", "out", "extra")
_DECODE_PTRS = ("keys", "boxes", "img_count", "img_maxc")


def _struct(s, prefix=""):
    out = {}
    for name, _ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, ctypes.Array):
            v = list(v)
        out[prefix + name] = v
    return out


def _raw_desc(d):
    """Field values of one descriptor, with the chain and decode blocks read now (they may not outlive the plan)."""
    r = _struct(d)
    chain, decode = r.pop("chain"), r.pop("decode")
    r["chain"] = None if not chain else _struct(_C.ConvChain.from_address(chain))
    r["decode"] = None if not decode else _struct(_C.HeadDecode.from_address(decode))
    if r["kind"] == _C.YB_OP_QUANTIZE and r["bias"]:
        r["bias.value"] = ctypes.c_float.from_address(r["bias"]).value      # fp32 {1/s}
    return r


class _Recorder:
    """Stands in for `_C.Plan`: records the descriptors it is given; run() does nothing."""
    log = None

    def __init__(self, descs, device):
        self.n_ops = len(descs)
        self.descs = [_raw_desc(d) for d in descs]
        _Recorder.log.append(self)

    def run(self, first=0, count=None):
        pass


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes()).hexdigest()[:16]


class _Symbols:
    """Maps raw pointers to symbols."""

    def __init__(self):
        self.ranges = []          # (start, end, kind, label, tensor or None)
        self._sha = {}

    def add(self, t, kind, label, hashed=True):
        if t is None:
            return
        p = t.data_ptr()
        self.ranges.append((p, p + t.numel() * t.element_size(), kind, label, t if hashed else None))

    def __call__(self, p, field):
        if not p:
            return None
        for lo, hi, kind, label, t in self.ranges:
            if lo <= p < hi:
                if kind == "arena" or kind == "nms_ws":
                    return [kind, p - lo]
                if t is not None:
                    key = (lo, hi)
                    if key not in self._sha:
                        self._sha[key] = _sha(t)
                    return [kind, label, p - lo, self._sha[key]]
                return [kind, label, p - lo]
        return ["tensor", field]


def _symbols(low, inst, extra, dgrad):
    s = _Symbols()
    s.add(inst.arena, "arena", None, hashed=False)
    if inst.fused_post is not None:
        s.add(inst.fused_post.ws, "nms_ws", None, hashed=False)
    for i, op in enumerate(low.L.ops):
        s.add(op.weight, "op", [i, "weight"])
        s.add(op.bias, "op", [i, "bias"])
    if dgrad:
        for lvl, (w, b) in enumerate(engine.head_dgrad_weights(low)):
            s.add(w, "head_dgrad", [lvl, "weight"])
            s.add(b, "head_dgrad", [lvl, "bias"])
    for role, t in extra:
        s.add(t, "tensor", role, hashed=False)
    return s


def _launch(raw, sym):
    """Readable serialization of one recorded descriptor: {field: value} with symbolic pointers."""
    out = {}
    for k, v in raw.items():
        if k in ("chain", "decode"):
            continue
        out[k] = sym(v, k) if k in _DESC_PTRS else v
    if raw["chain"] is not None:
        for k, v in raw["chain"].items():
            out["chain." + k] = sym(v, "chain." + k) if k in _CHAIN_PTRS else v
    if raw["decode"] is not None:
        for k, v in raw["decode"].items():
            out["decode." + k] = sym(v, "decode." + k) if k in _DECODE_PTRS else v
    return out


def _plan_meta(inst):
    base = inst.arena.data_ptr()
    return {"launch_ops": [list(g) for g in inst.launch_ops], "op_names": list(inst.op_names),
            "op_flops": list(inst.op_flops), "arena_bytes": inst.arena_bytes, "unshared_bytes": inst.unshared_bytes,
            "front_ops": inst.front_ops, "front_chunks": inst.front_chunks,
            "buffers": {k: t.data_ptr() - base for k, t in inst.buffers.items()}}


# ---------------------------------------------------------------------------------------------------------------------
# models and cases
# ---------------------------------------------------------------------------------------------------------------------
DETECTORS = [("yolov5n", "r6.0"), ("yolov5s", "r6.0"), ("yolov5m", "r6.0"), ("yolov5l", "r6.0"), ("yolov5x", "r6.0"),
             ("yolov5n6", "r6.0"), ("yolov5s", "r3.1"), ("yolov5s", "r4.0")]


def _model(family):
    """(module the engine lowers, the YOLO module with post_config() or None) of a named family, deterministic."""
    if family == "yolov5ts":
        import test_ts
        from yolort_b200.models import yolov5ts

        m = yolov5ts().eval()
        m.load_state_dict(test_ts._sd())
        return m.model, m.model
    if family == "yolov5_mobilenet_v3_small_fpn":
        import test_lite

        m = test_lite._new().eval()
        m.load_state_dict(test_lite._sd())
        return m, m
    if family.startswith("darknet_"):
        import test_darknet
        from yolort_b200.models import darknet

        m = getattr(darknet, family)().eval()
        m.load_state_dict(test_darknet._sd(family))
        return m, None
    import test_fp8

    ctor, version = family.split("@")
    m = test_fp8._model(ctor, version)
    return m.model, m.model


def _cases():
    cases = []
    common = ["default", "keep_intermediates", "chunked", "no_chains"]
    stems = ["stem_band", "stem_superpixel", "stem_im2col"]
    heads = ["fused_decode", "head_dgrad"]
    for ctor, version in DETECTORS:
        for cfg in common + stems + heads:
            if not (ctor == "yolov5x" and cfg == "stem_band"):      # the banded stem needs 4 * Cout <= 256
                cases.append(f"{ctor}@{version}/float16/{cfg}")
    for cfg in common + stems + heads:
        cases.append(f"yolov5s@r6.0/bfloat16/{cfg}")
    for family in ("yolov5ts", "yolov5_mobilenet_v3_small_fpn"):
        for cfg in common + heads:
            cases.append(f"{family}/float16/{cfg}")
    for family in ("darknet_s_r4_0", "darknet_n_r6_0"):
        for cfg in common + stems:
            cases.append(f"{family}/float16/{cfg}")
    for cfg in ("default", "keep_intermediates", "chunked", "quantize_feature"):
        cases.append(f"yolov5s@r6.0/fp8/{cfg}")
    return cases


_MODELS = {}


def _model_cached(family):
    if family not in _MODELS:
        _MODELS.clear()            # cases of one family are consecutive: keep one model at a time
        _MODELS[family] = _model(family)
    return _MODELS[family]


def fingerprint(case, mp):
    """[(item key, {field: value})] of one case."""
    family, dt, cfg = case.split("/")
    net, yolo = _model_cached(family)
    dtype = torch.bfloat16 if dt == "bfloat16" else torch.float16
    log = []
    mp.setattr(_Recorder, "log", log)
    mp.setattr(_C, "Plan", _Recorder)
    mp.setattr(_C, "device_guard", lambda device: contextlib.nullcontext())
    fp8 = None
    if dt == "fp8":
        import test_fp8

        L = engine.lower_yolo(net, dtype, CPU, fp8=True)[0]
        fp8 = types.SimpleNamespace(amax=test_fp8._amax(L))
    stem = cfg[len("stem_"):] if cfg.startswith("stem_") else "auto"
    low = engine.Lowered(net, dtype, CPU, stem, fp8=fp8)
    N, H, W = (16, 320, 320) if cfg == "chunked" else (2, 256, 256)
    kw = {"keep_intermediates": cfg == "keep_intermediates", "chunked": cfg == "chunked",
          "fuse_chains": cfg != "no_chains"}
    if cfg == "fused_decode":
        kw["post"] = yolo.post_config()
    inst = engine.PlanInstance(low, N, H, W, **kw)
    items = [("meta", _plan_meta(inst))]
    extra = []
    if cfg == "chunked":
        assert inst.front_chunks == 4
        for k in range(inst.front_chunks):
            inst.run_front_chunk(k)
    if cfg == "head_dgrad":
        convs = low.head_convs()
        assert convs is not None
        for lvl, (b, conv) in enumerate(zip(low.head_bufs, convs)):
            g = engine.head_dgrad(low, lvl, N, H // b.div, W // b.div, conv.in_channels)
            extra += [(f"dgrad{lvl}.dy", g.dy), (f"dgrad{lvl}.dx", g.dx)]
    if cfg == "quantize_feature":
        key = "p4"
        x = torch.linspace(-3, 3, inst.features[key].numel(), dtype=dtype).view(inst.features[key].shape)
        extra.append(("quantize.x", x))
        inst.quantize_feature(key, x)
    sym = _symbols(low, inst, extra, dgrad=cfg == "head_dgrad")
    names = {id(inst.plan): "plan"}
    if inst.plan_fused is not None:
        names[id(inst.plan_fused)] = "plan_fused"
    assert (inst.plan_fused is not None) == (cfg == "fused_decode")
    for n, p in enumerate(log):
        tag = names.get(id(p), f"log{n}")
        for j, raw in enumerate(p.descs):
            items.append((f"{tag}[{j}]", _launch(raw, sym)))
    items.append(("plans", {"n": len(log), "sizes": [p.n_ops for p in log]}))
    return items


def _h(obj, n=16):
    return hashlib.sha256(json.dumps(obj, separators=(",", ":")).encode()).hexdigest()[:n]


def digests(items):
    fields = {}
    for key, rec in items:
        for f, v in rec.items():
            fields.setdefault(f, []).append([key, v])
    return {"sha": _h(items, 64), "items": [_h([key, rec], 10) for key, rec in items],
            "fields": {f: _h(v, 10) for f, v in sorted(fields.items())}}


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _cases())
def test_plan_fingerprint(case, monkeypatch):
    want = _golden()[case]
    items = fingerprint(case, monkeypatch)
    got = digests(items)
    if got["sha"] == want["sha"]:
        return
    bad_fields = sorted(f for f in set(got["fields"]) | set(want["fields"])
                        if got["fields"].get(f) != want["fields"].get(f))
    for i, h in enumerate(got["items"]):
        if i >= len(want["items"]) or want["items"][i] != h:
            key, rec = items[i]
            if key == "meta":
                rec = {k: rec[k] for k in bad_fields if k in rec}
            pytest.fail(f"{case}: first differing item: {key}; fields that differ: {bad_fields}; "
                        f"now: {json.dumps(rec)[:4000]}")
    pytest.fail(f"{case}: {len(want['items']) - len(got['items'])} fewer items than the golden; fields that differ: "
                f"{bad_fields}")


def test_golden_covers_exactly_the_cases():
    assert sorted(_golden()) == sorted(_cases())


if __name__ == "__main__":
    import __graft_entry__  # noqa: F401   (puts the repository root on sys.path)

    _C.lib()
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        for c in _cases():
            out[c] = digests(fingerprint(c, mp))
            print(c, out[c]["sha"][:16], flush=True)
    with open(GOLDEN, "w") as f:
        f.write("{\n" + ",\n".join(f"{json.dumps(c)}: {json.dumps(out[c], sort_keys=True, separators=(',', ':'))}"
                                    for c in sorted(out)) + "\n}\n")
