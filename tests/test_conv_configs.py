"""Launch configurations of every convolution the plans and the case tables create, without a GPU.

`_C.conv_config` reports how the library launches a convolution: kernel, tiling, residency, pipeline depth, shared
memory, grid and CTAs per SM.  This test records it for
  * every YB_OP_CONV descriptor of every plan that tests/test_plan_fingerprint.py builds (read while the descriptor's
    pointers are live),
  * every case of tests/conv_cases.py and tests/conv_cases_one_group.py,
  * the e4m3 shapes of tests/test_gpu_fp8.py, as host-only descriptors,
and compares them with tests/golden/conv_configs.json.  Identical configurations mean identical launch shapes, so a
change to the host side of the convolution kernels that keeps them cannot move tiling, occupancy or launch shapes.

Unique configurations are stored once; each case lists indices into that table.  `python tests/test_conv_configs.py`
rewrites the golden (at SM count 132, the count the library assumes without a GPU)."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import conv_cases  # noqa: E402
import conv_cases_one_group  # noqa: E402
import test_plan_fingerprint as fingerprints  # noqa: E402
from yolort_b200 import _C  # noqa: E402
from yolort_b200.engine import pack_weight_e4m3  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_configs.json")
PLAN_CASES = fingerprints._cases()


def _config(d):
    """conv_config of `d`, or the library's error for a descriptor it rejects (the forced banded stem of a model whose
    stem does not qualify)."""
    try:
        return _C.conv_config(d)
    except _C.NativeLibraryError as e:
        return {"error": str(e)}


def _plan_configs(case, mp):
    """conv_config of every convolution descriptor the plans of one fingerprint case hand to the library."""
    cfgs = []
    raw_desc = fingerprints._raw_desc

    def record(d):
        if d.kind == _C.YB_OP_CONV:
            cfgs.append(_config(d))
        return raw_desc(d)

    mp.setattr(fingerprints, "_raw_desc", record)
    fingerprints.fingerprint(case, mp)
    return cfgs


def _table_configs(cases):
    out = []
    for c in cases:
        d, _chain = conv_cases.build_desc(c, conv_cases.fake_ptr)
        out.append(_C.conv_config(d))
    return out


def _e4m3_desc(k, s, cin, cout, out, residual, act_code, shape):
    """The descriptor tests/test_gpu_fp8.py::conv_case builds, over never-dereferenced addresses."""
    import test_gpu_fp8 as t8

    N, H, W = shape
    p = k // 2
    wq = pack_weight_e4m3(torch.zeros(cout, cin, k, k, dtype=torch.float64), torch.ones(cout, dtype=torch.float64),
                          torch.device("cpu"))
    esz = 1 if out == "e4m3" else 2
    ptr = conv_cases.fake_ptr
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_CONV, _C.YB_F8E4M3
    d.N, d.H, d.W, d.Cin, d.in_cstride, d.in_ = N, H, W, cin, cin + 2 * t8.PAD, ptr("x") + t8.PAD
    d.Ho, d.Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    d.Cout, d.out_cstride, d.out = cout, cout + 2 * t8.PAD, ptr("out") + t8.PAD * esz
    d.ksize, d.stride, d.pad, d.act = k, s, p, act_code
    d.weight, d.Cout_pad, d.Cin_pad, d.bias = ptr("w"), wq.shape[0], wq.shape[2], ptr("b")
    if residual:
        d.residual, d.res_cstride = ptr("res") + t8.PAD, cout + 2 * t8.PAD
    d.reserved = {"e4m3": 0, "f16": _C.YB_CONV_E4M3_F16_OUT, "bf16": _C.YB_CONV_E4M3_BF16_OUT}[out]
    return d


def _e4m3_configs():
    import test_gpu_fp8 as t8

    return [_C.conv_config(_e4m3_desc(*c)) for c in t8.CASES]


def _cases():
    return PLAN_CASES + ["conv_cases", "conv_cases_one_group", "test_gpu_fp8"]


def configs(case, mp):
    if case == "conv_cases":
        return _table_configs(conv_cases.CASES)
    if case == "conv_cases_one_group":
        return _table_configs(conv_cases_one_group.CASES)
    if case == "test_gpu_fp8":
        return _e4m3_configs()
    return _plan_configs(case, mp)


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _cases())
def test_conv_configs(case, monkeypatch):
    if conv_cases.SMS != 132:
        pytest.skip(f"the golden is recorded at 132 SMs, this device has {conv_cases.SMS}")
    golden = _golden()
    want = [golden["configs"][i] for i in golden["cases"][case]]
    got = configs(case, monkeypatch)
    assert len(got) == len(want), f"{case}: {len(got)} convolutions, the golden has {len(want)}"
    for i, (g, w) in enumerate(zip(got, want)):
        diff = {k: (g.get(k), v) for k, v in sorted(w.items()) if g.get(k) != v}    # keys added later are not compared
        if diff:
            pytest.fail(f"{case}: convolution {i} differs (now, golden): {diff}")


def test_golden_covers_exactly_the_cases():
    assert sorted(_golden()["cases"]) == sorted(_cases())


if __name__ == "__main__":
    _C.lib()
    table, index, cases = [], {}, {}
    with pytest.MonkeyPatch.context() as mp:
        for c in _cases():
            rows = []
            for cfg in configs(c, mp):
                key = json.dumps(cfg, sort_keys=True)
                if key not in index:
                    index[key] = len(table)
                    table.append(cfg)
                rows.append(index[key])
            cases[c] = rows
            print(c, len(rows), "convolutions", flush=True)
    with open(GOLDEN, "w") as f:
        f.write('{\n"configs": [\n' + ",\n".join(json.dumps(t, sort_keys=True, separators=(",", ":")) for t in table)
                + '\n],\n"cases": {\n' + ",\n".join(f"{json.dumps(c)}: {json.dumps(cases[c], separators=(',', ':'))}"
                                                   for c in sorted(cases)) + "\n}\n}\n")
