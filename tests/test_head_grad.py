"""Host logic of the 1x1-convolution weight gradient (yb_conv_wgrad_config / yb_conv_wgrad_workspace_bytes /
yb_conv_wgrad argument checks): the pixel slices of every head shape of the shipped detection architectures cover each
pixel exactly once, in order; workspace sizes follow the configuration; bad arguments are rejected with a message.
No kernel is launched."""
import ctypes

import pytest

import head_grad_cases as HC
from yolort_b200 import _C

BASE = 1 << 20       # fake 16-byte aligned device addresses: nothing here is dereferenced


def problems(shapes, dtype=_C.YB_F16, out_dtype=_C.YB_F32, db=True):
    probs = (_C.WgradProblem * len(shapes))()
    addr = BASE
    for pr, (P, co, ci) in zip(probs, shapes):
        pr.dtype, pr.out_dtype, pr.P, pr.Cout, pr.Cin = dtype, out_dtype, P, co, ci
        pr.dy_stride, pr.x_stride = (co + 15) // 16 * 16, (ci + 7) // 8 * 8
        pr.dy, pr.x, pr.dw = addr, addr + (1 << 30), addr + (2 << 30)
        pr.db = addr + (3 << 30) if db else None
        addr += 1 << 32
    return probs


def last_error():
    return _C.lib().yb_last_error().decode()


CASES = HC.all_head_problems() + HC.edge_problems()


@pytest.mark.parametrize("name,shapes", CASES, ids=[c[0] for c in CASES])
def test_slices_cover_every_pixel_once_in_order(name, shapes):
    cfg = _C.conv_wgrad_config(problems(shapes))
    assert cfg["grid"] == min(cfg["items"], cfg["grid"]) and cfg["grid"] >= 1
    items = 0
    for (P, co, ci), q in zip(shapes, cfg["problems"]):
        L, S = q["slice_len"], q["slices"]
        assert L % cfg["stage_pixels"] == 0 and S >= 1
        bounds = [(s * L, min((s + 1) * L, P)) for s in range(S)]
        assert bounds[0][0] == 0 and bounds[-1][1] == P
        assert all(a < b for a, b in bounds)                              # no empty slice
        assert all(b == a2 for (_, b), (a2, _) in zip(bounds, bounds[1:]))  # contiguous, in order: each pixel once
        assert q["co_tiles"] * cfg["tile_rows"] >= co > (q["co_tiles"] - 1) * cfg["tile_rows"]
        assert q["ci_tiles"] * cfg["tile_cols"] >= ci > (q["ci_tiles"] - 1) * cfg["tile_cols"]
        items += q["co_tiles"] * q["ci_tiles"] * S
    assert cfg["items"] == items


@pytest.mark.parametrize("name,shapes", CASES, ids=[c[0] for c in CASES])
def test_workspace_follows_the_config(name, shapes):
    cfg = _C.conv_wgrad_config(problems(shapes))
    want = 0
    for (P, co, ci), q in zip(shapes, cfg["problems"]):
        width = min((ci + 63) // 64, cfg["tile_cols"] // 64) * 64
        want += q["co_tiles"] * q["ci_tiles"] * q["slices"] * (cfg["tile_rows"] * width + cfg["tile_rows"]) * 4
    assert cfg["workspace_bytes"] == want
    assert cfg["smem_bytes"] <= 227 * 1024
    # the split does not depend on the output dtype or on db
    assert _C.conv_wgrad_config(problems(shapes, out_dtype=_C.YB_BF16, db=False))["problems"] == cfg["problems"]


def _reject(probs, match, n=None):
    n = len(probs) if n is None else n
    info = (ctypes.c_int32 * (8 + 4 * max(n, 1)))()
    assert _C.lib().yb_conv_wgrad_config(probs, n, info) == -1
    assert match in last_error(), last_error()
    assert _C.lib().yb_conv_wgrad_workspace_bytes(probs, n) == 0
    assert _C.lib().yb_conv_wgrad(probs, n, BASE, 1 << 30, None) == -1     # before anything touches the device
    assert match in last_error()


@pytest.mark.parametrize("field,value,match", [
    ("dtype", _C.YB_F32, "dtype must be f16 or bf16"),
    ("dtype", _C.YB_F8E4M3, "dtype must be f16 or bf16"),
    ("out_dtype", _C.YB_U8, "out_dtype must be"),
    ("dy_stride", 260, "multiples of 8"),
    ("x_stride", 132, "multiples of 8"),
    ("dy_stride", 248, "exceeds the dy row stride"),
    ("x_stride", 120, "exceeds the x row stride"),
    ("dy", BASE + 8, "16-byte aligned"),
    ("P", 0, "out of range"),
    ("Cout", 0, "must be positive"),
])
def test_bad_arguments_are_rejected(field, value, match):
    probs = problems([(6400, 255, 128), (1600, 255, 256)])
    for pr in (probs if field in ("dtype", "out_dtype") else probs[1:]):     # the call's dtypes / one bad problem
        setattr(pr, field, value)
    _reject(probs, match)


def test_mixed_dtypes_and_problem_counts_are_rejected():
    probs = problems([(6400, 255, 128), (1600, 255, 256)])
    probs[1].dtype = _C.YB_BF16
    _reject(probs, "every problem")
    _reject(problems([(64, 18, 64)]), "problems", n=0)
    _reject(problems([(64, 18, 64)] * 9), "problems")
