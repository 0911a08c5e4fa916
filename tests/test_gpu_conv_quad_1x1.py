"""Two-tile tasks over one streamed weight slab (four consumer warpgroups) of the 1x1 / im2col kernel on the H100: every
case against fp64, and every launch that takes them bit-identical to the two-warpgroup launch of the same op (reserved
bit YB_CONV_PAIR_N64).  Each output element gets the same k16 MMA sequence and epilogue either way."""
import dataclasses

import pytest
import torch

import conv_cases
import conv_cases_quad_1x1 as t
import yolort_b200.models as M
from yolort_b200 import _C

DEV = torch.device("cuda:0")

# (model, batch, canvas side, dtype, least number of launches expected on two-tile tasks)
MODELS = {"yolov5s": ("yolov5s", 32, 640, torch.float16, 15),
          "yolov5m_bf16": ("yolov5m", 128, 640, torch.bfloat16, 14),
          "yolov5l": ("yolov5l", 16, 640, torch.float16, 7),
          "yolov5l_1280": ("yolov5l", 16, 1280, torch.float16, 9)}


def _is_quad(d) -> bool:
    cfg = _C.conv_config(d)
    return not cfg["patch_kernel"] and cfg["consumer_groups"] == 4 and cfg["tiles_per_pass"] == 2


@pytest.mark.gpu
@pytest.mark.parametrize("case", t.CASES, ids=lambda c: c.name)
def test_quad_1x1_case(case):
    """fp64 bound, untouched surroundings and repeatability (conv_cases.check_case); a quad launch also gives the bits
    of the two-warpgroup launch."""
    conv_cases.check_case(case)
    d, _ch = conv_cases.build_desc(case, conv_cases.fake_ptr)
    if not _is_quad(d):
        return
    ops = conv_cases.operands(case, DEV)
    ops["out0"] = ops["out"].clone()
    out, _ = conv_cases._launch(case, ops, DEV)
    out = out.clone()
    pair = dataclasses.replace(case, reserved=case.reserved | _C.YB_CONV_PAIR_N64)
    o1, _ = conv_cases._launch(pair, ops, DEV)
    assert torch.equal(o1, out), "quad launch differs from the two-warpgroup launch"


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_quad_1x1_launches_match_two_warpgroups_bit_for_bit(model):
    """Every launch of the plan on two-tile tasks writes exactly the bytes the two-warpgroup launch of the same op writes
    on the same input (the whole arena is compared)."""
    name, N, S, dtype, least = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(plan.input.dtype))
    ops = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _is_quad(d)]
    assert len(ops) >= least, [plan.op_names[i] for i in ops]
    arena = plan.arena
    changed = 0
    for i in ops:
        plan.run(0, i)
        torch.cuda.synchronize()
        before = arena.clone()
        plan.run(i, 1)
        torch.cuda.synchronize()
        got = arena.clone()
        changed += not torch.equal(got, before)   # a deep layer of an untrained model may rewrite the same bytes
        arena.copy_(before)
        d1 = _C.OpDesc.from_buffer_copy(plan._descs[i])
        d1.reserved |= _C.YB_CONV_PAIR_N64
        assert _C.conv_config(d1)["consumer_groups"] == 2
        pair = _C.Plan([d1], DEV)
        pair.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: quad output differs from two warpgroups"
        del pair
    assert changed or not ops, "no quad launch changed the arena"
