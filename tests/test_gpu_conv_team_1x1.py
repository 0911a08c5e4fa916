"""Two consumer teams (chained 1x1 tiles over one resident weight copy) of the 1x1 / im2col kernel on the H100: every
case against fp64, and every launch that takes them bit-identical to the two-warpgroup launch of the same op (reserved
bit YB_CONV_NO_TEAMS).  Each output element gets the same k16 MMA sequence and epilogue either way."""
import dataclasses

import pytest
import torch

import conv_cases
import conv_cases_team_1x1 as t
import yolort_b200.models as M
from yolort_b200 import _C

DEV = torch.device("cuda:0")

# (model, batch, canvas side, dtype, launches expected on two teams: the C3 cv1 || cv2 -> m.0.cv1 chains at N = 128)
MODELS = {"yolov5s": ("yolov5s", 32, 640, torch.float16, {"body.4.cv1+cv2", "pan.layer_blocks.0.cv1+cv2"}),
          "yolov5l": ("yolov5l", 16, 640, torch.float16, {"body.2.cv1+cv2"}),
          "yolov5l_1280": ("yolov5l", 16, 1280, torch.float16, {"body.2.cv1+cv2"}),
          "yolov5m_bf16": ("yolov5m", 128, 640, torch.bfloat16, set())}


def _is_team(d) -> bool:
    cfg = _C.conv_config(d)
    return not cfg["patch_kernel"] and cfg["consumer_groups"] == 4 and cfg["layout"] == "1x4"


@pytest.mark.gpu
@pytest.mark.parametrize("case", t.CASES, ids=lambda c: c.name)
def test_team_1x1_case(case):
    """fp64 bound, untouched surroundings and repeatability (conv_cases.check_case); a two-team launch also gives the
    bits of the two-warpgroup launch, first output and tail alike."""
    conv_cases.check_case(case)
    d, _ch = conv_cases.build_desc(case, conv_cases.fake_ptr)
    if not _is_team(d):
        return
    ops = conv_cases.operands(case, DEV)
    ops["out0"] = ops["out"].clone()
    out, out2 = conv_cases._launch(case, ops, DEV)
    out, out2 = out.clone(), out2.clone()
    pair = dataclasses.replace(case, reserved=case.reserved | _C.YB_CONV_NO_TEAMS)
    o1, o2 = conv_cases._launch(pair, ops, DEV)
    assert torch.equal(o1, out), "two-team launch differs from the two-warpgroup launch"
    assert torch.equal(o2, out2), "tail output differs"


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_team_1x1_launches_match_two_warpgroups_bit_for_bit(model):
    """Every launch of the plan on two teams writes exactly the bytes the two-warpgroup launch of the same op writes on
    the same input (the whole arena is compared)."""
    name, N, S, dtype, expect = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(plan.input.dtype))
    ops = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _is_team(d)]
    names = {plan.op_names[i].split(" ")[0] for i in ops}
    assert names == expect and len(ops) == len(expect), names
    arena = plan.arena
    for i in ops:
        plan.run(0, i)
        torch.cuda.synchronize()
        before = arena.clone()
        plan.run(i, 1)
        torch.cuda.synchronize()
        got = arena.clone()
        assert not torch.equal(got, before), plan.op_names[i]
        arena.copy_(before)
        d1 = _C.OpDesc.from_buffer_copy(plan._descs[i])
        d1.reserved |= _C.YB_CONV_NO_TEAMS
        assert _C.conv_config(d1)["consumer_groups"] == 2
        pair = _C.Plan([d1], DEV)
        pair.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: two-team output differs from two warpgroups"
        del pair
