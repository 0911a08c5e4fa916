"""Split tail of the 1x1 / im2col kernel on the H100: every case against fp64, and every launch that splits its last
round bit-identical to the launch that keeps those tiles whole (reserved bit YB_CONV_NO_TAIL_SPLIT).  Only N is split,
so each output element gets the same k16 MMA sequence and epilogue either way."""
import dataclasses

import pytest
import torch

import conv_cases
import conv_cases_tail_split as ts
import yolort_b200.models as M
from yolort_b200 import _C

DEV = torch.device("cuda:0")

# c2 (yolov5s batch 32, fp16), c3's model (yolov5m, bf16) and yolov5n
MODELS = {"yolov5s": ("yolov5s", 32, 640, torch.float16), "yolov5m": ("yolov5m", 128, 640, torch.bfloat16),
          "yolov5n": ("yolov5n", 32, 640, torch.float16)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ts.CASES, ids=lambda c: c.name)
def test_tail_split_case(case):
    """fp64 bound, untouched surroundings and repeatability (conv_cases.check_case); a split launch also gives the bits
    of the whole-tile launch."""
    conv_cases.check_case(case)
    d, _ch = conv_cases.build_desc(case, conv_cases.fake_ptr)
    if _C.conv_config(d)["tail_split"] < 2:
        return
    t = conv_cases.operands(case, DEV)
    t["out0"] = t["out"].clone()
    out, _ = conv_cases._launch(case, t, DEV)
    whole = dataclasses.replace(case, reserved=case.reserved | _C.YB_CONV_NO_TAIL_SPLIT)
    o1, _ = conv_cases._launch(whole, t, DEV)
    assert torch.equal(o1, out), "split-tail launch differs from the whole-tile launch"


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_split_launches_match_whole_tiles_bit_for_bit(model):
    """Every launch of the plan that splits its last round writes exactly the bytes the whole-tile launch of the same op
    writes on the same input (the whole arena is compared)."""
    name, N, S, dtype = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(dtype))
    ops = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _C.conv_config(d)["tail_split"] > 1]
    assert ops
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
        d1.reserved |= _C.YB_CONV_NO_TAIL_SPLIT
        assert _C.conv_config(d1)["tail_split"] == 1
        whole = _C.Plan([d1], DEV)
        whole.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: split-tail output differs from the whole-tile launch"
        del whole
