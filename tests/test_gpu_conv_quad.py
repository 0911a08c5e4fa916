"""Four consumer warpgroups (128-column pair tasks) of the halo-patch kernel on the H100: every case against fp64, and
every launch that takes them bit-identical to the 64-column pair launch of the same op (reserved bit
YB_CONV_PAIR_N64).  Each output element gets the same k16 MMA sequence (chunk, tap, k) and epilogue either way."""
import dataclasses

import pytest
import torch

import conv_cases
import conv_cases_quad as q
import yolort_b200.models as M
from yolort_b200 import _C

DEV = torch.device("cuda:0")

# c2 (yolov5s batch 32, fp16), c3's model (yolov5m, bf16) and c4 (yolov5l batch 16, fp16)
MODELS = {"yolov5s": ("yolov5s", 32, 640, torch.float16), "yolov5m": ("yolov5m", 128, 640, torch.bfloat16),
          "yolov5l": ("yolov5l", 16, 640, torch.float16)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", q.CASES, ids=lambda c: c.name)
def test_quad_case(case):
    """fp64 bound, untouched surroundings and repeatability (conv_cases.check_case); a four-warpgroup launch also gives
    the bits of the 64-column pair launch."""
    conv_cases.check_case(case)
    d, _ch = conv_cases.build_desc(case, conv_cases.fake_ptr)
    if _C.conv_config(d)["consumer_groups"] != 4:
        return
    t = conv_cases.operands(case, DEV)
    t["out0"] = t["out"].clone()
    out, _ = conv_cases._launch(case, t, DEV)
    pairs = dataclasses.replace(case, reserved=case.reserved | _C.YB_CONV_PAIR_N64)
    o1, _ = conv_cases._launch(pairs, t, DEV)
    assert torch.equal(o1, out), "four-warpgroup launch differs from the 64-column pair launch"


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_quad_launches_match_64_column_pairs_bit_for_bit(model):
    """Every launch of the plan on four consumer warpgroups writes exactly the bytes the 64-column pair launch of the
    same op writes on the same input (the whole arena is compared)."""
    name, N, S, dtype = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(dtype))
    ops = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _C.conv_config(d)["consumer_groups"] == 4]
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
        d1.reserved |= _C.YB_CONV_PAIR_N64
        assert _C.conv_config(d1)["consumer_groups"] == 2
        pairs = _C.Plan([d1], DEV)
        pairs.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: four-warpgroup output differs from the 64-column pairs"
        del pairs
