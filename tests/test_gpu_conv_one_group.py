"""Two CTAs per SM of one consumer warpgroup each (64-row tiles) for the 1x1 / im2col kernel: which launches of the
benchmark models take it (host logic), and on the H100 every case against fp64 and every such launch bit-identical to
the one-CTA launch of the same op (reserved bit 4): each warpgroup keeps its 64 rows, its MMA sequence and its
epilogue, whichever CTA it belongs to."""
import dataclasses

import pytest
import torch

import conv_cases
import conv_cases_one_group as og
import yolort_b200.models as M
from yolort_b200 import _C, engine

DEV = torch.device("cuda:0")

# the c2 launches (yolov5s, batch 32, 640², fp16) planned on the one-group layout
C2_ONE_GROUP = {
    "body.6.cv1+cv2", "body.6.cv3", "pan.inner_blocks.3.cv3", "pan.layer_blocks.2.cv1+cv2", "pan.layer_blocks.2.cv3",
    "head.head.0", "head.head.1",
}

MODELS = {"yolov5s": ("yolov5s", 32, 640, torch.float16), "yolov5m": ("yolov5m", 16, 640, torch.bfloat16),
          "yolov5n": ("yolov5n", 32, 640, torch.float16)}


def _layout(d) -> str:
    return _C.conv_config(d)["layout"]


def test_c2_launches_on_the_one_group_layout(monkeypatch):
    """The rule (a 256-column N tile in the one-CTA plan, no chained tail, at least 3 x SMs 128-row tiles, weights
    resident as two 128-column N tiles, a plan in half the SM's shared memory) picks exactly these c2 launches: the
    40² and 80² layers with 256 output channels."""
    class _NoPlan:                       # the native plan needs a GPU; everything before it is host logic
        def __init__(self, descs, device):
            self.n_ops = len(descs)

    monkeypatch.setattr(_C, "Plan", _NoPlan)
    low = engine.Lowered(M.yolov5s().eval().model, torch.float16, torch.device("cpu"))
    inst = engine.PlanInstance(low, 32, 640, 640)
    convs = [(d, n) for d, n in zip(inst._descs, inst.op_names) if d.kind == _C.YB_OP_CONV]
    assert {n for d, n in convs if _layout(d) == "2x1"} == C2_ONE_GROUP
    for d, n in convs:
        if n in C2_ONE_GROUP:
            cfg = _C.conv_config(d)
            assert cfg["grid"] == 2 * 132 and cfg["epilogue_groups"] == 1 and cfg["smem_bytes"] + 2256 <= 228 * 1024 // 2 - 1024


@pytest.mark.gpu
@pytest.mark.parametrize("case", og.CASES, ids=lambda c: c.name)
def test_one_group_case(case):
    """fp64 bound, untouched surroundings and repeatability (conv_cases.check_case); a one-group launch also gives the
    bits of its one-CTA launch."""
    d, _ch = conv_cases.build_desc(case, conv_cases.fake_ptr)
    assert _layout(d) == case.name.split()[1]
    conv_cases.check_case(case)
    if _layout(d) != "2x1":
        return
    t = conv_cases.operands(case, DEV)
    t["out0"] = t["out"].clone()
    stored = case if case.chain is None else dataclasses.replace(case, chain=dataclasses.replace(case.chain, store_first=True))
    out, out2 = conv_cases._launch(stored, t, DEV)
    one = dataclasses.replace(stored, reserved=stored.reserved | _C.YB_CONV_ONE_CTA)
    o1, o21 = conv_cases._launch(one, t, DEV)
    assert torch.equal(o1, out), "one-group launch differs from the one-CTA launch"
    if case.chain is not None:
        assert torch.equal(o21, out2), "one-group tail differs from the one-CTA launch"


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_one_group_launches_match_one_cta_bit_for_bit(model):
    """Every launch of the plan on the one-group layout writes exactly the bytes the one-CTA launch of the same op
    writes on the same input (the whole arena is compared)."""
    name, N, S, dtype = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(dtype))
    ops = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _layout(d) == "2x1"]
    assert ops
    if model == "yolov5s":
        assert {plan.op_names[i] for i in ops} == C2_ONE_GROUP
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
        d1.reserved |= _C.YB_CONV_ONE_CTA
        assert _layout(d1) == "1x2"
        one = _C.Plan([d1], DEV)
        one.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: one-group output differs from the one-CTA launch"
        del one
