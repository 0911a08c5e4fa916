"""Two CTAs per SM for the shallow convolution launches: which launches of the benchmark models take it (host logic,
no GPU needed) and, on the H100, bit-identical outputs against the one-CTA launch of the same op (YB_CONV_ONE_CTA) on
the same input -- the per-tile arithmetic and summation order do not depend on how many CTAs share an SM."""
import pytest
import torch

import yolort_b200.models as M
from yolort_b200 import _C, engine

DEV = torch.device("cuda:0")

# (constructor, batch, canvas, dtype, launches expected on two CTAs per SM): the benchmark configurations c2 (yolov5s),
# c3 (yolov5m, global batch 128 on one GPU), c4 (yolov5l, the smallest and largest canvas of its mix), c5 (yolov5x),
# and yolov5n, whose narrow levels also take the halo-patch kernel's two-CTA instance
CASES = {
    "c2": ("yolov5s", 32, 640, torch.float16, {"body.1", "body.2.cv1+cv2 -> body.2.m.0.cv1",
                                               "body.2.m.0.cv2 -> body.2.cv3"}),
    "c3": ("yolov5m", 128, 640, torch.bfloat16, {"body.2.m.0.cv1", "body.2.m.1.cv1"}),
    "c4_640": ("yolov5l", 16, 640, torch.float16, set()),
    "c4_1280": ("yolov5l", 16, 1280, torch.float16, set()),
    "c5": ("yolov5x", 64, 1280, torch.float16, set()),
    "n": ("yolov5n", 32, 640, torch.float16, {
        "body.1", "body.2.cv1+cv2", "body.2.m.0.cv1", "body.2.m.0.cv2", "body.2.cv3", "body.3",
        "body.4.cv1+cv2 -> body.4.m.0.cv1", "body.4.m.0.cv2", "body.4.m.1.cv1", "body.4.m.1.cv2 -> body.4.cv3",
        "pan.inner_blocks.4", "pan.layer_blocks.0.cv1+cv2 -> pan.layer_blocks.0.m.0.cv1",
        "pan.layer_blocks.0.m.0.cv2 -> pan.layer_blocks.0.cv3"}),
}


def _ctas(d) -> int:
    return _C.conv_config(d)["ctas_per_sm"]


@pytest.mark.parametrize("case", sorted(CASES))
def test_two_ctas_per_sm_where_the_shape_selects_it(monkeypatch, case):
    """yb_conv_config reports two CTAs per SM for exactly the expected launches: the stem and every deep level keep
    one; reserved bit 4 brings every launch back to one."""
    name, N, S, dtype, expected = CASES[case]

    class _NoPlan:                       # the native plan needs a GPU; everything before it is host logic
        def __init__(self, descs, device):
            self.n_ops = len(descs)

    monkeypatch.setattr(_C, "Plan", _NoPlan)
    low = engine.Lowered(getattr(M, name)().eval().model, dtype, torch.device("cpu"))
    inst = engine.PlanInstance(low, N, S, S)
    convs = [(d, n) for d, n in zip(inst._descs, inst.op_names) if d.kind == _C.YB_OP_CONV]
    two = {n for d, n in convs if _ctas(d) == 2}
    assert two == expected
    assert _ctas(convs[0][0]) == 1                                           # the stem
    assert all(_ctas(d) == 1 for d, n in convs if n.startswith(("body.6", "body.8", "head.")))
    for d, n in convs:
        if n in two:
            cfg = _C.conv_config(d)
            static = 1296 if cfg["patch_kernel"] else 2256         # the kernels' static shared memory (ptxas -v)
            assert cfg["grid"] == 2 * 132 and cfg["smem_bytes"] + static <= 228 * 1024 // 2 - 1024
            d1 = _C.OpDesc.from_buffer_copy(d)
            d1.reserved |= _C.YB_CONV_ONE_CTA
            one = _C.conv_config(d1)
            assert one["ctas_per_sm"] == 1 and one["grid"] == 132 and one["chained"] == cfg["chained"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c2", "c3", "n"])
def test_two_cta_launches_match_one_cta_bit_for_bit(case):
    """Every launch of the plan that runs on two CTAs per SM writes exactly the bytes the one-CTA launch of the same op
    writes on the same input (the whole arena is compared)."""
    name, N, S, dtype, expected = CASES[case]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(dtype))
    two = [i for i, d in enumerate(plan._descs) if d.kind == _C.YB_OP_CONV and _ctas(d) == 2]
    assert {plan.op_names[i] for i in two} == expected
    arena = plan.arena
    for i in two:
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
        assert _ctas(d1) == 1
        one = _C.Plan([d1], DEV)
        one.run()
        torch.cuda.synchronize()
        assert torch.equal(arena, got), f"{plan.op_names[i]}: two-CTA output differs from the one-CTA launch"
        del one
