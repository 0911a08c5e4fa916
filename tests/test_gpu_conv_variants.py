"""Every launch variant of the fp16/bf16 convolution kernels (conv_cases.VARIANTS: two CTAs per SM, one consumer
warpgroup, the split tail, four consumer warpgroups) writes exactly the bits of each of its pinned launches: every case
of the variants' case tables (conv_cases.check_case, which also bounds the case against fp64), and every conv launch of
the benchmark models over the whole arena.  Which model launches take each variant is host logic, checked without a
GPU.  Each output element gets the same k16 MMA sequence and epilogue whichever launch computes it."""
import pytest
import torch

import conv_cases_one_group
import conv_cases_quad
import conv_cases_quad_1x1
import conv_cases_tail_split
import conv_cases_team
import conv_cases_team_1x1
import yolort_b200.models as M
from conv_cases import SMS, VARIANTS, check_case, check_pinned, variants
from yolort_b200 import _C, engine

DEV = torch.device("cuda:0")

# The variants' own case tables; the cases of tests/conv_cases.py go through check_case in tests/test_gpu_conv_cases.py.
TABLES = (conv_cases_one_group, conv_cases_quad, conv_cases_quad_1x1, conv_cases_tail_split, conv_cases_team,
          conv_cases_team_1x1)

# (constructor, batch, canvas side, dtype): the benchmark configurations c2 (yolov5s), c3's model (yolov5m, at the
# global batch of 128 on one GPU and at 16), c4 (yolov5l, the smallest and largest canvas of its mix), yolov5n, whose
# narrow levels take the halo-patch kernel's two-CTA instance, and c5 (yolov5x), whose launches are checked on the host
# only.
MODELS = {
    "yolov5s": ("yolov5s", 32, 640, torch.float16),
    "yolov5m": ("yolov5m", 128, 640, torch.bfloat16),
    "yolov5m_b16": ("yolov5m", 16, 640, torch.bfloat16),
    "yolov5l": ("yolov5l", 16, 640, torch.float16),
    "yolov5l_1280": ("yolov5l", 16, 1280, torch.float16),
    "yolov5n": ("yolov5n", 32, 640, torch.float16),
    "yolov5x_1280": ("yolov5x", 64, 1280, torch.float16),
}
GPU_MODELS = sorted(set(MODELS) - {"yolov5x_1280"})

# The conv launches of each model that take each variant on a 132-SM H100 (the stem and every deep level of a model
# not listed under "2x2" keep one CTA per SM, and so on).
EXPECTED = {
    "yolov5s": {
        "patch team": {"body.0(stem: banded 3x3 over s2d super-pixels)", "body.4.m.0.cv2 -> body.4.m.1.cv1",
            "body.4.m.1.cv2 -> body.4.cv3", "pan.layer_blocks.0.m.0.cv2 -> pan.layer_blocks.0.cv3"},
        "2x2": {"body.1", "body.2.cv1+cv2 -> body.2.m.0.cv1", "body.2.m.0.cv2 -> body.2.cv3"},
        "1x1 team": {"body.4.cv1+cv2 -> body.4.m.0.cv1", "pan.layer_blocks.0.cv1+cv2 -> pan.layer_blocks.0.m.0.cv1"},
        "1x1 quad": {"body.5", "body.7", "body.8.cv1+cv2", "body.8.cv3", "body.8.m.0.cv1", "head.head.2",
            "pan.inner_blocks.0.cv1", "pan.inner_blocks.0.cv2", "pan.inner_blocks.1", "pan.inner_blocks.3.cv1+cv2",
            "pan.layer_blocks.1", "pan.layer_blocks.3", "pan.layer_blocks.4.cv1+cv2", "pan.layer_blocks.4.cv3",
            "pan.layer_blocks.4.m.0.cv1"},
        "2x1": {"body.6.cv1+cv2", "body.6.cv3", "head.head.0", "head.head.1", "pan.inner_blocks.3.cv3",
            "pan.layer_blocks.2.cv1+cv2", "pan.layer_blocks.2.cv3"},
        "split tail": {"body.6.cv1+cv2", "body.6.cv3", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1",
            "head.head.0", "head.head.1", "pan.inner_blocks.3.cv3", "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.4",
            "pan.layer_blocks.2.cv1+cv2", "pan.layer_blocks.2.cv3", "pan.layer_blocks.2.m.0.cv1"},
        "patch quad": {"body.6.m.0.cv2", "body.6.m.1.cv2", "body.6.m.2.cv2", "pan.inner_blocks.3.m.0.cv2",
            "pan.layer_blocks.2.m.0.cv2"},
    },
    "yolov5m": {
        "2x2": {"body.2.m.0.cv1", "body.2.m.1.cv1"},
        "2x1": {"body.4.cv1+cv2", "body.4.cv3", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1", "body.6.m.3.cv1",
            "body.6.m.4.cv1", "body.6.m.5.cv1", "head.head.0", "pan.inner_blocks.3.m.0.cv1",
            "pan.inner_blocks.3.m.1.cv1", "pan.layer_blocks.0.cv3", "pan.layer_blocks.2.m.0.cv1",
            "pan.layer_blocks.2.m.1.cv1"},
        "split tail": {"body.4.m.0.cv1", "body.4.m.1.cv1", "body.4.m.2.cv1", "body.4.m.3.cv1", "body.6.m.0.cv1",
            "body.6.m.1.cv1", "body.6.m.2.cv1", "body.6.m.3.cv1", "body.6.m.4.cv1", "body.6.m.5.cv1",
            "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.3.m.1.cv1", "pan.layer_blocks.0.m.0.cv1",
            "pan.layer_blocks.0.m.1.cv1", "pan.layer_blocks.2.m.0.cv1", "pan.layer_blocks.2.m.1.cv1"},
        "1x1 quad": {"body.7", "body.8.cv1+cv2", "body.8.cv3", "body.8.m.0.cv1", "body.8.m.1.cv1", "head.head.2",
            "pan.inner_blocks.0.cv1", "pan.inner_blocks.0.cv2", "pan.inner_blocks.1", "pan.layer_blocks.3",
            "pan.layer_blocks.4.cv1+cv2", "pan.layer_blocks.4.cv3", "pan.layer_blocks.4.m.0.cv1",
            "pan.layer_blocks.4.m.1.cv1"},
        "patch quad": {"body.8.m.0.cv2", "body.8.m.1.cv2", "pan.layer_blocks.4.m.0.cv2", "pan.layer_blocks.4.m.1.cv2"},
    },
    "yolov5m_b16": {
        "split tail": {"body.2.cv1+cv2", "body.2.cv3", "body.4.cv1+cv2", "body.4.cv3", "body.4.m.0.cv1",
            "body.4.m.1.cv1", "body.4.m.2.cv1", "body.4.m.3.cv1", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1",
            "body.6.m.3.cv1", "body.6.m.4.cv1", "body.6.m.5.cv1", "body.7", "body.8.cv1+cv2", "body.8.cv3",
            "body.8.m.0.cv1", "body.8.m.1.cv1", "head.head.0", "head.head.1", "pan.inner_blocks.0.cv1",
            "pan.inner_blocks.0.cv2", "pan.inner_blocks.1", "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.3.m.1.cv1",
            "pan.inner_blocks.4", "pan.layer_blocks.0.cv3", "pan.layer_blocks.0.m.0.cv1", "pan.layer_blocks.0.m.1.cv1",
            "pan.layer_blocks.1", "pan.layer_blocks.2.m.0.cv1", "pan.layer_blocks.2.m.1.cv1", "pan.layer_blocks.3",
            "pan.layer_blocks.4.cv1+cv2", "pan.layer_blocks.4.cv3", "pan.layer_blocks.4.m.0.cv1",
            "pan.layer_blocks.4.m.1.cv1"},
        "2x2": {"body.2.m.0.cv1", "body.2.m.1.cv1"},
        "2x1": {"body.4.cv1+cv2", "body.4.cv3", "head.head.0", "pan.layer_blocks.0.cv3"},
    },
    "yolov5l": {
        "1x1 team": {"body.2.cv1+cv2 -> body.2.m.0.cv1"},
        "patch team": {"body.2.m.0.cv2 -> body.2.m.1.cv1", "body.2.m.1.cv2 -> body.2.m.2.cv1",
            "body.2.m.2.cv2 -> body.2.cv3"},
        "2x1": {"body.4.cv1+cv2", "body.4.cv3", "head.head.0", "pan.layer_blocks.0.cv3"},
        "split tail": {"body.4.cv1+cv2", "body.4.cv3", "body.4.m.0.cv1", "body.4.m.1.cv1", "body.4.m.2.cv1",
            "body.4.m.3.cv1", "body.4.m.4.cv1", "body.4.m.5.cv1", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1",
            "body.6.m.3.cv1", "body.6.m.4.cv1", "body.6.m.5.cv1", "body.6.m.6.cv1", "body.6.m.7.cv1", "body.6.m.8.cv1",
            "head.head.0", "head.head.1", "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.3.m.1.cv1",
            "pan.inner_blocks.3.m.2.cv1", "pan.inner_blocks.4", "pan.layer_blocks.0.cv3", "pan.layer_blocks.0.m.0.cv1",
            "pan.layer_blocks.0.m.1.cv1", "pan.layer_blocks.0.m.2.cv1", "pan.layer_blocks.1",
            "pan.layer_blocks.2.m.0.cv1", "pan.layer_blocks.2.m.1.cv1", "pan.layer_blocks.2.m.2.cv1"},
        "1x1 quad": {"body.5", "body.6.cv1+cv2", "body.6.cv3", "pan.inner_blocks.3.cv1+cv2", "pan.inner_blocks.3.cv3",
            "pan.layer_blocks.2.cv1+cv2", "pan.layer_blocks.2.cv3"},
        "patch quad": {"body.6.m.0.cv2", "body.6.m.1.cv2", "body.6.m.2.cv2", "body.6.m.3.cv2", "body.6.m.4.cv2",
            "body.6.m.5.cv2", "body.6.m.6.cv2", "body.6.m.7.cv2", "body.6.m.8.cv2", "pan.inner_blocks.3.m.0.cv2",
            "pan.inner_blocks.3.m.1.cv2", "pan.inner_blocks.3.m.2.cv2", "pan.layer_blocks.2.m.0.cv2",
            "pan.layer_blocks.2.m.1.cv2", "pan.layer_blocks.2.m.2.cv2"},
    },
    "yolov5l_1280": {
        "1x1 team": {"body.2.cv1+cv2 -> body.2.m.0.cv1"},
        "patch team": {"body.2.m.0.cv2 -> body.2.m.1.cv1", "body.2.m.1.cv2 -> body.2.m.2.cv1",
            "body.2.m.2.cv2 -> body.2.cv3"},
        "2x1": {"body.4.cv1+cv2", "body.4.cv3", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1", "body.6.m.3.cv1",
            "body.6.m.4.cv1", "body.6.m.5.cv1", "body.6.m.6.cv1", "body.6.m.7.cv1", "body.6.m.8.cv1", "head.head.0",
            "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.3.m.1.cv1", "pan.inner_blocks.3.m.2.cv1",
            "pan.layer_blocks.0.cv3", "pan.layer_blocks.2.m.0.cv1", "pan.layer_blocks.2.m.1.cv1",
            "pan.layer_blocks.2.m.2.cv1"},
        "split tail": {"body.4.cv1+cv2", "body.4.cv3", "body.4.m.0.cv1", "body.4.m.1.cv1", "body.4.m.2.cv1",
            "body.4.m.3.cv1", "body.4.m.4.cv1", "body.4.m.5.cv1", "body.6.m.0.cv1", "body.6.m.1.cv1", "body.6.m.2.cv1",
            "body.6.m.3.cv1", "body.6.m.4.cv1", "body.6.m.5.cv1", "body.6.m.6.cv1", "body.6.m.7.cv1", "body.6.m.8.cv1",
            "head.head.0", "head.head.2", "pan.inner_blocks.3.m.0.cv1", "pan.inner_blocks.3.m.1.cv1",
            "pan.inner_blocks.3.m.2.cv1", "pan.layer_blocks.0.cv3", "pan.layer_blocks.0.m.0.cv1",
            "pan.layer_blocks.0.m.1.cv1", "pan.layer_blocks.0.m.2.cv1", "pan.layer_blocks.2.m.0.cv1",
            "pan.layer_blocks.2.m.1.cv1", "pan.layer_blocks.2.m.2.cv1"},
        "1x1 quad": {"body.8.m.0.cv1", "body.8.m.1.cv1", "body.8.m.2.cv1", "pan.inner_blocks.0.cv1",
            "pan.inner_blocks.1", "pan.layer_blocks.3", "pan.layer_blocks.4.m.0.cv1", "pan.layer_blocks.4.m.1.cv1",
            "pan.layer_blocks.4.m.2.cv1"},
        "patch quad": {"body.8.m.0.cv2", "body.8.m.1.cv2", "body.8.m.2.cv2", "pan.layer_blocks.4.m.0.cv2",
            "pan.layer_blocks.4.m.1.cv2", "pan.layer_blocks.4.m.2.cv2"},
    },
    "yolov5n": {
        "2x2": {"body.1", "body.2.cv1+cv2", "body.2.cv3", "body.2.m.0.cv1", "body.2.m.0.cv2", "body.3",
            "body.4.cv1+cv2 -> body.4.m.0.cv1", "body.4.m.0.cv2", "body.4.m.1.cv1", "body.4.m.1.cv2 -> body.4.cv3",
            "pan.inner_blocks.4", "pan.layer_blocks.0.cv1+cv2 -> pan.layer_blocks.0.m.0.cv1",
            "pan.layer_blocks.0.m.0.cv2 -> pan.layer_blocks.0.cv3"},
        "1x1 quad": {"body.7", "body.8.cv1+cv2", "body.8.cv3", "head.head.2", "pan.inner_blocks.0.cv2",
            "pan.layer_blocks.3", "pan.layer_blocks.4.cv1+cv2", "pan.layer_blocks.4.cv3"},
        "2x1": {"head.head.0", "head.head.1"},
        "split tail": {"head.head.0", "head.head.1"},
    },
    "yolov5x_1280": {
        "2x1": {"body.2.cv1+cv2", "body.2.cv3", "body.4.m.0.cv1", "body.4.m.1.cv1", "body.4.m.2.cv1", "body.4.m.3.cv1",
            "body.4.m.4.cv1", "body.4.m.5.cv1", "body.4.m.6.cv1", "body.4.m.7.cv1", "pan.layer_blocks.0.m.0.cv1",
            "pan.layer_blocks.0.m.1.cv1", "pan.layer_blocks.0.m.2.cv1", "pan.layer_blocks.0.m.3.cv1"},
    },
}


def _pinned(d, bit: int):
    d1 = _C.OpDesc.from_buffer_copy(d)
    d1.reserved |= bit
    return d1


@pytest.mark.parametrize("model", sorted(MODELS))
def test_model_launches_take_the_expected_variants(monkeypatch, model):
    """yb_conv_config puts exactly the expected launches on each variant; each pinning bit plans them on the launch the
    variant names, and two CTAs per SM fit in half of the SM's shared memory."""
    if SMS != 132:
        pytest.skip(f"the expectations are those of a 132-SM H100, this device has {SMS}")

    class _NoPlan:                       # the native plan needs a GPU; everything before it is host logic
        def __init__(self, descs, device):
            self.n_ops = len(descs)

    monkeypatch.setattr(_C, "Plan", _NoPlan)
    name, N, S, dtype = MODELS[model]
    inst = engine.PlanInstance(engine.Lowered(getattr(M, name)().eval().model, dtype, torch.device("cpu")), N, S, S)
    taken = {}
    for d, n in zip(inst._descs, inst.op_names):      # inst owns the chain structs the descriptors point to
        if d.kind != _C.YB_OP_CONV:
            continue
        cfg = _C.conv_config(d)
        for v in variants(cfg):
            taken.setdefault(v, set()).add(n)
            for bit in VARIANTS[v].bits:
                check_pinned(_C.conv_config(_pinned(d, bit)), cfg, v, bit, n)
        if cfg["resident_ctas"] == 2:
            static = 1296 if cfg["patch_kernel"] else 2256         # the kernels' static shared memory (ptxas -v)
            assert cfg["grid"] == 2 * 132 and cfg["smem_bytes"] + static <= 228 * 1024 // 2 - 1024, (n, cfg)
    assert taken == EXPECTED[model]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for t in TABLES for c in t.CASES],
                         ids=[f"{t.__name__}:{c.name}" for t in TABLES for c in t.CASES])
def test_case_matches_pinned_launches(case):
    """fp64 bound, untouched surroundings, repeatability and the bits of every pinned launch, first output and tail
    (conv_cases.check_case)."""
    check_case(case)


@pytest.mark.gpu
@pytest.mark.parametrize("model", GPU_MODELS)
def test_model_launches_match_pinned_launches(model):
    """The plan runs op by op; every conv launch that takes a variant writes exactly the bytes each of its pinned launches
    writes on the same input (the whole arena is compared)."""
    name, N, S, dtype = MODELS[model]
    torch.manual_seed(0)
    m = getattr(M, name)(size=(S, S)).eval().to(DEV)
    if dtype == torch.bfloat16:
        m = m.to(torch.bfloat16)
    plan = m.model.get_plan(N, S, S)
    plan.input.copy_(torch.rand(plan.input.shape, device=DEV).to(plan.input.dtype))
    arena = plan.arena
    compared, unchanged = {}, set()
    for i, d in enumerate(plan._descs):
        taken = variants(_C.conv_config(d)) if d.kind == _C.YB_OP_CONV else []
        if not taken:
            plan.run(i, 1)
            continue
        n = plan.op_names[i]
        torch.cuda.synchronize()
        before = arena.clone()
        plan.run(i, 1)
        torch.cuda.synchronize()
        got = arena.clone()
        if torch.equal(got, before):
            unchanged.add(n)
            assert all(VARIANTS[v].may_keep_arena for v in taken), f"{n} left the arena unchanged"
        for v in taken:
            for bit in VARIANTS[v].bits:
                arena.copy_(before)
                pinned = _C.Plan([_pinned(d, bit)], DEV)
                pinned.run()
                torch.cuda.synchronize()
                assert torch.equal(arena, got), f"{n}: {v} launch differs from its pinned launch (reserved bit {bit:#x})"
                del pinned
            compared.setdefault(v, set()).add(n)
    print({v: len(names) for v, names in compared.items()}, "launches compared;", sorted(unchanged), "unchanged")
    for v, names in compared.items():
        assert names - unchanged, f"no {v} launch changed the arena"
    if SMS == 132:
        assert compared == EXPECTED[model]
