"""The training loss on the device (yolort_b200.models.box_head.SetCriterion, csrc/yolo_loss.cu): the assignment
bit-identical to the reference's fixtures (tests/golden/loss.npz) and the restatement, losses and gradients within
the stated bounds in fp32 / fp16 / bf16, at the fixture shapes and at yolov5s / yolov5x6 training shapes; repeated calls
bit-identical; autograd; the YOLO training path; invalid device targets."""
import json
import os

import numpy as np
import pytest
import torch

import loss_cases as LC
from oracle import restate_loss as R
from yolort_b200 import _C
from yolort_b200.models.box_head import SetCriterion

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "loss.npz"))
with open(os.path.join(os.path.dirname(__file__), "golden", "loss.json")) as _f:
    META = json.load(_f)
CASES = LC.cases()
KEYS = ("cls_logits", "bbox_regression", "objectness")
SCALE = 65536.0
LOSS_RTOL = 1e-5
G_RTOL, G_ATOL = 2e-5, 2e-7     # |got - want| <= G_RTOL |want| + G_ATOL max|want|, per level (measured: <= 0.62 of it)


def device_loss(crit, targets, heads, grad=1.0):
    """Losses (fp64 numpy [3]) and d(sum of grad * losses) / d heads."""
    heads = [h.detach().to(DEV).requires_grad_(True) for h in heads]
    out = crit(targets, heads)
    assert list(out) == list(KEYS) and all(v.shape == (1,) and v.dtype == torch.float32 for v in out.values())
    gs = torch.autograd.grad([out[k] for k in KEYS], heads,
                             [torch.full((1,), grad, device=DEV) for _ in KEYS], allow_unused=True)
    gs = [torch.zeros_like(h) if g is None else g for g, h in zip(gs, heads)]
    return np.array([float(out[k].detach()) for k in KEYS]), gs


def device_matches(crit, targets, heads):
    heads = [h.to(DEV).contiguous() for h in heads]
    params = crit._params(int(heads[0].shape[0]))
    levels = _C.yolo_loss_levels(heads, crit.strides, crit.anchor_grids)
    t = targets.to(DEV).float().contiguous()
    _, status, ws = _C.yolo_loss_forward(params, levels, t, torch.device(DEV))
    rec, bounds = _C.yolo_loss_matches(params, levels, int(t.shape[0]), ws)
    assert int(status.item()) == 0
    out = []
    for l in range(len(heads)):
        r = rec[bounds[l]: bounds[l + 1]]
        assert torch.all(r[:, 0] == l)
        out.append({"idx": r[:, [1, 2, 3, 4, 5]].to(torch.int64).numpy(), "tbox": r[:, 8:12].numpy().copy(),
                    "anchor": r[:, 12:14].numpy().copy()})
    return out


def assert_losses(got, want, what):
    want = np.asarray(want, np.float64)
    assert np.all(np.abs(got - want) <= LOSS_RTOL * np.abs(want)), (what, got, want)


def _t64(x):
    return (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))).to(DEV, torch.float64)


def assert_grad(got, want, what):
    """|got - want| <= G_RTOL |want| + G_ATOL max|want| (on the device: the training shapes hold 10^8 values)."""
    got, want = _t64(got), _t64(want)
    if not want.numel():
        return
    bound = G_RTOL * want.abs() + G_ATOL * want.abs().max()
    excess = float(((got - want).abs() - bound).max())
    print(f"grad {what}: max(err - bound) {excess:.3e}, max rel {float(((got - want).abs() / bound).max()):.3e}")
    assert excess <= 0.0, (what, excess)


def ulp(r: torch.Tensor) -> torch.Tensor:
    """One unit in the last place of each value of a fp16 / bf16 tensor (subnormals included), fp64."""
    info = torch.finfo(r.dtype)
    mant = {torch.float16: 10, torch.bfloat16: 7}[r.dtype]
    e = torch.floor(torch.log2(r.double().abs().clamp(min=info.tiny)))
    return torch.clamp(torch.exp2(e - mant), min=info.smallest_normal * 2.0 ** -mant)


def assert_within_one_ulp(got: torch.Tensor, want64, what):
    r = _t64(want64).to(got.dtype)
    err = (got.to(DEV).double() - r.double()).abs()
    worst = float((err / ulp(r)).max()) if err.numel() else 0.0
    print(f"ulp {what}: worst {worst:.3f} ulp")
    assert worst <= 1.0, (what, worst)


def fixture_grads(name, k, l):
    return GOLD[f"{name}/{k}/{l}/grad"], GOLD[f"{name}/{k}/{l}/dense"]


def gathered(g, idx):
    b, a, gj, gi = (torch.from_numpy(idx[:, j]).to(g.device) for j in range(4))
    return g[b, a, gj, gi]


@pytest.mark.parametrize("name", sorted(CASES))
def test_assignment_is_the_reference(name):
    case = CASES[name]
    crit = SetCriterion(**case["kw"])
    for k, (targets, heads) in enumerate(case["calls"]):
        for l, m in enumerate(device_matches(crit, targets, heads)):
            q = f"{name}/{k}/{l}"
            assert np.array_equal(m["idx"], GOLD[q + "/idx"]), q
            assert np.array_equal(m["tbox"], GOLD[q + "/tbox"].view(np.int32)), q
            assert np.array_equal(m["anchor"], GOLD[q + "/anchor"].view(np.int32)), q


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("host_targets", [True, False])
def test_fp32_losses_and_gradients_are_the_reference(name, host_targets):
    case = CASES[name]
    crit = SetCriterion(**case["kw"])
    for k, (targets, heads) in enumerate(case["calls"]):
        losses, gs = device_loss(crit, targets if host_targets else targets.to(DEV), heads)
        assert_losses(losses, GOLD[f"{name}/{k}/losses"], (name, k))
        if case["kw"].get("auto_balance"):
            assert np.allclose(crit.balance, GOLD[f"{name}/{k}/balance"], rtol=1e-5, atol=0), (k, crit.balance)
        for l, g in enumerate(gs):
            at, dense = fixture_grads(name, k, l)
            assert_grad(gathered(g, GOLD[f"{name}/{k}/{l}/idx"]), at, (name, k, l, "matched"))
            assert_grad(g[..., 4].reshape(-1)[torch.from_numpy(LC.dense_sample(g.shape)).to(DEV)], dense,
                        (name, k, l, "dense"))


@pytest.mark.parametrize("name", ["basic", "hyper", "dup", "p6", "nc1", "edges"])
def test_fp16_gradients_under_a_grad_scaler_are_the_reference(name):
    case = CASES[name]
    targets, heads = case["calls"][0]
    losses, gs = device_loss(SetCriterion(**case["kw"]), targets, [h.half() for h in heads], grad=SCALE)
    assert_losses(losses, GOLD[f"{name}/0/losses"], name)
    for l, g in enumerate(gs):
        assert g.dtype == torch.float16
        at, dense = fixture_grads(name, 0, l)
        assert_within_one_ulp(gathered(g, GOLD[f"{name}/0/{l}/idx"]), at.astype(np.float64) * SCALE, (name, l))
        cells = torch.from_numpy(LC.dense_sample(g.shape)).to(DEV)
        assert_within_one_ulp(g[..., 4].reshape(-1)[cells], dense.astype(np.float64) * SCALE, (name, l, "dense"))


def restated(case_kw, targets, heads64):
    kw = {k: v for k, v in case_kw.items() if k not in ("fl_gamma", "auto_balance")}
    heads64 = [h.detach().requires_grad_(True) for h in heads64]
    losses, _, asg = R.loss(targets, heads64, **kw)
    gs = torch.autograd.grad([losses[k] for k in KEYS if losses[k].requires_grad], heads64, allow_unused=True)
    gs = [torch.zeros_like(h) if g is None else g for g, h in zip(gs, heads64)]
    return np.array([float(losses[k]) for k in KEYS]), gs, asg


@pytest.mark.parametrize("name", ["basic", "dup", "p6", "edges"])
def test_bf16_gradients_are_the_fp64_restatement(name):
    case = CASES[name]
    targets, heads = case["calls"][0]
    hb = [h.bfloat16() for h in heads]
    want_l, want_g, _ = restated(case["kw"], targets.to(DEV), [h.to(DEV).double() for h in hb])
    losses, gs = device_loss(SetCriterion(**case["kw"]), targets, hb, grad=SCALE)
    assert_losses(losses, want_l, name)
    for l, (g, w) in enumerate(zip(gs, want_g)):
        assert g.dtype == torch.bfloat16
        assert_within_one_ulp(g, w * SCALE, (name, l))


def big_case(kind):
    if kind == "yolov5s_b32_640":
        shapes = LC.head_shapes(32, 640, 640, LC.P5_STRIDES, 3, 80)
        kw = {"strides": LC.P5_STRIDES, "anchor_grids": LC.P5_ANCHORS, "num_classes": 80}
        n = 32
    else:
        shapes = LC.head_shapes(16, 1280, 1280, LC.P6_STRIDES, 3, 80)
        kw = {"strides": LC.P6_STRIDES, "anchor_grids": LC.P6_ANCHORS, "num_classes": 80}
        n = 16
    return kw, shapes, LC.random_targets(n, 80, 7 * n, 900 + n)


@pytest.mark.parametrize("kind", ["yolov5s_b32_640", "yolov5x6_b16_1280"])
def test_training_shapes_are_the_fp64_restatement(kind):
    kw, shapes, targets = big_case(kind)
    heads = LC.head_outputs(shapes, 7, device=DEV)
    crit = SetCriterion(**kw)
    for l, (m, ref) in enumerate(zip(device_matches(crit, targets, heads),
                                     R.assign(targets.to(DEV), shapes, R.grid_anchors(kw["anchor_grids"],
                                                                                      kw["strides"], DEV), 4.0))):
        idx = torch.stack([ref["b"], ref["a"], ref["gj"], ref["gi"], ref["cls"]], 1).cpu().numpy()
        assert np.array_equal(m["idx"], idx), l
        assert np.array_equal(m["tbox"], ref["tbox"].cpu().numpy().view(np.int32)), l
    want_l, want_g, _ = restated(kw, targets.to(DEV), [h.double() for h in heads])
    losses, gs = device_loss(crit, targets, heads)
    assert_losses(losses, want_l, kind)
    for l, (g, w) in enumerate(zip(gs, want_g)):
        assert_grad(g, w, (kind, l))
    del gs
    losses16, gs16 = device_loss(crit, targets, [h.half() for h in heads], grad=SCALE)
    assert_losses(losses16, want_l, kind)
    for l, (g, w) in enumerate(zip(gs16, want_g)):
        assert_within_one_ulp(g, w * SCALE, (kind, l, "fp16"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_repeated_calls_give_the_same_bits(dtype):
    case = CASES["dup"]
    targets, heads = case["calls"][0]
    heads = [h.to(dtype) for h in heads]
    crit = SetCriterion(**case["kw"])
    a_l, a_g = device_loss(crit, targets, heads, grad=3.0)
    b_l, b_g = device_loss(crit, targets.to(DEV), heads, grad=3.0)
    assert np.array_equal(a_l.view(np.int64), b_l.view(np.int64))
    for x, y in zip(a_g, b_g):
        assert torch.equal(x.view(torch.int16 if dtype != torch.float32 else torch.int32),
                           y.view(torch.int16 if dtype != torch.float32 else torch.int32))


def test_backward_fills_grad_and_no_grad_keeps_no_state():
    case = CASES["basic"]
    targets, heads = case["calls"][0]
    heads = [h.to(DEV).requires_grad_(True) for h in heads]
    crit = SetCriterion(**case["kw"])
    out = crit(targets, heads)
    loss = out["cls_logits"] + out["bbox_regression"] + out["objectness"]
    loss.backward()
    assert all(h.grad is not None and h.grad.shape == h.shape and bool(h.grad.abs().sum() > 0) for h in heads)
    with torch.no_grad():
        out2 = crit(targets, heads)
    assert all(v.grad_fn is None for v in out2.values())
    assert torch.equal(torch.cat(list(out.values())).detach(), torch.cat(list(out2.values())))
    assert torch.is_grad_enabled()


def test_only_the_used_loss_term_reaches_the_gradient():
    case = CASES["basic"]
    targets, heads = case["calls"][0]
    heads = [h.to(DEV).requires_grad_(True) for h in heads]
    out = SetCriterion(**case["kw"])(targets, heads)
    g = torch.autograd.grad(out["objectness"] * 2.0, heads)
    for l, x in enumerate(g):
        assert float(x[..., :4].abs().max()) == 0.0 and float(x[..., 5:].abs().max()) == 0.0
        at, dense = fixture_grads("basic", 0, l)
        cells = torch.from_numpy(LC.dense_sample(x.shape)).to(DEV)
        assert_grad(x[..., 4].reshape(-1)[cells], 2.0 * dense, l)


@pytest.mark.parametrize("row,bit", [
    ((2, 0, 0.5, 0.5, 0.1, 0.1), "image"),
    ((-1, 0, 0.5, 0.5, 0.1, 0.1), "image"),
    ((0, 8, 0.5, 0.5, 0.1, 0.1), "class"),
    ((0, 0, float("nan"), 0.5, 0.1, 0.1), "non-finite"),
    ((0, 0, 0.5, 0.5, float("-inf"), 0.1), "non-finite"),
])
def test_invalid_device_targets_raise(row, bit):
    case = CASES["basic"]
    targets, heads = case["calls"][0]
    t = torch.cat([targets, torch.tensor([row], dtype=torch.float32)]).to(DEV)
    with pytest.raises(ValueError, match=bit):
        SetCriterion(**case["kw"])(t, [h.to(DEV) for h in heads])
    losses, _ = device_loss(SetCriterion(**case["kw"]), targets.to(DEV), heads)   # the device is still usable
    assert_losses(losses, GOLD["basic/0/losses"], "after")


def test_yolo_training_mode_returns_the_criterion_loss():
    from parity_util import layouts, synth_state_dict
    from yolort_b200.models import yolov5n

    m = yolov5n(size=(128, 128), score_thresh=0.15)
    m.load_state_dict(synth_state_dict(layouts()["n"], knob_obj=7.0, knob_cls=4.5, seed=0))
    model = m.model
    crit = SetCriterion(model.anchor_generator.strides, model.anchor_generator.anchor_grids, model.num_classes)
    model.compute_loss = crit
    m = m.to(DEV).train()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(3)).to(DEV)
    targets = LC.random_targets(2, 80, 9, 5).to(DEV)
    got = model(x, targets)
    want = crit(targets, model.head(model.backbone(x)))
    assert list(got) == list(KEYS)
    for k in KEYS:
        assert torch.equal(got[k], want[k]) and bool(torch.isfinite(got[k]).all())
    model.compute_loss = None
    with pytest.raises(NotImplementedError):
        model(x, targets)
    m.eval()
