"""Training the detection head on the device: the split-K weight-gradient kernel (csrc/conv_wgrad_sm90.cu) against
fp64 at every head shape of the shipped architectures, the differentiable YOLOHead (weight, bias and feature
gradients, accumulation, determinism), the in-place head refresh after optimizer steps, and a short training run."""
import warnings

import pytest
import torch

import head_grad_cases as HC
import loss_cases as LC
from parity_util import layouts, synth_state_dict
from yolort_b200 import _C
from yolort_b200.models.box_head import SetCriterion

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BOUND = 2.0 ** -14       # |err| <= BOUND * sum_p |dY| |X| (+ half an ulp of a 16-bit output)
HALF_ULP = {torch.float32: 0.0, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}   # relative to |ref|
WORST = {}               # worst |err| / bound per test group (printed with -s, recorded in DESIGN.md)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k in sorted(WORST):
        print(f"worst |err| / bound  {k}: {WORST[k]:.4f}")


def _note(key, frac):
    WORST[key] = max(WORST.get(key, 0.0), frac)


def _pad16(c):
    return (c + 15) // 16 * 16


def make_problem(P, co, ci, dtype, gen):
    dy_full = torch.zeros((P, _pad16(co)), dtype=dtype, device=DEV)
    dy_full[:, :co] = (torch.randn((P, co), generator=gen, device=DEV) * 0.5).to(dtype)
    x = (torch.randn((P, ci), generator=gen, device=DEV)).to(dtype)
    return dy_full, x


def check_wgrad(problems, dtype, out_dtype, key, seed=0, with_db=True):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    specs, data = [], []
    for P, co, ci in problems:
        dy, x = make_problem(P, co, ci, dtype, gen)
        dw = torch.full((co, ci), float("nan"), dtype=out_dtype, device=DEV)
        db = torch.full((co,), float("nan"), dtype=out_dtype, device=DEV) if with_db else None
        specs.append((dy, x, dw, db))
        data.append((dy[:, :co], x))
    _C.conv_wgrad(specs, torch.device(DEV))
    torch.cuda.synchronize()
    for (dy, x, dw, db), (dyv, xv) in zip(specs, data):
        d64, x64 = dyv.double(), xv.double()
        ref = d64.t() @ x64
        S = d64.abs().t() @ x64.abs()
        err = (dw.double() - ref).abs()
        bound = BOUND * S + HALF_ULP[out_dtype] * ref.abs()
        assert bool(torch.isfinite(dw.double()).all())
        _note(key, float((err / bound.clamp_min(1e-30)).max()))
        assert bool((err <= bound).all()), (key, float((err - bound).max()))
        if db is not None:
            rb, Sb = d64.sum(0), d64.abs().sum(0)
            eb = (db.double() - rb).abs()
            bb = BOUND * Sb + HALF_ULP[out_dtype] * rb.abs()
            _note(key + " db", float((eb / bb.clamp_min(1e-30)).max()))
            assert bool((eb <= bb).all()), (key, "db")
    return specs


@pytest.mark.parametrize("name,problems", HC.all_head_problems(), ids=[c[0] for c in HC.all_head_problems()])
def test_wgrad_every_head_shape(name, problems):
    check_wgrad(problems, torch.float16, torch.float32, "heads fp16->fp32")


@pytest.mark.parametrize("name,problems", HC.edge_problems(), ids=[c[0] for c in HC.edge_problems()])
def test_wgrad_edge_shapes(name, problems):
    check_wgrad(problems, torch.float16, torch.float32, "edges fp16->fp32")
    check_wgrad(problems, torch.bfloat16, torch.bfloat16, "edges bf16->bf16", with_db=False)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_wgrad_dtypes(dtype, out_dtype):
    check_wgrad(HC.head_problems("s_r60", 32, 640), dtype, out_dtype, f"s {dtype}->{out_dtype}")


def test_wgrad_is_deterministic():
    probs = HC.head_problems("s_r60", 8, 640)
    a = check_wgrad(probs, torch.float16, torch.float32, "determinism", seed=5)
    b = check_wgrad(probs, torch.float16, torch.float32, "determinism", seed=5)
    for (_, _, dw1, db1), (_, _, dw2, db2) in zip(a, b):
        assert torch.equal(dw1, dw2) and torch.equal(db1, db2)


def test_wgrad_rejects_a_short_workspace():
    dy, x = make_problem(1000, 255, 128, torch.float16, torch.Generator(device=DEV).manual_seed(0))
    dw = torch.empty((255, 128), dtype=torch.float32, device=DEV)
    probs = _C.wgrad_problems([(dy, x, dw, None)])
    need = int(_C.lib().yb_conv_wgrad_workspace_bytes(probs, 1))
    ws = torch.empty((need,), dtype=torch.uint8, device=DEV)
    rc = _C.lib().yb_conv_wgrad(probs, 1, ws.data_ptr(), need - 16, None)
    assert rc == -3 and b"workspace" in _C.lib().yb_last_error()


# ---- the differentiable head ------------------------------------------------------------------------------------
def _detector(name, size=128):
    """(wrapper module to train / state_dict, its YOLO) with synthetic weights, on the GPU, fp32 parameters."""
    if name == "lite":
        import json
        import os

        from oracle.make_golden_lite import synth_state_dict_lite
        from yolort_b200.models.yolo_lite import yolov5_mobilenet_v3_small_fpn

        m = yolov5_mobilenet_v3_small_fpn(pretrained_backbone=False, num_classes=80, score_thresh=0.15)
        with open(os.path.join(os.path.dirname(__file__), "golden", "state_dict_layouts_lite.json")) as f:
            m.load_state_dict(synth_state_dict_lite(json.load(f)["lite"]))
        m = m.to(DEV)
        return m, m
    from yolort_b200 import models as M

    ctor = {"s": M.yolov5s, "n": M.yolov5n, "n6": M.yolov5n6,
            "s_r31": lambda **k: M.yolov5s(upstream_version="r3.1", **k)}[name]
    m = ctor(size=(size, size), score_thresh=0.15)
    m.load_state_dict(synth_state_dict(layouts()[name], knob_obj=7.0, knob_cls=4.5, seed=0))
    m = m.to(DEV)
    return m, m.model


def _batch(yolo, n=2, size=128, seed=3):
    x = torch.rand(n, 3, size, size, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return x, LC.random_targets(n, yolo.num_classes, 12, seed).to(DEV)


def _criterion(yolo):
    ag = yolo.anchor_generator
    return SetCriterion(ag.strides, ag.anchor_grids, yolo.num_classes)


def _capture(yolo):
    """Forward hook on the head: records its input features and the incoming gradient of each output."""
    rec = {"feats": None, "grads": {}}

    def hook(mod, inputs, outputs):
        rec["feats"] = [f.detach() for f in inputs[0]]
        for l, o in enumerate(outputs):
            if o.requires_grad:
                o.register_hook(lambda g, l=l: rec["grads"].__setitem__(l, g.detach().clone()))
    return rec, yolo.head.register_forward_hook(hook)


def _ref_param_grads(yolo, feats, grads):
    """fp64 dW, db per level from the incoming gradients and the features, with S = sum |dY| |X| for the bound."""
    out = []
    for l, (f, conv) in enumerate(zip(feats, yolo.head.head)):
        g = grads[l]
        n, a, h, w, k = g.shape
        dy = g.permute(0, 2, 3, 1, 4).reshape(n * h * w, a * k).double()
        x = f.permute(0, 2, 3, 1).reshape(n * h * w, -1).double()
        out.append((dy.t() @ x, dy.abs().t() @ x.abs(), dy.sum(0), dy.abs().sum(0)))
    return out


def _assert_param_grads(yolo, ref, key):
    for conv, (rw, sw, rb, sb) in zip(yolo.head.head, ref):
        gw = conv.weight.grad.double().view(rw.shape)
        gb = conv.bias.grad.double()
        _note(key, float(((gw - rw).abs() / (BOUND * sw).clamp_min(1e-30)).max()))
        assert bool(((gw - rw).abs() <= BOUND * sw).all()), key
        assert bool(((gb - rb).abs() <= BOUND * sb).all()), key


@pytest.mark.parametrize("name", ["s", "n6", "s_r31", "lite"])
def test_head_gradients_match_fp64(name):
    m, yolo = _detector(name)
    yolo.backbone.requires_grad_(False)
    yolo.compute_loss = _criterion(yolo)
    yolo.train()
    x, targets = _batch(yolo)
    rec, h = _capture(yolo)
    with warnings.catch_warnings():
        warnings.simplefilter("error")          # a frozen backbone draws no warning
        loss = sum(yolo(x, targets).values())
        loss.backward()
    h.remove()
    assert len(rec["grads"]) == len(yolo.head.head)
    _assert_param_grads(yolo, _ref_param_grads(yolo, rec["feats"], rec["grads"]), f"e2e {name}")
    assert all(p.grad is None for p in yolo.backbone.parameters())
    assert all(c.weight.grad.dtype == torch.float32 for c in yolo.head.head)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_feature_gradients_match_fp64(dtype):
    m, yolo = _detector("s")
    if dtype == torch.bfloat16:
        m = m.to(dtype)
    yolo.backbone.requires_grad_(False)
    x, _ = _batch(yolo)
    feats = [f.detach().clone().requires_grad_() for f in yolo.backbone(x)]
    outs = yolo.head(feats)
    gen = torch.Generator(device=DEV).manual_seed(1)
    rs = [torch.randn(o.shape, generator=gen, device=DEV).to(o.dtype) for o in outs]
    torch.autograd.backward(outs, rs)
    tol = 2.0 ** -9 if dtype == torch.float16 else 2.0 ** -6
    for f, r, conv in zip(feats, rs, yolo.head.head):
        n, a, h, w, k = r.shape
        dy = r.permute(0, 2, 3, 1, 4).reshape(-1, a * k).double()
        wq = conv.weight.detach().to(dtype).double().view(a * k, -1)
        ref = (dy @ wq).view(n, h, w, -1).permute(0, 3, 1, 2)
        assert f.grad is not None and f.grad.shape == f.shape
        err = (f.grad.double() - ref).abs()
        _note(f"dgrad {dtype}", float((err / (tol * (1 + ref.abs()))).max()))
        assert bool((err <= tol * (1 + ref.abs())).all())


def _step_grads(yolo, x, targets):
    loss = sum(yolo(x, targets).values())
    loss.backward()
    return [p.grad.clone() for p in yolo._head_params()]


def test_gradient_accumulation_and_determinism():
    m, yolo = _detector("s")
    yolo.backbone.requires_grad_(False)
    yolo.compute_loss = _criterion(yolo)
    yolo.train()
    (x1, t1), (x2, t2) = _batch(yolo, seed=3), _batch(yolo, seed=4)
    g1 = _step_grads(yolo, x1, t1)
    yolo.zero_grad(set_to_none=True)
    g1b = _step_grads(yolo, x1, t1)
    assert all(torch.equal(a, b) for a, b in zip(g1, g1b))     # determinism
    yolo.zero_grad(set_to_none=True)
    g2 = _step_grads(yolo, x2, t2)
    yolo.zero_grad(set_to_none=True)
    _step_grads(yolo, x1, t1)
    acc = _step_grads(yolo, x2, t2)
    assert all(torch.equal(a, b + c) for a, b, c in zip(acc, g1, g2))
    yolo.zero_grad(set_to_none=True)
    l1 = sum(yolo(x1, t1).values())
    l2 = sum(yolo(x2, t2).values())            # both forwards before either backward
    l1.backward()
    l2.backward()
    assert all(torch.equal(p.grad, b + c) for p, b, c in zip(yolo._head_params(), g1, g2))


def _fresh_like(m, name="s"):
    m2, y2 = _detector(name)
    m2.load_state_dict(m.state_dict())
    return m2, y2


def _equal_dets(a, b):
    return len(a) == len(b) and all(torch.equal(d1[k], d2[k]) for d1, d2 in zip(a, b) for k in d1)


@pytest.mark.parametrize("graphs", [False, True])
def test_optimizer_steps_refresh_the_head_in_place(graphs):
    m, yolo = _detector("s")
    yolo.engine().graphs = graphs
    yolo.backbone.requires_grad_(False)
    yolo.compute_loss = _criterion(yolo)
    x, targets = _batch(yolo)
    opt = torch.optim.SGD(yolo.head.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    yolo.eval()
    with torch.no_grad():
        yolo(x)
    n_plans = len(yolo.engine()._plans)
    for step in range(10):
        yolo.train()
        sum(yolo(x, targets).values()).backward()
        opt.step()
        opt.zero_grad()
        yolo.eval()
        with torch.no_grad():
            dets = yolo(x)
            logits = yolo.head(yolo.backbone(x))
        _, y2 = _fresh_like(m)
        y2.eval()
        with torch.no_grad():
            assert _equal_dets(dets, y2(x)), step
            assert all(torch.equal(a, b) for a, b in zip(logits, y2.head(y2.backbone(x)))), step
        assert yolo.engine().lowerings == 1 and len(yolo.engine()._plans) >= n_plans
    assert yolo.engine().head_refreshes >= 10
    with torch.no_grad():
        next(yolo.backbone.parameters()).mul_(1.0)        # any backbone edit: full re-lowering
        yolo(x)
    assert yolo.engine().lowerings == 2


def test_training_recipe_lowers_the_loss_and_matches_an_fp64_replica():
    m, yolo = _detector("s")
    yolo.backbone.requires_grad_(False)
    yolo.compute_loss = _criterion(yolo)
    yolo.train()
    x, targets = _batch(yolo, n=4)
    params = list(yolo.head.parameters())
    replica = [p.detach().clone().requires_grad_() for p in params]
    kw = dict(lr=0.01, momentum=0.9, weight_decay=5e-4)
    opt, ropt = torch.optim.SGD(params, **kw), torch.optim.SGD(replica, **kw)
    scaler = torch.amp.GradScaler("cuda")
    rec, h = _capture(yolo)
    losses = []
    for _ in range(20):
        loss = sum(yolo(x, targets).values())
        losses.append(float(loss.detach()))
        scale = scaler.get_scale()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
        if scaler.get_scale() < scale:      # the scaler skipped this step: so does the replica
            continue
        ref = _ref_param_grads(yolo, rec["feats"], rec["grads"])
        for l, (rw, _, rb, _) in enumerate(ref):
            replica[2 * l].grad = (rw / scale).float().view_as(replica[2 * l])
            replica[2 * l + 1].grad = (rb / scale).float()
        ropt.step()
    h.remove()
    assert losses[-1] < losses[0], losses
    for p, r in zip(params, replica):
        assert float((p.detach() - r.detach()).norm()) <= 1e-3 * float(r.detach().norm())


def test_no_grad_and_frozen_heads_keep_todays_outputs_and_the_warning_fires_once():
    m, yolo = _detector("s")
    x, targets = _batch(yolo)
    feats = yolo.backbone(x)
    with torch.no_grad():
        ref = yolo.head(feats)
    assert all(o.grad_fn is None for o in ref)
    live = yolo.head(feats)
    assert all(o.grad_fn is not None for o in live)
    assert all(torch.equal(a, b) for a, b in zip(ref, live))
    yolo.head.requires_grad_(False)
    frozen = yolo.head(feats)
    assert all(o.grad_fn is None and torch.equal(a, o) for a, o in zip(ref, frozen))
    yolo.head.requires_grad_(True)
    yolo.compute_loss = _criterion(yolo)
    yolo.train()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        sum(yolo(x, targets).values()).backward()
        sum(yolo(x, targets).values()).backward()
    hits = [str(v.message) for v in w if "requires_grad_(False)" in str(v.message)]
    assert len(hits) == 1 and "model.model.backbone.requires_grad_(False)" in hits[0]
