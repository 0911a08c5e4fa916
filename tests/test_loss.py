"""The training loss on the host: the torch restatement (oracle/restate_loss.py) against the reference's fixtures
(tests/golden/loss.npz), SetCriterion's constructor attributes, and the host-side validation of targets."""
import json
import os

import numpy as np
import pytest
import torch

import loss_cases as LC
from oracle import ref_import
from oracle import restate_loss as R
from yolort_b200.models.box_head import SetCriterion

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "loss.npz"))
with open(os.path.join(os.path.dirname(__file__), "golden", "loss.json")) as _f:
    META = json.load(_f)
CASES = LC.cases()
KEYS = ("cls_logits", "bbox_regression", "objectness")


def restate(case, targets, heads, balance):
    kw = {k: v for k, v in case["kw"].items() if k not in ("fl_gamma", "auto_balance")}
    return R.loss(targets, heads, balance=balance, **kw)


def run_case(name, dtype=torch.float32):
    """Every call of the case through the restatement; yields (call, losses, objs, assignment, heads, balance)."""
    case = CASES[name]
    balance = list(R.BALANCE_DEFAULTS[: len(case["kw"]["strides"])])
    strides = case["kw"]["strides"]
    ssi = strides.index(16) if 16 in strides else 0
    for k, (targets, heads) in enumerate(case["calls"]):
        heads = [h.to(dtype).requires_grad_(True) for h in heads]
        losses, objs, asg = restate(case, targets, heads, balance)
        yield k, losses, objs, asg, heads, balance
        if case["kw"].get("auto_balance"):
            balance = R.update_balance(balance, [float(o.detach()) for o in objs], ssi)


def test_fixture_metadata():
    assert sorted(META) == sorted(CASES)
    for name, case in CASES.items():
        assert [c["n_targets"] for c in META[name]["calls"]] == [int(t.shape[0]) for t, _ in case["calls"]]


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_assignment_is_the_reference(name):
    for k, _, _, asg, heads, _ in run_case(name):
        for i, m in enumerate(asg):
            q = f"{name}/{k}/{i}"
            idx = torch.stack([m["b"], m["a"], m["gj"], m["gi"], m["cls"]], 1).numpy()
            assert np.array_equal(idx, GOLD[q + "/idx"]), q
            assert np.array_equal(m["tbox"].numpy().view(np.int32), GOLD[q + "/tbox"].view(np.int32)), q
            assert np.array_equal(m["anchor"].numpy().view(np.int32), GOLD[q + "/anchor"].view(np.int32)), q


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_losses_and_gradients_are_the_reference(name):
    case = CASES[name]
    for k, losses, objs, asg, heads, balance in run_case(name):
        got = np.array([float(losses[key].detach()) for key in KEYS])
        want = GOLD[f"{name}/{k}/losses"].astype(np.float64)
        assert np.all(np.abs(got - want) <= 1e-6 * np.abs(want)), (name, k, got, want)
        grads = {}
        for key in KEYS:
            if losses[key].requires_grad:
                grads[key] = torch.autograd.grad(losses[key], heads, retain_graph=True, allow_unused=True)
            else:
                grads[key] = [None] * len(heads)
        for i, h in enumerate(heads):
            z = torch.zeros_like(h)
            g = torch.cat([(grads["bbox_regression"][i] if grads["bbox_regression"][i] is not None else z)[..., :4],
                           (grads["objectness"][i] if grads["objectness"][i] is not None else z)[..., 4:5],
                           (grads["cls_logits"][i] if grads["cls_logits"][i] is not None else z)[..., 5:]], -1)
            q = f"{name}/{k}/{i}"
            m = asg[i]
            at = g[m["b"], m["a"], m["gj"], m["gi"]].detach().numpy()
            dense = g[..., 4].reshape(-1)[LC.dense_sample(h.shape)].detach().numpy()
            for got_g, want_g in ((at, GOLD[q + "/grad"]), (dense, GOLD[q + "/dense"])):
                scale = max(float(np.abs(want_g).max()) if want_g.size else 0.0, 1e-30)
                assert np.all(np.abs(got_g - want_g) <= 1e-5 * scale), q
        if case["kw"].get("auto_balance"):
            strides = case["kw"]["strides"]
            nxt = R.update_balance(balance, [float(o.detach()) for o in objs], strides.index(16))
            assert np.allclose(nxt, GOLD[f"{name}/{k}/balance"], rtol=1e-6, atol=0), (k, nxt)


def test_restatement_in_fp64_is_close_to_fp32():
    _, losses32, _, _, _, _ = next(run_case("basic"))
    _, losses64, _, _, _, _ = next(run_case("basic", torch.float64))
    for key in KEYS:
        assert abs(float(losses32[key]) - float(losses64[key])) <= 1e-5 * abs(float(losses64[key])) + 1e-12


def crit_attrs(c):
    return {k: getattr(c, k) for k in ("num_classes", "strides", "anchor_grids", "num_anchors", "balance", "ssi",
                                         "sort_obj_iou", "cls_pos", "obj_pos", "smooth_pos", "smooth_neg", "gr",
                                         "auto_balance", "box_gain", "cls_gain", "obj_gain", "anchor_thresh")}


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference tree")
@pytest.mark.parametrize("name", sorted(CASES))
def test_constructor_attributes_are_the_reference(name):
    ref_import.import_reference()
    from yolort.models.box_head import SetCriterion as RefCriterion

    kw = CASES[name]["kw"]
    assert crit_attrs(SetCriterion(**kw)) == crit_attrs(RefCriterion(**kw))
    tensor_kw = dict(kw, strides=torch.tensor(kw["strides"]))
    mine = SetCriterion(**tensor_kw)
    assert crit_attrs(mine) == crit_attrs(RefCriterion(**kw))
    assert all(type(s) is int for s in mine.strides)


def test_constructor_attributes():
    c = SetCriterion(LC.P6_STRIDES, LC.P6_ANCHORS, 80, label_smoothing=0.1)
    assert c.balance == [4.0, 1.0, 0.4, 0.1] and c.ssi == 1 and c.num_anchors == 3
    assert (c.smooth_pos, c.smooth_neg) == (1.0 - 0.5 * 0.1, 0.5 * 0.1) and c.gr == 1.0 and c.sort_obj_iou is False
    c = SetCriterion(torch.tensor([8, 32]), LC.P5_ANCHORS[:1] + LC.P5_ANCHORS[2:], 3)
    assert c.strides == [8, 32] and c.ssi == 0 and c.balance == [4.0, 1.0]


@pytest.mark.parametrize("row,why", [
    ((2, 0, 0.5, 0.5, 0.1, 0.1), "image"),
    ((-1, 0, 0.5, 0.5, 0.1, 0.1), "image"),
    ((0, 8, 0.5, 0.5, 0.1, 0.1), "class"),
    ((0, -1, 0.5, 0.5, 0.1, 0.1), "class"),
    ((0, 0, float("nan"), 0.5, 0.1, 0.1), "finite"),
    ((0, 0, 0.5, 0.5, float("inf"), 0.1), "finite"),
])
def test_malformed_host_targets_raise(row, why):
    c = SetCriterion(LC.P5_STRIDES, LC.P5_ANCHORS, 8)
    heads = LC.head_outputs(LC.head_shapes(2, 64, 64, LC.P5_STRIDES, 3, 8), 0)
    t = torch.tensor([(0, 1, 0.5, 0.5, 0.2, 0.2), row], dtype=torch.float32)
    with pytest.raises(ValueError, match=why):
        c(t, heads)


@pytest.mark.parametrize("bad", [torch.zeros((3, 5)), torch.zeros((3, 6), dtype=torch.int64), torch.zeros(6)])
def test_malformed_target_shapes_raise(bad):
    c = SetCriterion(LC.P5_STRIDES, LC.P5_ANCHORS, 8)
    heads = LC.head_outputs(LC.head_shapes(2, 64, 64, LC.P5_STRIDES, 3, 8), 0)
    with pytest.raises(ValueError):
        c(bad, heads)


def test_heads_must_match_the_criterion():
    c = SetCriterion(LC.P5_STRIDES, LC.P5_ANCHORS, 8)
    heads = LC.head_outputs(LC.head_shapes(2, 64, 64, LC.P5_STRIDES, 3, 4), 0)
    with pytest.raises(ValueError):
        c(torch.zeros((0, 6)), heads)
    with pytest.raises(ValueError):
        c(torch.zeros((0, 6)), heads[:2])
