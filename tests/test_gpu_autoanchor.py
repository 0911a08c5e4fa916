"""AutoAnchor on the GPU (csrc/autoanchor.cu through yolort_b200/v5/utils/autoanchor.py): the reference's fixtures
end to end, every kernel bit for bit against oracle/restate_autoanchor.py, replays, and the models' use of replaced
anchors."""
import logging
import os
import random
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import autoanchor_cases as AC  # noqa: E402
from oracle import restate_autoanchor as R  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(ROOT, "tests", "golden", "autoanchor.npz"))


class _Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

        self.debug = []

    def emit(self, record):
        (self.lines if record.levelno >= logging.INFO else self.debug).append(record.getMessage())


def _run(name, model=None):
    from yolort_b200.models import yolov5n
    from yolort_b200.v5.utils import autoanchor as AA

    make, call, kw, seed = AC.CASES[name]
    ds = make()
    h = _Lines()
    AA.LOGGER.addHandler(h)
    AA.LOGGER.setLevel(logging.DEBUG)
    random.seed(seed)
    np.random.seed(seed)
    try:
        if call == "kmean":
            res = AA.kmean_anchors(ds, n=kw["n"], img_size=640, thr=4.0, gen=kw["gen"], verbose=True)
        else:
            if model is None:
                model = yolov5n(size=(128, 128), strides=AC.P5_STRIDES, anchor_grids=AC.P5_ANCHORS)
            AA.check_anchors(ds, model, thr=4.0, imgsz=640)
            res = np.array(model.model.anchor_generator.anchors_px(), dtype=np.float64).reshape(-1, 2)
    finally:
        AA.LOGGER.removeHandler(h)
    accepted = [int(m.group(1)) for m in map(re.compile(r".*generation (\d+):").match, h.debug) if m]
    return res, h.lines, accepted


@pytest.mark.parametrize("name", list(AC.CASES))
def test_fixture_end_to_end(name):
    res, lines, accepted = _run(name)
    assert accepted == G[f"{name}/accepted"].tolist()
    ref_lines = str(G[f"{name}/log"]).split("\x00")
    assert repr(random.getstate()) == str(G[f"{name}/py_state"])
    assert np.array_equal(np.random.get_state()[1], G[f"{name}/np_state"])
    assert np.random.get_state()[2] == int(G[f"{name}/np_pos"])
    if str(G[f"{name}/error"]):
        # the reference fails after logging the caught error (autoanchor.py:59 evaluates the metric of the unflattened
        # [nl, na, 2] anchors); here the current anchors are kept
        assert lines[:len(ref_lines)] == ref_lines
        assert lines[len(ref_lines):] == [f"{R.PREFIX}Original anchors better than new anchors. Proceeding with "
                                          "original anchors."]
        assert np.array_equal(res, np.array(AC.P5_ANCHORS, dtype=np.float64).reshape(-1, 2))
        return
    assert lines == ref_lines
    assert np.array_equal(res, G[f"{name}/anchors"])


def _wh(ds, img_size=640):
    shapes = img_size * ds.shapes / ds.shapes.max(1, keepdims=True)
    wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, ds.labels)])
    return wh0, wh0[(wh0 >= 2.0).any(1)]


def _coco_like(n=860_000, seed=0):
    rng = np.random.default_rng(seed)
    return np.clip(rng.lognormal(3.6, 0.9, (n, 2)), 2.0, 640.0)


@pytest.mark.parametrize("name,size", [("poor9", 0), ("poor12", 0), ("coco", 30_000), ("coco", 860_000)])
def test_kmeans_kernel_equals_restatement(name, size):
    from yolort_b200 import _C

    wh = _coco_like(size) if name == "coco" else _wh(AC.CASES[name][0]())[1]
    k = 9 if name != "poor12" else 12
    obs = wh / wh.std(0)
    np.random.seed(5)
    idx = R.draw_kpoints(obs.shape[0], k, 30)
    d_obs = torch.from_numpy(obs).cuda()
    books, sizes, dist, _ = _C.kmeans(d_obs, d_obs[torch.from_numpy(idx).cuda()])
    books2, sizes2, dist2, _ = _C.kmeans(d_obs, d_obs[torch.from_numpy(idx).cuda()])
    assert torch.equal(books, books2) and torch.equal(dist, dist2)
    # at 860 k labels the restatement takes about a minute per trial on the CPU: three trials stand for the thirty
    for t in range(30 if obs.shape[0] < 100_000 else 3):
        book, d, _ = R.kmeans_trial(obs, obs[idx[t]])
        assert int(sizes[t]) == book.shape[0]
        assert np.array_equal(books[t, :book.shape[0]].cpu().numpy(), book), t
        assert float(dist[t]) == d, t


@pytest.mark.parametrize("n_labels,gen,na", [(2_000, 1000, 9), (100_000, 1000, 9), (860_000, 100, 12)])
def test_evolution_kernel_equals_restatement(n_labels, gen, na):
    from yolort_b200.v5.utils import autoanchor as AA

    wh = _coco_like(n_labels, seed=n_labels).astype(np.float32)
    rng = np.random.default_rng(1)
    k0 = np.sort(rng.uniform(8, 300, (na, 2)), axis=0)
    np.random.seed(3)
    random.seed(3)
    v = AA.draw_mutations(na, gen)
    d = torch.from_numpy(wh).cuda()
    k, fit, acc = AA.evolve_anchors(d, k0, v, 0.25)
    k2, fit2, acc2 = AA.evolve_anchors(d, k0, v, 0.25)
    assert np.array_equal(k, k2) and np.array_equal(fit, fit2) and acc == acc2
    kr, fitr, accr = R.evolve(wh, k0, v, 0.25)
    assert acc == accr and np.array_equal(fit, fitr) and np.array_equal(k, kr)


@pytest.mark.parametrize("f64", [False, True])
def test_metric_kernel_counts(f64):
    from yolort_b200 import _C

    wh = _coco_like(200_000, seed=4).astype(np.float32)
    k = np.array(AC.P5_ANCHORS, dtype=np.float32).reshape(-1, 2).astype(np.float64)
    c, s = _C.anchor_metric(torch.from_numpy(wh).cuda(), torch.from_numpy(k), 0.25, f64)
    ref = R.metric_stats(wh, k, 0.25, f64)
    assert c.tolist() == list(ref[:2])
    assert np.allclose(s.cpu().numpy(), ref[2:], rtol=1e-12)


def _model(grids):
    from yolort_b200.models import yolov5n
    from oracle.make_golden import synth_state_dict
    import json

    with open(os.path.join(ROOT, "tests", "golden", "state_dict_layouts.json")) as f:
        shapes = json.load(f)["n"]
    m = yolov5n(size=(128, 128), score_thresh=0.15, anchor_grids=grids).eval()
    m.load_state_dict(synth_state_dict(shapes, knob_obj=7.0, knob_cls=4.5, seed=0))
    return m.cuda()


def _same(x, y):
    assert len(x) == len(y)
    for p, q in zip(x, y):
        for key in p:
            assert torch.equal(p[key], q[key]), key


def _inputs():
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand(2, 3, 128, 128, device="cuda", generator=g)
    ims = [torch.rand(3, 100, 90, device="cuda", generator=g), torch.rand(3, 128, 96, device="cuda", generator=g)]
    return x, ims


def _outputs(m, x, ims, monkeypatch):
    """Every decode path: forward, predict-style list input, TTA, the padded decode, the fused head epilogue."""
    out = {"forward": m.model(x), "list": m(ims), "tta": m(ims, augment=True)}
    plan = m.model.get_plan(2, 128, 128)
    m.model._write_samples(plan, x)
    out["padded"] = list(m.model.detect_padded(plan))
    monkeypatch.setenv("YB_FUSED_DECODE", "1")
    out["fused"] = m.model(x)
    monkeypatch.delenv("YB_FUSED_DECODE")
    return out


def _same_outputs(a, b):
    for key in a:
        if key == "padded":
            for u, w in zip(a[key], b[key]):
                assert torch.equal(u, w), key
        else:
            _same(a[key], b[key])


def test_check_anchors_replacement_reaches_every_path(monkeypatch):
    """check_anchors replaces the anchors of a model whose plans (fused epilogue included) were built with the old
    ones: every decode path and the loss then equal those of a model built with the new anchors."""
    from yolort_b200.models.box_head import SetCriterion

    replaced = _model(AC.P5_ANCHORS)
    crit = SetCriterion(AC.P5_STRIDES, AC.P5_ANCHORS, 80)
    replaced.model.compute_loss = crit
    x, ims = _inputs()
    old = _outputs(replaced, x, ims, monkeypatch)
    res, lines, _ = _run("poor_check", model=replaced)
    assert lines == str(G["poor_check/log"]).split("\x00")
    assert np.array_equal(res, G["poor_check/anchors"])
    new = G["poor_check/anchors"].astype(np.float32).reshape(3, 6).tolist()
    fresh = _model(new)
    assert replaced.model.anchor_generator.anchors_px() == fresh.model.anchor_generator.anchors_px()
    got, want = _outputs(replaced, x, ims, monkeypatch), _outputs(fresh, x, ims, monkeypatch)
    _same_outputs(got, want)
    assert any(not torch.equal(o["boxes"], n["boxes"]) for o, n in zip(old["forward"], got["forward"]))

    crit_b = SetCriterion(AC.P5_STRIDES, new, 80)
    assert crit.anchor_grids == fresh.model.anchor_generator.anchors_px()
    g = torch.Generator(device="cuda").manual_seed(1)
    heads = [torch.randn(2, 3, s, s, 85, device="cuda", generator=g) for s in (16, 8, 4)]
    targets = torch.tensor([[0, 3, 0.5, 0.5, 0.2, 0.3], [1, 7, 0.3, 0.6, 0.05, 0.1]], device="cuda")
    la, lb = crit(targets, heads), crit_b(targets, heads)
    for key in la:
        assert torch.equal(la[key], lb[key]), key


@pytest.mark.parametrize("name", ["good_fit", "few_clusters"])
def test_check_anchors_that_keeps_the_anchors_changes_nothing(name, monkeypatch):
    m = _model(AC.P5_ANCHORS)
    x, ims = _inputs()
    before = _outputs(m, x, ims, monkeypatch)
    px = m.model.anchor_generator.anchors_px()
    _run(name, model=m)
    assert m.model.anchor_generator.anchors_px() == px
    _same_outputs(_outputs(m, x, ims, monkeypatch), before)


def test_set_anchor_grids_leaves_other_models_alone(monkeypatch):
    a, b = _model(AC.P5_ANCHORS), _model(AC.P5_ANCHORS)
    x, ims = _inputs()
    before = _outputs(b, x, ims, monkeypatch)
    a.model.set_anchor_grids([[12, 15, 19, 33, 35, 26], [33, 64, 66, 47, 61, 124], [120, 95, 160, 205, 380, 330]])
    _same_outputs(_outputs(b, x, ims, monkeypatch), before)
