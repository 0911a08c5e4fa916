"""AutoAnchor on the CPU: the restatement of csrc/autoanchor.cu (oracle/restate_autoanchor.py) against numpy and
scipy, the public functions' input checks, and YOLO.set_anchor_grids on a CPU-built model."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import autoanchor_cases as AC  # noqa: E402
from oracle import restate_autoanchor as R  # noqa: E402


@pytest.mark.parametrize("n", [1, 7, 8, 9, 15, 16, 127, 128, 129, 136, 255, 256, 1000, 4097, 8192, 8193, 65537, 860001])
def test_pairwise_mean_equals_numpy(n):
    rng = np.random.default_rng(n)
    a = rng.random(n) * 10.0 ** rng.integers(-3, 4, n)
    assert R.np_mean(a) == np.mean(a)


@pytest.mark.parametrize("pts,k", [(200, 9), (1500, 12), (3000, 9)])
def test_kmeans_restatement_equals_scipy(pts, k):
    vq = pytest.importorskip("scipy.cluster.vq")
    rng = np.random.default_rng(pts)
    wh = rng.lognormal(3.0, 0.8, (pts, 2))
    obs = wh / wh.std(0)
    np.random.seed(pts)
    book, dist = vq.kmeans(obs, k, iter=30)
    state = np.random.get_state()[1].copy()
    np.random.seed(pts)
    book2, dist2 = R.kmeans(obs, obs[R.draw_kpoints(pts, k, 30)])
    assert np.array_equal(book, book2) and dist == dist2
    assert np.array_equal(state, np.random.get_state()[1])


def test_fitness_is_exact_sum():
    rng = np.random.default_rng(0)
    wh = rng.lognormal(3.0, 0.8, (5000, 2)).astype(np.float32)
    k = rng.uniform(5, 200, (9, 2))
    _, best = R.ratio_metric(wh, k.astype(np.float32))
    exact = sum(float(b) for b in best if b > np.float32(0.25))      # Python floats: exact for these 5000 terms
    assert R.fitness(wh, k, 0.25) == np.float32(np.float32(exact) / np.float32(5000))


def _fixture():
    return np.load(os.path.join(ROOT, "tests", "golden", "autoanchor.npz"))


def test_fixture_results_strings_restated():
    """The final print_results line of every kmean fixture, restated from the fixture's anchors."""
    g = _fixture()
    for name, (make, call, kw, _) in AC.CASES.items():
        if call != "kmean":
            continue
        ds = make()
        shapes = 640 * ds.shapes / ds.shapes.max(1, keepdims=True)
        wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, ds.labels)]).astype(np.float32)
        k = g[f"{name}/anchors"]
        stats = R.metric_stats(wh0, k, 0.25, True)
        assert R.results_string(k, stats, wh0.shape[0], 0.25, kw["n"], 640) == str(g[f"{name}/log"]).split("\x00")[-1]


def test_input_validation():
    from yolort_b200.v5.utils import autoanchor as AA

    ds = AC.make(1, 4, 4)
    with pytest.raises(NotImplementedError):
        AA.kmean_anchors("data/coco128.yaml")
    for bad in (dict(n=0), dict(n=2.5), dict(gen=-1), dict(thr=0.0), dict(thr=-4.0), dict(thr=float("nan")), dict(thr=float("inf"))):
        with pytest.raises(ValueError):
            AA.kmean_anchors(ds, **bad)
    with pytest.raises(ValueError):
        AA.kmean_anchors(AC.Dataset(ds.shapes.astype(np.float32), ds.labels))
    with pytest.raises(ValueError):
        AA.kmean_anchors(AC.Dataset(ds.shapes, [l.astype(np.float64) for l in ds.labels]))
    with pytest.raises(ValueError):
        AA.kmean_anchors(AC.Dataset(ds.shapes, ds.labels[:-1]))
    with pytest.raises(TypeError):
        AA.check_anchors(ds, object())


def test_set_anchor_grids_updates_every_copy():
    from yolort_b200.models import yolov5n
    from yolort_b200.models.box_head import SetCriterion

    model = yolov5n(size=(128, 128)).model
    crit = SetCriterion(model.anchor_generator.strides, model.anchor_generator.anchor_grids, 80)
    model.compute_loss = crit
    dropped = []

    class _Eng:
        def drop_plans(self):
            dropped.append(True)

    model._engine = _Eng()
    new = [[11.5, 14.25, 17, 31, 34, 24], [31, 62, 63, 46, 60, 120], [117, 91, 157, 199, 374, 327]]
    model.set_anchor_grids(new)
    px = model.anchor_generator.anchors_px()
    assert px == [[float(np.float32(v)) for v in lvl] for lvl in new]
    assert model.post_process.anchors_px == px and crit.anchor_grids == px
    assert model.post_config()["anchors_px"] == px and dropped == [True]
    for bad in ([[1, 2]], [lvl[:4] for lvl in new], [[-1.0] + lvl[1:] for lvl in new], [[float("inf")] + lvl[1:] for lvl in new]):
        with pytest.raises(ValueError):
            model.set_anchor_grids(bad)
    assert model.anchor_generator.anchors_px() == px


def test_check_anchor_order_reverses_levels():
    from yolort_b200.models import yolov5n
    from yolort_b200.v5.utils import autoanchor as AA

    wrapper = yolov5n(size=(128, 128))
    model = wrapper.model
    grids = model.anchor_generator.anchor_grids
    model.set_anchor_grids([[v * 2 ** (2 - 2 * i) for v in grids[2 - i]] for i in range(3)])   # largest first
    before = np.array(model.anchor_generator.anchors_px()).reshape(3, 3, 2) / np.array([8, 16, 32])[:, None, None]
    AA.check_anchor_order(wrapper)
    after = np.array(model.anchor_generator.anchors_px()).reshape(3, 3, 2) / np.array([8, 16, 32])[:, None, None]
    assert np.array_equal(after, before[::-1])


@pytest.mark.parametrize("name", [c for c, v in AC.CASES.items() if v[1] == "kmean"])
def test_restatement_equals_fixture(name):
    """The restated kmean_anchors (reference draws, restated k-means and exact-sum evolution) gives the reference's
    anchors, accepted generations and generator states."""
    import random

    pytest.importorskip("scipy")
    g = _fixture()
    make, _, kw, seed = AC.CASES[name]
    random.seed(seed)
    np.random.seed(seed)
    k, acc = R.kmean_anchors(make(), n=kw["n"], img_size=640, thr=4.0, gen=kw["gen"])
    assert np.array_equal(k, g[f"{name}/anchors"])
    assert acc == g[f"{name}/accepted"].tolist()
    assert repr(random.getstate()) == str(g[f"{name}/py_state"])
    assert np.array_equal(np.random.get_state()[1], g[f"{name}/np_state"])


def test_fixture_decisions_are_pinned():
    """Every case that evolves recorded its reference fitness per generation, and poor_check really replaced the
    anchors."""
    g = _fixture()
    for name in ("poor9", "poor12", "tiny", "poor_check"):
        gen = AC.CASES[name][2].get("gen", 1000)
        assert g[f"{name}/fitness"].shape == (gen + 1,) and len(g[f"{name}/accepted"]) > 0
    assert "New anchors saved to model" in str(g["poor_check/log"])


def test_threshold_at_most_one_keeps_no_generation():
    """thr = 1 / anchor_t >= 1: no ratio passes it, every fitness is 0 and the anchors stay (no launch needed)."""
    import torch
    from yolort_b200.v5.utils import autoanchor as AA

    k = np.array([[10.0, 13.0], [30.0, 61.0]])
    out, fit, acc = AA.evolve_anchors(torch.ones(4, 2), k, np.full((5, 2, 2), 1.1), 1.0)
    assert np.array_equal(out, k) and not fit.any() and fit.shape == (6,) and acc == []
