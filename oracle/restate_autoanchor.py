"""numpy restatement of what csrc/autoanchor.cu computes for YOLOv5's AutoAnchor (yolort/v5/utils/autoanchor.py).

Each function states the reference lines it restates.  The random draws are not restated: they are numpy's and
Python's own generators, called in the reference's order (`draw_*` below, mirrored by yolort_b200/v5/utils/autoanchor.py).
"""
import math
import random

import numpy as np

PREFIX = "\033[34m\033[1mAutoAnchor: \033[0m"      # colorstr("AutoAnchor: ") (autoanchor.py:15)


# ---- numpy's mean of a contiguous float64 vector --------------------------------------------------------------------
def pairwise_sum(a: np.ndarray) -> np.float64:
    """numpy's pairwise_sum (umath loops_utils.h): below 8 elements one accumulator from 0.0; up to 128 elements 8
    accumulators over strided blocks, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail; above, split at
    n/2 rounded down to a multiple of 8."""
    n = a.shape[0]
    if n < 8:
        res = np.float64(0.0)
        for x in a:
            res = res + x
        return res
    if n <= 128:
        m = n - n % 8
        r = np.cumsum(a[:m].reshape(-1, 8), axis=0)[-1]       # column j: a[j] + a[j+8] + ... in order
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for x in a[m:]:
            res = res + x
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def np_mean(a: np.ndarray) -> np.float64:
    """np.mean(a) of a contiguous float64 vector: add.reduce seeded with 0.0, then / n."""
    return (np.float64(0.0) + pairwise_sum(a)) / np.float64(a.shape[0])


# ---- scipy.cluster.vq.kmeans (scipy 1.18: _vq_impl.py kmeans / _kmeans, _vq.pyx vq / update_cluster_means) ----------
def vq(obs: np.ndarray, book: np.ndarray):
    """_vq_small_nf: dist = (c0 - o0)^2 + (c1 - o1)^2, each product rounded; the first minimum wins; sqrt last."""
    d0 = book[None, :, 0] - obs[:, 0, None]
    d1 = book[None, :, 1] - obs[:, 1, None]
    d = d0 * d0 + d1 * d1
    code = np.argmin(d, axis=1)
    return code, np.sqrt(d[np.arange(obs.shape[0]), code])


def update_cluster_means(obs: np.ndarray, code: np.ndarray, nc: int):
    """Sums each cluster's members in observation order from 0.0 (a sequential chain), then / count."""
    book = np.zeros((nc, 2))
    np.add.at(book, code, obs)                 # unbuffered: one addition per observation, in index order
    count = np.bincount(code, minlength=nc)
    has = count > 0
    book[has] /= count[has, None].astype(np.float64)
    return book, has


def kmeans_trial(obs: np.ndarray, guess: np.ndarray, thresh: float = 1e-5):
    """_kmeans (_vq_impl.py:222-274): (book, distortion, iterations)."""
    book = guess.copy()
    prev, diff, it = math.inf, math.inf, 0
    while diff > thresh:
        code, d = vq(obs, book)
        cur = np_mean(d)
        book, has = update_cluster_means(obs, code, book.shape[0])
        book = book[has]
        diff = abs(prev - cur)
        prev = cur
        it += 1
    _, d = vq(obs, book)
    return book, np_mean(d), it


def kmeans(obs: np.ndarray, guesses: np.ndarray, thresh: float = 1e-5):
    """kmeans(obs, k, iter=len(guesses)) with the trials' starting books given: the best by strict <, in order."""
    best_book, best = None, math.inf
    for g in guesses:
        book, dist, _ = kmeans_trial(obs, g, thresh)
        if dist < best:
            best_book, best = book, dist
    return best_book, best


def draw_kpoints(n_pts: int, k: int, trials: int) -> np.ndarray:
    """_kpoints with the legacy global RandomState (kmeans' rng=None): choice(n_pts, k, replace=False) per trial."""
    return np.stack([np.random.choice(n_pts, size=int(k), replace=False) for _ in range(trials)])


# ---- the ratio metric (autoanchor.py:38-44, 97-101, 107-122) ----------------------------------------------------
def ratio_metric(wh: np.ndarray, k: np.ndarray):
    """x [n, na] = min(r, 1 / r) over both sides, r = wh / k, in wh's / k's common dtype; best [n] = max over anchors."""
    r = wh[:, None] / k[None]
    one = r.dtype.type(1)
    x = np.minimum(r, one / r).min(2)
    return x, x.max(1)


def metric_stats(wh32: np.ndarray, k: np.ndarray, thr: float, f64: bool):
    """(labels with best > thr, pairs with x > thr, sum x, sum best, sum x[x > thr]) as the device reports them; the
    float32 metric compares with fl32(thr), as torch compares a float32 tensor with a Python float."""
    kk = k.astype(np.float64) if f64 else k.astype(np.float32)
    w = wh32.astype(np.float64) if f64 else wh32
    x, best = ratio_metric(w, kk)
    t = np.float64(thr) if f64 else np.float32(thr)
    past = x > t
    return (int((best > t).sum()), int(past.sum()), float(x.astype(np.float64).sum()),
            float(best.astype(np.float64).sum()), float(x[past].astype(np.float64).sum()))


def check_bpr_aat(n_best: int, n_x: int, n: int):
    """check_anchors' metric (autoanchor.py:42-43): bpr = fl32(n_best / n), aat = fl32(n_x / n), float32 means of exact
    float32 sums (exact below 2^24)."""
    return np.float32(np.float32(n_best) / np.float32(n)), np.float32(np.float32(n_x) / np.float32(n))


def results_string(k: np.ndarray, stats, n_wh0: int, thr: float, n: int, img_size: int) -> str:
    """print_results' string (autoanchor.py:107-121) for k sorted small to large and the float64 stats of wh0."""
    n_best, n_x, s_x, s_best, s_past = stats
    bpr = np.float32(np.float32(n_best) / np.float32(n_wh0))
    aat = np.float32(np.float32(np.float32(n_x) / np.float32(n_wh0 * n)) * np.float32(n))
    past = s_past / n_x if n_x else float("nan")
    s = (f"{PREFIX}thr={thr:.2f}: {float(bpr):.4f} best possible recall, {float(aat):.2f} anchors past thr\n"
         f"{PREFIX}n={n}, img_size={img_size}, metric_all={s_x / (n_wh0 * n):.3f}/{s_best / n_wh0:.3f}-mean/best, "
         f"past_thr={past:.3f}-mean: ")
    for x in k:
        s += "%i,%i, " % (round(x[0]), round(x[1]))
    return s[:-2]


# ---- the evolution (autoanchor.py:103-105, 157-172) -----------------------------------------------------------------
def unit_exponent(thr: float) -> int:
    """Every best ratio above thr is a float32 in (thr, 1]: a whole multiple of 2^(floor(log2 thr) - 23)."""
    return math.floor(math.log2(np.float32(thr))) - 23


def fitness(wh32: np.ndarray, k: np.ndarray, thr: float) -> np.float32:
    """anchor_fitness(k) with the sum of best * (best > thr) exact: fl32(fl32(S) / n)."""
    _, best = ratio_metric(wh32, k.astype(np.float32))
    e = unit_exponent(thr)
    q = np.where(best > np.float32(thr), best, np.float32(0)).astype(np.float64) * 2.0 ** -e
    S = int(q.astype(np.int64).sum()) * 2.0 ** e
    return np.float32(np.float32(S) / np.float32(wh32.shape[0]))


def draw_mutations(n: int, gen: int, mp: float = 0.9, s: float = 0.1) -> np.ndarray:
    """The gen mutation vectors of autoanchor.py:163-165, drawn in the reference's order (npr.random, random.random,
    npr.randn; redrawn while all ones)."""
    npr = np.random
    sh = (n, 2)
    out = np.empty((gen, n, 2))
    for g in range(gen):
        v = np.ones(sh)
        while (v == 1).all():
            v = ((npr.random(sh) < mp) * random.random() * npr.randn(*sh) * s + 1).clip(0.3, 3.0)
        out[g] = v
    return out


def evolve(wh32: np.ndarray, k0: np.ndarray, v: np.ndarray, thr: float):
    """(k, fitness after each generation [gen + 1], accepted generations) of the loop at autoanchor.py:162-171."""
    k = k0.copy()
    f = fitness(wh32, k, thr)
    fits, acc = [f], []
    for g in range(v.shape[0]):
        kg = (k.copy() * v[g]).clip(min=2.0)
        fg = fitness(wh32, kg, thr)
        if fg > f:
            f, k = fg, kg.copy()
            acc.append(g)
        fits.append(f)
    return k, np.array(fits, dtype=np.float32), acc


# ---- how firmly a float32 fitness decision is pinned (oracle/make_golden_autoanchor.py) -------------------------------
def sum_bound(n: int, mean: float) -> float:
    """A bound on |float32 fitness - exact fitness| for n <= 2^16 non-negative terms of mean `mean`, whatever order
    torch sums them in: its CPU sum is a cascade of 4 levels of sequential runs of at most 16 items, combined across at
    most 32 vector lanes and 64 thread partials, a summation tree of depth d <= 164, whose error is at most
    d * 2^-24 * S; plus two float32 ulps for the roundings of the sum and of the division."""
    assert n <= 1 << 16
    return 164 * 2.0 ** -24 * mean + 2 * float(np.spacing(np.float32(max(mean, 1e-30))))


def _f32_orders(n: int, seed: int = 0):
    """Index orders for float32 sums: in order, reversed, and 20 seeded permutations."""
    rng = np.random.default_rng(seed)
    yield np.arange(n)
    yield np.arange(n)[::-1]
    for _ in range(20):
        yield rng.permutation(n)


def _f32_sums(t: np.ndarray, order: np.ndarray):
    """(sequential sum, 16-lane blocked sum, pairwise sum) of t[order] in float32."""
    x = t[order].astype(np.float32)
    seq = np.cumsum(x, dtype=np.float32)[-1] if x.size else np.float32(0)
    pad = np.zeros((-x.size) % 16, np.float32)
    lanes = np.cumsum(np.concatenate([x, pad]).reshape(-1, 16), axis=0, dtype=np.float32)[-1]
    return seq, np.cumsum(lanes, dtype=np.float32)[-1], np.float32(np.sum(x, dtype=np.float32))


def decision_pinned(tg: np.ndarray, tf: np.ndarray) -> str:
    """How the decision fg > f between the fitness terms tg (mutated anchors) and tf (current anchors) is pinned:
    "same terms" (both sums are the same float32 operations: fg == f), "margin" (the exact means differ by more than
    twice sum_bound), "orders" (below that margin, float32 sums in 66 orders -- 22 index orders, each sequential,
    16-lane blocked and pairwise -- all take the exact sum's decision), or "" when it is not pinned."""
    if np.array_equal(tg, tf):
        return "same terms"
    n = tg.shape[0]
    eg, ef = float(tg.astype(np.float64).sum()) / n, float(tf.astype(np.float64).sum()) / n   # exact: < 2^53 units
    if abs(eg - ef) > 2 * sum_bound(n, max(eg, ef)):
        return "margin"
    fn = np.float32(n)
    for order in _f32_orders(n):
        for sg, sf in zip(_f32_sums(tg, order), _f32_sums(tf, order)):
            if (np.float32(sg / fn) > np.float32(sf / fn)) != (eg > ef):
                return ""
    return "orders"


# ---- kmean_anchors as a whole (autoanchor.py:131-174) ----------------------------------------------------------------
def kmean_anchors(dataset, n: int = 9, img_size: int = 640, thr: float = 4.0, gen: int = 1000):
    """kmean_anchors on a loaded dataset with the reference's draws and these restated steps: (anchors sorted small to
    large, accepted generations).  Raises where the reference raises (choice's ValueError, the assertion)."""
    thr = 1 / thr
    shapes = img_size * dataset.shapes / dataset.shapes.max(1, keepdims=True)
    wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, dataset.labels)])
    wh = wh0[(wh0 >= 2.0).any(1)]
    s = wh.std(0)
    obs = wh / s
    k, _ = kmeans(obs, obs[draw_kpoints(obs.shape[0], n, 30)])
    assert len(k) == n
    k = k * s
    k = k[np.argsort(k.prod(1))]
    k, _, acc = evolve(wh.astype(np.float32), k, draw_mutations(n, gen), thr)
    return k[np.argsort(k.prod(1))], acc
