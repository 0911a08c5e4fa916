"""Writes tests/golden/autoanchor.npz: the unmodified reference's check_anchors / kmean_anchors
(yolort/v5/utils/autoanchor.py) on the seeded datasets of tests/autoanchor_cases.py, each after
random.seed(seed); np.random.seed(seed).  Stored per case c:

    c/anchors               kmean_anchors' float64 [n, 2] result, or the Detect anchors in pixels after check_anchors
    c/log                   the AutoAnchor log lines, joined by "\\x00"
    c/py_state, c/np_state  random.getstate() and np.random.get_state() after the call
    c/error                 the exception check_anchors raised, if it raised ("" otherwise)
    c/accepted, c/fitness   the generations kmean_anchors' evolution kept, and the reference's float32 fitness f after
                            each generation ([0]: the starting anchors); empty when no evolution ran

Every decision `fg > f` of the evolution is read from the reference's own frame, checked to equal the exact sum's
decision and to be pinned (oracle/restate_autoanchor.py, decision_pinned): the two anchor sets give every label the
same fitness term (fg == f whatever the order), or the exact means differ by more than twice the bound on torch's
float32 summation error, or, below that margin, float32 sums in 66 other orders all take the same decision.  A
regeneration on another host, whose torch may sum in another order, is expected to take the same decisions, and so
does the exact-sum GPU evolution.

The versions it ran with are stored under meta/.

    python oracle/make_golden_autoanchor.py
"""
import logging
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import autoanchor_cases as AC  # noqa: E402
from oracle import restate_autoanchor as R  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402


class _Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


class _Detect(torch.nn.Module):
    """What check_anchors reads of upstream's Detect: anchors [nl, na, 2] in stride units, stride [nl]."""

    def __init__(self, strides, grids):
        super().__init__()
        s = torch.tensor(strides, dtype=torch.float32)
        self.register_buffer("anchors", torch.tensor(grids, dtype=torch.float32).view(len(strides), -1, 2) / s.view(-1, 1, 1))
        self.register_buffer("stride", s)


class _Model(torch.nn.Module):
    def __init__(self, strides, grids):
        super().__init__()
        self.model = torch.nn.ModuleList([_Detect(strides, grids)])


class _Decisions:
    """Records (fg, f, kg, k, wh) at the reference's `if fg > f:` line (autoanchor.py:168) of every kmean_anchors call."""

    def __init__(self, AA):
        import inspect

        src, start = inspect.getsourcelines(AA.kmean_anchors)
        self.line = start + next(i for i, l in enumerate(src) if l.strip() == "if fg > f:")
        self.code = AA.kmean_anchors.__code__
        self.rows = []

    def _local(self, frame, event, arg):
        if event == "line" and frame.f_lineno == self.line:
            L = frame.f_locals
            self.rows.append((np.float32(L["fg"]), np.float32(L["f"]), L["kg"].copy(), np.array(L["k"]).copy(),
                              L["wh"].numpy()))
        return self._local

    def _global(self, frame, event, arg):
        return self._local if event == "call" and frame.f_code is self.code else None

    def __enter__(self):
        sys.settrace(self._global)
        return self

    def __exit__(self, *exc):
        sys.settrace(None)


def _check_decisions(name, rows, thr=0.25):
    """Asserts every recorded decision is pinned and equals the exact sum's; returns (accepted, fitness after each
    generation, how many decisions each kind of pin settled)."""
    accepted, fits, kinds = [], [], {}
    for g, (fg, f, kg, k, wh) in enumerate(rows):
        if g == 0:
            fits.append(f)
        tg = np.where((b := R.ratio_metric(wh, kg.astype(np.float32))[1]) > np.float32(thr), b, 0)
        tf = np.where((b := R.ratio_metric(wh, k.astype(np.float32))[1]) > np.float32(thr), b, 0)
        kind = R.decision_pinned(tg, tf)
        assert kind, (name, g, "decision not pinned")
        assert (fg > f) == (tg.astype(np.float64).sum() > tf.astype(np.float64).sum()), (name, g)
        assert kind != "same terms" or fg == f, (name, g)
        kinds[kind] = kinds.get(kind, 0) + 1
        if fg > f:
            accepted.append(g)
            f = fg
        fits.append(f)
    return np.array(accepted, dtype=np.int64), np.array(fits, dtype=np.float32), kinds


def main():
    import_reference()
    import scipy
    from yolort.v5.utils import autoanchor as AA

    log = logging.getLogger("yolort.v5.utils.general")
    log.setLevel(logging.INFO)
    out = {"meta/versions": np.array(f"torch {torch.__version__}, numpy {np.__version__}, scipy {scipy.__version__}")}
    for name, (make, call, kw, seed) in AC.CASES.items():
        ds = make()
        h = _Lines()
        log.addHandler(h)
        random.seed(seed)
        np.random.seed(seed)
        err = ""
        rec = _Decisions(AA)
        try:
            if call == "kmean":
                with rec:
                    res = AA.kmean_anchors(ds, n=kw["n"], img_size=640, thr=4.0, gen=kw["gen"], verbose=True)
            else:
                model = _Model(AC.P5_STRIDES, AC.P5_ANCHORS)
                with rec:
                    AA.check_anchors(ds, model, thr=4.0, imgsz=640)
                d = model.model[-1]
                res = (d.anchors * d.stride.view(-1, 1, 1)).reshape(-1, 2).double().numpy()
        except Exception as e:          # noqa: BLE001 -- the reference's own failure is part of the fixture
            err, res = f"{type(e).__name__}: {e}", np.zeros((0, 2))
        log.removeHandler(h)
        acc, fits, kinds = _check_decisions(name, rec.rows)
        out[f"{name}/accepted"] = acc
        out[f"{name}/fitness"] = fits
        if rec.rows:
            print(f"{name}: {len(rec.rows)} decisions pinned ({kinds}), {len(acc)} accepted")
        out[f"{name}/anchors"] = np.asarray(res, dtype=np.float64)
        out[f"{name}/log"] = np.array("\x00".join(h.lines))
        out[f"{name}/py_state"] = np.array(repr(random.getstate()))
        out[f"{name}/np_state"] = np.asarray(np.random.get_state()[1])
        out[f"{name}/np_pos"] = np.array(np.random.get_state()[2])
        out[f"{name}/error"] = np.array(err)
        print(name, err or np.round(res, 1).tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "autoanchor.npz"), **out)


if __name__ == "__main__":
    main()
