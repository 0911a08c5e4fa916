"""Writes tests/golden/v5aug.npz: the unmodified reference's YOLOv5 augmentations
(yolort/v5/utils/augmentations.py: augment_hsv, random_perspective, cutout, mixup) through cv2 on the seeded cases of
tests/v5aug_cases.py, each after random.seed(s); np.random.seed(s), and the digests of cv2's full colour tables.
Inputs are regenerated from their seeds; stored per case c:

    c/draws, c/kinds       every value drawn from `random` / `np.random`, in order, and the call that drew it
    c/after                random.random() and np.random.random() right after the call
    c/shape, c/sha256      the output image's shape and the sha256 of its bytes (C order)
    c/out                  the output image, for outputs of at most OUT_MAX bytes
    c/labels_in, c/labels  the labels before and after
    tables/<name>          sha256 of cv2.cvtColor over oracle/restate_v5aug.py's all_bgr_image / all_hsv_image(w)

    python oracle/make_golden_v5aug.py
"""
import hashlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5aug_cases as VC  # noqa: E402
from oracle import restate_v5aug as R  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "v5aug.npz")
OUT_MAX = 12000


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def tables():
    import cv2

    out = {}
    bgr = R.all_bgr_image()
    out["tables/to_hsv_bgr"] = sha(cv2.cvtColor(bgr, cv2.COLOR_BGR2HSV))
    out["tables/to_hsv_rgb"] = sha(cv2.cvtColor(bgr, cv2.COLOR_RGB2HSV))
    for w in (256, 1):
        hsv = R.all_hsv_image(w)
        out[f"tables/from_hsv_bgr_w{w}"] = sha(cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR))
        out[f"tables/from_hsv_rgb_w{w}"] = sha(cv2.cvtColor(hsv, cv2.COLOR_HSV2RGB))
    for rgb in (False, True):  # the round trip of every triple with identity tables
        code = (cv2.COLOR_RGB2HSV, cv2.COLOR_HSV2RGB) if rgb else (cv2.COLOR_BGR2HSV, cv2.COLOR_HSV2BGR)
        out[f"tables/round_trip_{'rgb' if rgb else 'bgr'}"] = sha(cv2.cvtColor(cv2.cvtColor(bgr, code[0]), code[1]))
    return out


def main():
    import_reference()
    from yolort.v5.utils import augmentations as A

    arrays = {k: np.array(v) for k, v in tables().items()}
    for case in VC.CASES:
        name, fn = case["name"], case["fn"]
        im, labels, extra = VC.inputs(case)
        random.seed(case["seed"])
        np.random.seed(case["seed"])
        with VC.DrawLog() as log:
            if fn == "augment_hsv":
                out = im.copy()
                A.augment_hsv(out, **case["kw"])
                lab = labels
            elif fn == "random_perspective":
                out, lab = A.random_perspective(im.copy(), labels.copy(), **case["kw"])
            elif fn == "cutout":
                out = im.copy()
                lab = A.cutout(out, labels.copy(), **case["kw"])
            else:
                im2, labels2 = extra
                out, lab = A.mixup(im.copy(), labels.copy(), im2, labels2)
        arrays[f"{name}/after"] = np.array([random.random(), np.random.random()])
        arrays[f"{name}/draws"] = np.array(log.values, np.float64)
        arrays[f"{name}/kinds"] = np.array(log.kinds)
        arrays[f"{name}/shape"] = np.array(out.shape, np.int64)
        arrays[f"{name}/sha256"] = np.array(sha(out))
        if out.size <= OUT_MAX:
            arrays[f"{name}/out"] = out
        arrays[f"{name}/labels_in"] = labels
        arrays[f"{name}/labels"] = np.asarray(lab)
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, len(arrays), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
