"""Writes tests/golden/v5val.npz: YOLOv5's rect validation batches and val.py's rescale on the seeded cases of
tests/v5val_cases.py.  letterbox, scale_coords, clip_coords, xywh2xyxy, xywhn2xyxy and xyxy2xywhn are the unmodified
reference's (yolort/v5/utils); upstream v6.0's loader is not in the reference tree, so its rect block, load_image
(cv2.resize, INTER_AREA when it shrinks) and __getitem__ + collate_fn are restated here in upstream's order.
Stored:

    lb/<k>/sha256, lb/<k>/ratio, lb/<k>/pad, lb/<k>/shape   letterbox of LETTERBOX case k (BGR HWC)
    sc/coords, sc/shape0, sc/shape1, sc/ratio_pad, sc/out, sc/out_auto   scale_coords on CPU float32 tensors
    sc/xywh, sc/xyxy                                        xywh2xyxy
    ds/<name>/irect, ds/<name>/batch_shapes                 the rect block
    ds/<name>/<b>/sha256                                    per sample of batch b: sha256 of the CHW RGB image
    ds/<name>/<b>/targets, ds/<name>/<b>/shapes             collate_fn's targets, shapes as [h0, w0, gh, gw, dw, dh]

    python oracle/make_golden_v5val.py
"""
import hashlib
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5val_cases as C  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "v5val.npz")


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    import_reference()
    from yolort.v5.utils.augmentations import letterbox
    from yolort.v5.utils.general import clip_coords, scale_coords, xywh2xyxy, xywhn2xyxy, xyxy2xywhn

    z = {}
    for k, (_, (h, w), kw) in enumerate(C.LETTERBOX):
        im, ratio, pad = letterbox(C.image(h, w, 500 + k), **kw)
        z[f"lb/{k}/sha256"], z[f"lb/{k}/shape"] = sha(im), np.array(im.shape)
        z[f"lb/{k}/ratio"], z[f"lb/{k}/pad"] = np.array(ratio, np.float64), np.array(pad, np.float64)
    rng = np.random.default_rng(7)
    coords = rng.uniform(-20, 700, (64, 4)).astype(np.float32)
    coords[5, 1] = np.nan
    shape1, shape0, ratio_pad = (480, 672), (750, 1000), ((0.64, 0.64), (16.0, 0.0))
    z["sc/coords"], z["sc/shape1"], z["sc/shape0"] = coords, np.array(shape1), np.array(shape0)
    z["sc/ratio_pad"] = np.array([ratio_pad[0][0], ratio_pad[1][0], ratio_pad[1][1]])
    z["sc/out"] = scale_coords(shape1, torch.from_numpy(coords.copy()), shape0, ratio_pad).numpy()
    z["sc/out_auto"] = scale_coords(shape1, torch.from_numpy(coords.copy()), shape0).numpy()
    clipped = torch.from_numpy(coords.copy())
    clip_coords(clipped, (300, 400))
    z["sc/clip"] = clipped.numpy()
    z["sc/xywh"] = rng.uniform(0, 600, (32, 4)).astype(np.float32)
    z["sc/xyxy"] = xywh2xyxy(torch.from_numpy(z["sc/xywh"])).numpy()
    for name, (sizes, img_size, bs, stride, _, pad) in C.DATASETS.items():
        images, labels = C.dataset(name)
        # LoadImagesAndLabels.__init__, rect block (v6.0)
        s = np.array([(w, h) for h, w in sizes], dtype=np.float64)
        n = len(s)
        bi = np.floor(np.arange(n) / bs).astype(int)
        nb = bi[-1] + 1
        ar = s[:, 1] / s[:, 0]
        irect = ar.argsort()
        ims = [images[i] for i in irect]
        labs = [labels[i] for i in irect]
        ar = ar[irect]
        shapes = [[1, 1]] * nb
        for i in range(nb):
            ari = ar[bi == i]
            mini, maxi = ari.min(), ari.max()
            if maxi < 1:
                shapes[i] = [maxi, 1]
            elif mini > 1:
                shapes[i] = [1, 1 / mini]
        batch_shapes = np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
        z[f"ds/{name}/irect"], z[f"ds/{name}/batch_shapes"] = irect, batch_shapes
        for b in range(nb):
            items = []
            for index in np.nonzero(bi == b)[0]:
                im = ims[index]
                h0, w0 = im.shape[:2]
                r = img_size / max(h0, w0)
                if r != 1:
                    im = cv2.resize(im, (int(w0 * r), int(h0 * r)),
                                    interpolation=cv2.INTER_AREA if r < 1 else cv2.INTER_LINEAR)
                h, w = im.shape[:2]
                img, ratio, pd = letterbox(im, batch_shapes[bi[index]], auto=False, scaleup=False)
                lab = labs[index].copy()
                if lab.size:
                    lab[:, 1:] = xywhn2xyxy(lab[:, 1:], ratio[0] * w, ratio[1] * h, padw=pd[0], padh=pd[1])
                if len(lab):
                    lab[:, 1:5] = xyxy2xywhn(lab[:, 1:5], w=img.shape[1], h=img.shape[0], clip=True, eps=1E-3)
                out = np.zeros((len(lab), 6), np.float32)
                out[:, 1:] = lab
                img = np.ascontiguousarray(img.transpose((2, 0, 1))[::-1])
                items.append((img, out, [h0, w0, h / h0, w / w0, pd[0], pd[1]]))
            for i, it in enumerate(items):       # collate_fn
                it[1][:, 0] = i
            z[f"ds/{name}/{b}/sha256"] = np.array([sha(it[0]) for it in items])
            z[f"ds/{name}/{b}/targets"] = np.concatenate([it[1] for it in items], 0)
            z[f"ds/{name}/{b}/shapes"] = np.array([it[2] for it in items], np.float64)
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
