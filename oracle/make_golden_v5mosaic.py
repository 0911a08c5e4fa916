"""Writes tests/golden/v5mosaic.npz: YOLOv5's mosaic training batches (the augment=True, rect=False branch of upstream
v6.0's LoadImagesAndLabels.__getitem__ and collate_fn) on the seeded dataset of tests/v5mosaic_cases.py.  The
reference tree does not vendor the loader, so its steps are restated here as upstream v6.0 orders them; every step
calls the unmodified reference's functions (yolort/v5/utils/augmentations.py: letterbox, random_perspective, mixup,
augment_hsv; yolort/v5/utils/general.py: xywhn2xyxy, xyxy2xywhn) or cv2 (cv2.resize, the numpy mosaic canvas).
Stored per case c, each after random.seed(seed); np.random.seed(seed):

    c/draws, c/kinds        every value drawn, in order, and the call that drew it
    c/py_state, c/np_state  random.getstate() and np.random.get_state() after the batch
    c/sha256                the sha256 of collate_fn's uint8 [N, 3, s, s] RGB images (C order)
    c/targets               collate_fn's float32 [n, 6] targets
    load/<k>/sha256, load/<k>/shape   load_image of dataset image k
    load_mosaic/sha256, load_mosaic/labels   load_mosaic(5) after seed 9 (BGR [s, s, 3], labels xyxy)

    python oracle/make_golden_v5mosaic.py
"""
import hashlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import v5mosaic_cases as MC  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "v5mosaic.npz")


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Loader:
    """Upstream v6.0's LoadImagesAndLabels(augment=True, rect=False) over in-memory images."""

    def __init__(self, ims, labels, s, hyp):
        import cv2
        from yolort.v5.utils import augmentations as A
        from yolort.v5.utils import general as G

        self.cv2, self.A, self.G = cv2, A, G
        self.ims, self.labels, self.img_size, self.hyp = ims, labels, s, hyp
        self.n = len(ims)
        self.indices = range(self.n)
        self.mosaic_border = [-s // 2, -s // 2]

    def load_image(self, i):
        im = self.ims[i]
        h0, w0 = im.shape[:2]
        r = self.img_size / max(h0, w0)
        if r != 1:
            im = self.cv2.resize(im, (int(w0 * r), int(h0 * r)), interpolation=self.cv2.INTER_LINEAR)
        return im, (h0, w0), im.shape[:2]

    def load_mosaic(self, index):
        labels4 = []
        s = self.img_size
        yc, xc = [int(random.uniform(-x, 2 * s + x)) for x in self.mosaic_border]  # mosaic center x, y
        indices = [index] + random.choices(self.indices, k=3)  # 3 additional image indices
        random.shuffle(indices)
        for i, index in enumerate(indices):
            img, _, (h, w) = self.load_image(index)
            if i == 0:  # top left
                img4 = np.full((s * 2, s * 2, img.shape[2]), 114, dtype=np.uint8)
                x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
                x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h
            elif i == 1:  # top right
                x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
                x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
            elif i == 2:  # bottom left
                x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
                x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, w, min(y2a - y1a, h)
            else:  # bottom right
                x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
                x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
            img4[y1a:y2a, x1a:x2a] = img[y1b:y2b, x1b:x2b]
            padw, padh = x1a - x1b, y1a - y1b
            labels = self.labels[index].copy()
            if labels.size:
                labels[:, 1:] = self.G.xywhn2xyxy(labels[:, 1:], w, h, padw, padh)
            labels4.append(labels)
        labels4 = np.concatenate(labels4, 0)
        np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
        img4, labels4, _ = self.A.copy_paste(img4, labels4, [], p=self.hyp["copy_paste"])
        hyp = self.hyp
        return self.A.random_perspective(img4, labels4, [], degrees=hyp["degrees"], translate=hyp["translate"],
                                         scale=hyp["scale"], shear=hyp["shear"], perspective=hyp["perspective"],
                                         border=self.mosaic_border)

    def __getitem__(self, index):
        hyp = self.hyp
        if random.random() < hyp["mosaic"]:
            img, labels = self.load_mosaic(index)
            if random.random() < hyp["mixup"]:
                img, labels = self.A.mixup(img, labels, *self.load_mosaic(random.randint(0, self.n - 1)))
        else:
            img, (h0, w0), (h, w) = self.load_image(index)
            img, ratio, pad = self.A.letterbox(img, self.img_size, auto=False, scaleup=True)
            labels = self.labels[index].copy()
            if labels.size:
                labels[:, 1:] = self.G.xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0],
                                                  padh=pad[1])
            img, labels = self.A.random_perspective(img, labels, degrees=hyp["degrees"], translate=hyp["translate"],
                                                    scale=hyp["scale"], shear=hyp["shear"],
                                                    perspective=hyp["perspective"])
        nl = len(labels)
        if nl:
            labels[:, 1:5] = self.G.xyxy2xywhn(labels[:, 1:5], w=img.shape[1], h=img.shape[0], clip=True, eps=1E-3)
        self.A.augment_hsv(img, hgain=hyp["hsv_h"], sgain=hyp["hsv_s"], vgain=hyp["hsv_v"])
        if random.random() < hyp["flipud"]:
            img = np.flipud(img)
            if nl:
                labels[:, 2] = 1 - labels[:, 2]
        if random.random() < hyp["fliplr"]:
            img = np.fliplr(img)
            if nl:
                labels[:, 1] = 1 - labels[:, 1]
        labels_out = np.zeros((nl, 6), np.float32)
        if nl:
            labels_out[:, 1:] = labels
        img = img.transpose((2, 0, 1))[::-1]  # HWC to CHW, BGR to RGB
        return np.ascontiguousarray(img), labels_out

    @staticmethod
    def collate_fn(batch):
        img, label = zip(*batch)
        for i, lab in enumerate(label):
            lab[:, 0] = i  # add target image index for build_targets()
        return np.stack(img, 0), np.concatenate(label, 0)


def main():
    import_reference()
    ims, labs = MC.dataset()
    arrays = {}
    for case in MC.CASES:
        name = case["name"]
        loader = Loader(ims, labs, MC.S, MC.hyp(case))
        random.seed(case["seed"])
        np.random.seed(case["seed"])
        with MC.DrawLog() as log:
            imgs, targets = Loader.collate_fn([loader[i] for i in case["indices"]])
        arrays[f"{name}/py_state"], arrays[f"{name}/np_state"] = MC.generator_states()
        arrays[f"{name}/draws"] = np.array(log.values, np.float64)
        arrays[f"{name}/kinds"] = np.array(log.kinds)
        arrays[f"{name}/sha256"] = np.array(sha(imgs))
        arrays[f"{name}/shape"] = np.array(imgs.shape, np.int64)
        arrays[f"{name}/targets"] = targets
    loader = Loader(ims, labs, MC.S, MC.SCRATCH)
    for k in range(len(ims)):
        im = loader.load_image(k)[0]
        arrays[f"load/{k}/sha256"] = np.array(sha(im))
        arrays[f"load/{k}/shape"] = np.array(im.shape, np.int64)
    random.seed(9)
    np.random.seed(9)
    img4, labels4 = loader.load_mosaic(5)
    arrays["load_mosaic/sha256"] = np.array(sha(img4))
    arrays["load_mosaic/labels"] = labels4
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, len(arrays), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
