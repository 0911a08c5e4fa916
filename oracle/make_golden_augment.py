"""Writes tests/golden/augment.npz: the unmodified reference default_train_transforms()
(yolort/data/transforms.py:21-32) on the seeded uint8 tensor images of tests/augment_cases.py, image by image after one
torch.manual_seed per case, and the reference YOLOTransform(images, targets) target batch of the result.  The tensor
path is used, not PIL: the reference's PILToTensor only accepts PIL images, so it is dropped from the list (on a tensor
it would be the identity).  Inputs are regenerated from their seeds; stored per case s and image k:

    s<s>/draws, s<s>/kinds   every value drawn from the default generator, in order, and the call that drew it
    s<s>/rand_after          torch.rand(1) right after the last image
    s<s>/<k>/shape           the output [3, H, W]
    s<s>/<k>/sha256          sha256 of the fp32 output bytes (C order)
    s<s>/<k>/u8              the output * 255 as uint8, for images of at most U8_MAX elements
    s<s>/<k>/boxes, labels   the output target
    s<s>/targets_batched     YOLOTransform(*augment_cases.LETTERBOX)(images, targets)[1]

    python oracle/make_golden_augment.py
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import augment_cases as AC  # noqa: E402
from oracle.ref_import import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
U8_MAX = 40000


def main():
    import_reference()
    from yolort.data import transforms as T
    from yolort.models.transform import YOLOTransform

    arrays = {}
    for s in AC.SEEDS:
        images, targets = AC.batch(s)
        pipe = T.default_train_transforms()
        pipe.transforms = [t for t in pipe.transforms if not isinstance(t, T.PILToTensor)]
        torch.manual_seed(s)
        outs = []
        with AC.DrawLog() as log:
            for im, tg in zip(images, targets):
                outs.append(pipe(im.clone(), {k: v.clone() for k, v in tg.items()}))
        arrays[f"s{s}/rand_after"] = torch.rand(1).numpy()
        arrays[f"s{s}/draws"] = np.array(log.values, np.float64)
        arrays[f"s{s}/kinds"] = np.array(log.kinds)
        for k, (im, tg) in enumerate(outs):
            assert im.dtype == torch.float32
            a = im.numpy()
            u8 = np.round(a * 255).astype(np.uint8)
            assert np.array_equal(u8.astype(np.float32) / np.float32(255), a)
            arrays[f"s{s}/{k}/shape"] = np.array(a.shape, np.int64)
            arrays[f"s{s}/{k}/sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest())
            if u8.size <= U8_MAX:
                arrays[f"s{s}/{k}/u8"] = u8
            arrays[f"s{s}/{k}/boxes"] = tg["boxes"].numpy()
            arrays[f"s{s}/{k}/labels"] = tg["labels"].numpy()
        lb = YOLOTransform(*AC.LETTERBOX)
        _, tb = lb([im for im, _ in outs], [{k: v.clone() for k, v in tg.items()} for _, tg in outs])
        arrays[f"s{s}/targets_batched"] = tb.numpy()
    np.savez_compressed(os.path.join(OUT, "augment.npz"), **arrays)
    print("wrote", os.path.join(OUT, "augment.npz"), len(arrays), "arrays")


if __name__ == "__main__":
    main()
