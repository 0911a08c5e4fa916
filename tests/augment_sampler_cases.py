"""Inputs of the device parameter sampler's tests (tests/test_augment_sampler.py on the CPU,
tests/test_gpu_augment_sampler.py): seeded batches whose labels name their boxes, an image with 300 boxes, and a
transform list with non-default parameters."""
import torch

import augment_cases as AC
from yolort_b200.data import transforms as T


def many_boxes(h=480, w=640, n=300, seed=0):
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * torch.tensor([w - 8.0, h - 8.0])
    wh = torch.rand(n, 2, generator=g) * torch.tensor([w / 3, h / 3]) + 1
    boxes = torch.cat([xy, torch.minimum(xy + wh, torch.tensor([float(w), float(h)]))], 1)
    return {"boxes": boxes, "labels": torch.arange(n, dtype=torch.int64)}


def custom_transforms():
    """Non-default parameters: a narrower photometric distort without contrast, a coloured zoom-out, two IoU crops."""
    return [T.RandomPhotometricDistort(contrast=(1.0, 1.0), hue=(-0.1, 0.2), p=0.8),
            T.RandomZoomOut(fill=[10, 200, 30], side_range=(1.5, 2.5), p=0.7),
            T.RandomIoUCrop(min_scale=0.1, max_scale=0.9, min_aspect_ratio=0.3, max_aspect_ratio=3.0,
                            sampler_options=[0.2, 0.6, 1.0], trials=7),
            T.RandomIoUCrop(sampler_options=[0.0, 0.5, 2.0], trials=50),
            T.RandomHorizontalFlip(p=0.3), T.PILToTensor()]


def sampler_cases():
    """(name, transforms, sizes, targets) of the batches the sampler is checked on (here and on the GPU)."""
    def batch(seed):     # labels that name their box, so the tests can follow each box
        images, targets = AC.batch(seed)
        return ([tuple(im.shape[1:]) for im in images],
                [dict(t, labels=torch.arange(len(t["labels"])) + 100 * k) for k, t in enumerate(targets)])

    cases = [(f"seed{seed}", T.default_train_transforms().transforms) + batch(seed) for seed in AC.SEEDS]
    cases.append(("300 boxes", T.default_train_transforms().transforms, [(480, 640), (97, 131)],
                  [many_boxes(), {"boxes": AC.target(0, 2, 97, 131)["boxes"],
                                  "labels": torch.arange(len(AC.target(0, 2, 97, 131)["boxes"])) + 1000}]))
    sizes, targets = batch(3)
    cases.append(("custom", custom_transforms(), sizes + [(480, 640)], targets + [many_boxes(seed=1)]))
    return cases


CASES = sampler_cases()
