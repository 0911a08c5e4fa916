"""Training-augmentation inputs shared by oracle/make_golden_augment.py, tests/test_augment.py (CPU) and
tests/test_gpu_augment.py: seeded uint8 [3, H, W] images and xyxy targets, regenerated rather than stored.  Every batch
has an odd-sized image, an image without boxes and an image whose boxes touch the border.  Pixel counts stay below
2^24 / 255, so torch's fp32 mean of the grayscale image is exact and the contrast op is bit-identical to it."""
import torch

SEEDS = (0, 1, 2, 3, 4, 5)
SIZES = ((97, 131), (64, 64), (150, 203), (33, 47))
NO_BOXES = 1          # the image of SIZES without boxes
BORDER = 2            # the image whose boxes touch the border
# YOLOTransform of the target-batch fixture
LETTERBOX = (128, 160)


def image(seed: int, k: int, h: int, w: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(1000 * seed + k)
    # a smooth gradient plus noise, so the channels differ and grayscale / hue see every kind of pixel
    yy = torch.arange(h).view(1, h, 1).float() / max(h - 1, 1)
    xx = torch.arange(w).view(1, 1, w).float() / max(w - 1, 1)
    base = torch.stack([yy[0].expand(h, w), xx[0].expand(h, w), (yy[0] + xx[0]).expand(h, w) / 2]) * 255
    noise = torch.randint(-40, 41, (3, h, w), generator=g).float()
    return (base + noise).clamp(0, 255).to(torch.uint8)


def target(seed: int, k: int, h: int, w: int):
    g = torch.Generator().manual_seed(7919 * seed + k + 1)
    n = 0 if k == NO_BOXES else int(torch.randint(1, 6, (1,), generator=g))
    xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.7, h * 0.7])
    wh = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.6, h * 0.6]) + 2
    boxes = torch.cat([xy, torch.minimum(xy + wh, torch.tensor([float(w), float(h)]))], 1)
    if k == BORDER and n:
        boxes[0, 0], boxes[0, 1] = 0.0, 0.0
        boxes[-1, 2], boxes[-1, 3] = float(w), float(h)
    labels = torch.randint(0, 80, (n,), generator=g)
    return {"boxes": boxes.to(torch.float32), "labels": labels}


def batch(seed: int):
    """(images, targets) of one case: uint8 CPU images, fp32 / int64 CPU targets."""
    images = [image(seed, k, h, w) for k, (h, w) in enumerate(SIZES)]
    targets = [target(seed, k, h, w) for k, (h, w) in enumerate(SIZES)]
    return images, targets


class DrawLog:
    """Records every value drawn from torch's default generator through torch.rand / randint / randperm and
    Tensor.uniform_ while active: the calls the reference's transforms make."""

    def __init__(self):
        self.kinds, self.values = [], []

    def __enter__(self):
        self._saved = (torch.rand, torch.randint, torch.randperm, torch.Tensor.uniform_)
        rand, randint, randperm, uniform_ = self._saved

        def wrap(kind, fn):
            def f(*a, **k):
                out = fn(*a, **k)
                self.kinds.append(kind)
                self.values.extend(float(v) for v in out.reshape(-1).tolist())
                return out
            return f

        torch.rand, torch.randint, torch.randperm = wrap("rand", rand), wrap("randint", randint), wrap("randperm", randperm)
        torch.Tensor.uniform_ = wrap("uniform_", uniform_)
        return self

    def __exit__(self, *a):
        torch.rand, torch.randint, torch.randperm, torch.Tensor.uniform_ = self._saved
        return False
