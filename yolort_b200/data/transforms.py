"""The reference's training augmentations (yolort/data/transforms.py:17-336) on the GPU.

Same names, constructor signatures and call contract: each transform is called as `t(image, target)` and returns
`(image, target)`.  Images are CUDA uint8 `[3, H, W]` tensors (for example `yolort_b200.io.decode_jpeg`'s output, read
in place whatever its strides); targets are `{"boxes": [n, 4] xyxy pixels, "labels": [n], ...}` on the CPU or the GPU.

The parity target is the reference applied to uint8 TENSORS, which takes torchvision's tensor arithmetic
(torchvision/transforms/_functional_tensor.py), not PIL's `ImageEnhance` arithmetic.  Under `torch.manual_seed(s)` a
sequence of calls draws the same random numbers as the reference and gives the same pixels, boxes and labels.

How it runs:
- Every random parameter is drawn on the host from torch's default CPU generator, in the reference's order, before any
  pixel is touched; box arithmetic runs on a host copy in the reference's fp32 operations and order (one copy per
  batch for device targets).
- Each image's draws become a recipe: pointwise colour ops, channel permutations, zoom-out, crop and flip in call
  order.  `csrc/augment.cu` computes every output pixel of the batch in one launch (plus one launch of the contrast
  mean per contrast round), into one device buffer; the outputs are views into it.
- `ConvertImageDtype(torch.float)` (or `ToTensor`) as the last transform is the kernel's output dtype: byte / 255.0
  with IEEE division, as torchvision computes it.

Differences from the reference: a PIL image raises TypeError, a non-uint8 or non-3-D image ValueError, a CPU image
NativeLibraryError (there is no CPU path); targets with "masks" or "keypoints" raise NotImplementedError.  The
caller's target tensors are not modified in place (the reference's zoom-out and flip write into them).

`Compose.apply_batch(images, targets, generator=g)` with a CUDA `torch.Generator` draws the parameters on the device
instead (`csrc/augment_sample.cu`): the reference's transforms, parameter distributions and acceptance rules on a
Philox4x32-10 stream keyed by one draw from `g`, so `g.manual_seed(s)` reproduces a batch.  It does not reproduce the
reference's random numbers and does not touch torch's default generator; oracle/sample_augment.py restates its rules.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torchvision
from torch import nn, Tensor

from .. import _C

__all__ = ["collate_fn", "default_train_transforms", "default_val_transforms", "Compose", "RandomPhotometricDistort",
           "RandomZoomOut", "RandomIoUCrop", "RandomHorizontalFlip", "PILToTensor", "ToTensor", "ConvertImageDtype"]


def collate_fn(batch):
    return tuple(zip(*batch))


def default_train_transforms(hflip_prob=0.5):
    return Compose([
        RandomPhotometricDistort(),
        RandomZoomOut(),
        RandomIoUCrop(),
        RandomHorizontalFlip(p=hflip_prob),
        PILToTensor(),
        ConvertImageDtype(torch.float),
    ])


def default_val_transforms():
    return ToTensor()


class _State:
    """One image while its parameters are drawn: current size, host boxes / labels, recipe, output dtype."""

    def __init__(self, hw: Tuple[int, int], target: Optional[Dict[str, Tensor]]):
        self.h, self.w = hw
        self.target = target
        self.ops: List[tuple] = []
        self.float_out = False


class _Transform(nn.Module):
    """An augmentation the native recipe can express.  Called alone it is `Compose([self])`."""

    def _draw(self, st: _State) -> None:
        raise NotImplementedError

    def _sampler(self, s: "_C.AugSampler") -> Tuple[int, int]:
        """Describes the transform to the device sampler in `s`; returns the most ops and contrast ops it can add to
        a recipe."""
        raise TypeError(f"{type(self).__name__} has no device sampler")

    def forward(self, image: Tensor, target: Optional[Dict[str, Tensor]] = None):
        return Compose([self])(image, target)


class Compose:
    def __init__(self, transforms):
        self.transforms = transforms

    def __call__(self, image, target=None):
        images, targets = self.apply_batch([image], [target])
        return images[0], targets[0]

    # -- host side: parameters, boxes and recipes (no device work) -----------------------------------------------
    def _check_transforms(self) -> None:
        for i, t in enumerate(self.transforms):
            if not isinstance(t, _Transform):
                raise TypeError(f"Compose: transform {i} ({type(t).__name__}) is not one of "
                                "yolort_b200.data.transforms' augmentations")
            if isinstance(t, ConvertImageDtype) and t.dtype != torch.uint8 and i != len(self.transforms) - 1:
                raise NotImplementedError("ConvertImageDtype(float) / ToTensor must be the last transform: the "
                                          "recipes compute on uint8 images")

    def plan(self, sizes: Sequence[Tuple[int, int]], targets: Sequence[Optional[Dict[str, Tensor]]]):
        """Draws every image's parameters in turn (image 0's transforms, then image 1's, ...: what calling the
        reference Compose image by image draws) and applies them to host copies of the targets.  Returns the states:
        output size, recipe and target of each image."""
        self._check_transforms()
        states = []
        for hw, tg in zip(sizes, targets):
            st = _State(hw, tg)
            for t in self.transforms:
                t._draw(st)
            states.append(st)
        return states

    # -- the batch -------------------------------------------------------------------------------------------
    def apply_batch(self, images: Sequence[Tensor], targets: Optional[Sequence[Optional[Dict[str, Tensor]]]] = None,
                    generator: Optional[torch.Generator] = None):
        """Augments a batch: the parameters of every image are drawn as `plan` does, then all pixels are computed
        at once.  Returns (images, targets); the images are views into one device buffer.

        With `generator` (a CUDA torch.Generator on the images' device) the parameters are drawn on the device from
        one 64-bit key taken from it (see `sample`); torch's default generator is not used."""
        images = list(images)
        if not images:
            return [], []
        targets = [None] * len(images) if targets is None else list(targets)
        if len(targets) != len(images):
            raise ValueError(f"{len(images)} images and {len(targets)} targets")
        if generator is not None:
            descs, out_targets = self.sample(images, targets, generator)
            return _run_descs(images, descs, self._float_out()), out_targets
        for im in images:
            _check_image(im)
        dev = images[0].device
        for im in images:
            if im.device != dev:
                raise ValueError("apply_batch: every image must be on the same device")
        host_targets, target_dev = _host_targets(targets)
        states = self.plan([(int(im.shape[1]), int(im.shape[2])) for im in images], host_targets)
        return run_recipes(images, states), _device_targets(states, targets, target_dev)

    # -- the device sampler ----------------------------------------------------------------------------------
    def _float_out(self) -> bool:
        float_out = False
        for t in self.transforms:
            if isinstance(t, ConvertImageDtype):
                float_out = t.dtype == torch.float32
        return float_out

    def _sampler_table(self) -> "ctypes.Array":
        """The transforms as yb_aug_sampler entries.  Raises what `plan` raises for a transform list it cannot run,
        TypeError for a transform without a device sampler and NotImplementedError when some recipe could exceed the
        descriptor's YB_AUG_MAX_OPS ops or YB_AUG_MAX_CONTRAST contrast ops (a bound from the list, not the draws)."""
        self._check_transforms()
        if len(self.transforms) > _C.YB_AUG_MAX_TRANSFORMS:
            raise NotImplementedError(f"{len(self.transforms)} transforms (the device sampler takes at most "
                                      f"{_C.YB_AUG_MAX_TRANSFORMS})")
        table = (_C.AugSampler * len(self.transforms))()
        ops = contrast = 0
        for s, t in zip(table, self.transforms):
            o, c = t._sampler(s)
            ops, contrast = ops + o, contrast + c
        if ops > _C.YB_AUG_MAX_OPS or contrast > _C.YB_AUG_MAX_CONTRAST:
            raise NotImplementedError(f"the transforms can draw a recipe of {ops} ops with {contrast} contrast ops (at "
                                      f"most {_C.YB_AUG_MAX_OPS} and {_C.YB_AUG_MAX_CONTRAST})")
        return table

    def sample(self, images: Sequence[Tensor], targets: Sequence[Optional[Dict[str, Tensor]]],
               generator: torch.Generator):
        """Draws every image's parameters on the device and carries its boxes through them; no pixel is computed.
        Returns (descriptors, targets): the yb_aug_image recipes `apply_batch` computes the pixels from, and each
        target with its kept boxes and labels on the device it came from (other keys pass through).  Every input
        error is raised before anything is drawn; the read-back of the descriptors is the one host synchronisation."""
        table = self._sampler_table()
        need_target = any(isinstance(t, RandomIoUCrop) for t in self.transforms)
        boxes, labels = _sampled_boxes(targets, need_target)
        _check_generator(generator)
        for im in images:
            _check_image(im)
        dev = images[0].device
        if any(im.device != dev for im in images):
            raise ValueError("apply_batch: every image must be on the same device")
        _check_generator(generator, dev)
        to_host = any(t is not None and t["boxes"].device.type == "cpu" for t in targets)
        descs, counts, status, out_boxes, out_labels = _C.augment_sample(table, images, _draw_key(generator, dev),
                                                                        boxes, labels, to_host)
        failed = [i for i, s in enumerate(status) if s & _C.YB_AUG_ST_CROP_ROUNDS]
        if failed:
            raise RuntimeError(f"RandomIoUCrop accepted no window in {_C.YB_AUG_CROP_ROUNDS} rounds for image(s) "
                               f"{failed}: no box centre lies inside any window its options allow")
        out, row = [], 0
        for t, b, l, c in zip(targets, boxes, labels, counts):
            if t is not None:
                t = dict(t)
                t["boxes"] = out_boxes[row: row + c].to(b.device)
                t["labels"] = out_labels[row: row + c].to(l.device)
            row += int(b.shape[0])
            out.append(t)
        return descs, out


def _check_generator(generator, dev: Optional[torch.device] = None) -> None:
    if not isinstance(generator, torch.Generator) or generator.device.type != "cuda":
        got = generator.device if isinstance(generator, torch.Generator) else type(generator).__name__
        raise ValueError(f"generator must be a CUDA torch.Generator on the images' device, got {got}")
    idx = lambda d: torch.cuda.current_device() if d.index is None else d.index  # noqa: E731
    if dev is not None and idx(generator.device) != idx(dev):
        raise ValueError(f"generator is on {generator.device}, the images on {dev}")


def _draw_key(generator: torch.Generator, dev: torch.device) -> Tensor:
    """The call's Philox key: two 32-bit words drawn by a device op, so the host never reads the generator's state."""
    return torch.empty(2, dtype=torch.int64, device=dev).random_(0, 1 << 32, generator=generator)


def _sampled_boxes(targets, need_target: bool):
    """The boxes and labels of each image, checked for the device sampler (none for an image without a target)."""
    boxes, labels = [], []
    for i, t in enumerate(targets):
        if t is None:
            if need_target:
                raise ValueError(f"image {i} has no target: RandomIoUCrop needs one")
            boxes.append(torch.zeros((0, 4), dtype=torch.float32))
            labels.append(torch.zeros((0,), dtype=torch.int64))
            continue
        for key in ("masks", "keypoints"):
            if key in t:
                raise NotImplementedError(f"targets with {key!r} are not supported by the GPU augmentations")
        if "boxes" not in t or "labels" not in t:
            raise ValueError("a target must hold 'boxes' and 'labels'")
        b, l = t["boxes"], t["labels"]
        if not (isinstance(b, Tensor) and b.dtype == torch.float32 and b.dim() == 2 and b.shape[1] == 4):
            raise ValueError(f"image {i}: boxes must be a float32 [n, 4] tensor")
        if not (isinstance(l, Tensor) and l.dtype == torch.int64 and l.shape == (b.shape[0],)):
            raise ValueError(f"image {i}: labels must be an int64 [n] tensor with one label per box")
        boxes.append(b)
        labels.append(l)
    return boxes, labels


def run_recipes(images: Sequence[Tensor], states: Sequence["_State"]) -> List[Tensor]:
    """Computes the planned images (one launch, plus one per contrast round); the outputs are views into one buffer."""
    descs = (_C.AugImage * len(images))()
    for d, im, st in zip(descs, images, states):
        _fill_desc(d, im, st)
    return _run_descs(images, descs, states[0].float_out)


def _run_descs(images: Sequence[Tensor], descs, float_out: bool) -> List[Tensor]:
    total = 0
    for d in descs:
        d.out_offset = total
        total += -(-3 * d.out_h * d.out_w // 16) * 16     # every image starts 64-byte aligned
    out = torch.empty((total,), dtype=torch.float32 if float_out else torch.uint8, device=images[0].device)
    _C.augment(descs, out, images)
    return [out[d.out_offset: d.out_offset + 3 * d.out_h * d.out_w].view(3, d.out_h, d.out_w) for d in descs]


def _check_image(im) -> None:
    if not isinstance(im, Tensor):
        raise TypeError(f"images must be uint8 [3, H, W] CUDA tensors, got {type(im).__name__} (PIL images are not "
                        "supported: decode to a tensor, e.g. with yolort_b200.io.decode_jpeg)")
    if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[0] != 3:
        raise ValueError(f"images must be uint8 [3, H, W] tensors, got {im.dtype} {tuple(im.shape)}")
    _C.require_cuda(im, "training augmentations")


def _host_targets(targets):
    """Host copies of the targets (one device-to-host copy for all device boxes and labels of the batch) and the
    device they came from."""
    dev = None
    for t in targets:
        if t is None:
            continue
        for key in ("masks", "keypoints"):
            if key in t:
                raise NotImplementedError(f"targets with {key!r} are not supported by the GPU augmentations")
        if "boxes" not in t or "labels" not in t:
            raise ValueError("a target must hold 'boxes' and 'labels'")
        if t["boxes"].is_cuda:
            dev = t["boxes"].device
    if dev is None:
        return [None if t is None else dict(t) for t in targets], None
    present = [t for t in targets if t is not None]
    boxes = torch.cat([t["boxes"].reshape(-1).to(dev) for t in present]).to("cpu", non_blocking=True)
    labels = torch.cat([t["labels"].reshape(-1).to(dev) for t in present]).to("cpu", non_blocking=True)
    torch.cuda.current_stream(dev).synchronize()
    pieces = []
    for b, l in zip(boxes.split([t["boxes"].numel() for t in present]),
                    labels.split([t["labels"].numel() for t in present])):
        pieces += [b, l]
    out, k = [], 0
    for t in targets:
        if t is None:
            out.append(None)
            continue
        h = dict(t)
        h["boxes"] = pieces[k].view(t["boxes"].shape)
        h["labels"] = pieces[k + 1].view(t["labels"].shape)
        k += 2
        out.append(h)
    return out, dev


def _device_targets(states, targets, dev):
    if dev is None:
        return [st.target for st in states]
    moved = [x for st in states if st.target is not None for x in (st.target["boxes"], st.target["labels"])]
    dmoved = [m.to(dev, non_blocking=True) for m in moved]
    out, k = [], 0
    for st in states:
        if st.target is None:
            out.append(None)
            continue
        t = dict(st.target)
        t["boxes"], t["labels"] = dmoved[k], dmoved[k + 1]
        k += 2
        out.append(t)
    return out


def _fill_desc(d: "_C.AugImage", im: Tensor, st: _State) -> None:
    if len(st.ops) > _C.YB_AUG_MAX_OPS:
        raise NotImplementedError(f"a recipe of {len(st.ops)} ops (at most {_C.YB_AUG_MAX_OPS})")
    d.src = im.data_ptr()
    d.stride_c, d.stride_y, d.stride_x = (int(v) for v in im.stride())
    d.src_h, d.src_w = int(im.shape[1]), int(im.shape[2])
    d.out_h, d.out_w = st.h, st.w
    d.n_ops = len(st.ops)
    for slot, (kind, args, factor) in zip(d.ops, st.ops):
        slot.kind = kind
        for j, a in enumerate(args):
            slot.arg[j] = int(a)
        if factor is not None:
            slot.factor = factor
            slot.one_minus = 1.0 - factor     # Python double, rounded to fp32 by ctypes: torchvision's _blend


# -- the transforms ------------------------------------------------------------------------------------------------
class RandomHorizontalFlip(_Transform):
    def __init__(self, p: float = 0.5):
        super().__init__()
        self.p = p

    def _draw(self, st: _State) -> None:
        if torch.rand(1) < self.p:
            st.ops.append((_C.YB_AUG_HFLIP, (st.w,), None))
            if st.target is not None:
                b = st.target["boxes"].clone()
                b[:, [0, 2]] = st.w - b[:, [2, 0]]
                st.target["boxes"] = b

    def _sampler(self, s) -> Tuple[int, int]:
        s.kind, s.p = _C.YB_AUG_S_HFLIP, self.p
        return 1, 0


class PILToTensor(_Transform):
    """The identity on a uint8 tensor image."""

    def _draw(self, st: _State) -> None:
        pass

    def _sampler(self, s) -> Tuple[int, int]:
        s.kind = _C.YB_AUG_S_NONE
        return 0, 0


class ConvertImageDtype(_Transform):
    def __init__(self, dtype: torch.dtype) -> None:
        super().__init__()
        if dtype not in (torch.uint8, torch.float32):
            raise NotImplementedError(f"ConvertImageDtype({dtype}): the GPU augmentations give uint8 or float32")
        self.dtype = dtype

    def _draw(self, st: _State) -> None:
        st.float_out = self.dtype == torch.float32

    def _sampler(self, s) -> Tuple[int, int]:
        s.kind = _C.YB_AUG_S_NONE
        return 0, 0


class ToTensor(ConvertImageDtype):
    """On a uint8 tensor image: ConvertImageDtype(torch.float)."""

    def __init__(self) -> None:
        super().__init__(torch.float32)


class RandomIoUCrop(_Transform):
    def __init__(self, min_scale: float = 0.3, max_scale: float = 1.0, min_aspect_ratio: float = 0.5,
                 max_aspect_ratio: float = 2.0, sampler_options: Optional[List[float]] = None, trials: int = 40):
        super().__init__()
        self.min_scale = min_scale
        self.max_scale = max_scale
        self.min_aspect_ratio = min_aspect_ratio
        self.max_aspect_ratio = max_aspect_ratio
        if sampler_options is None:
            sampler_options = [0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 1.0]
        self.options = sampler_options
        self.trials = trials

    def _draw(self, st: _State) -> None:
        if st.target is None:
            raise ValueError("The targets can't be None for this transform.")
        orig_w, orig_h = st.w, st.h
        boxes = st.target["boxes"]
        # the window arithmetic is the reference's fp32 tensor arithmetic, restated on numpy fp32 scalars (the same
        # roundings, without a torch dispatch per operation: the trial loop runs hundreds of times per batch)
        span, lo = np.float32(self.max_scale - self.min_scale), np.float32(self.min_scale)
        cx = (0.5 * (boxes[:, 0] + boxes[:, 2])).numpy()
        cy = (0.5 * (boxes[:, 1] + boxes[:, 3])).numpy()
        while True:
            idx = int(torch.randint(low=0, high=len(self.options), size=(1,)))
            min_jaccard_overlap = self.options[idx]
            if min_jaccard_overlap >= 1.0:       # leave the image as it is
                return
            for _ in range(self.trials):
                r = lo + span * torch.rand(2).numpy()
                new_w, new_h = int(np.float32(orig_w) * r[0]), int(np.float32(orig_h) * r[1])
                if not self.min_aspect_ratio <= new_w / new_h <= self.max_aspect_ratio:
                    continue
                r = torch.rand(2).numpy()
                left, top = int(np.float32(orig_w - new_w) * r[0]), int(np.float32(orig_h - new_h) * r[1])
                right, bottom = left + new_w, top + new_h
                if left == right or top == bottom:
                    continue
                inside = (left < cx) & (cx < right) & (top < cy) & (cy < bottom)
                if not inside.any():
                    continue
                inside = torch.from_numpy(inside)
                kept = boxes[inside]
                window = torch.tensor([[left, top, right, bottom]], dtype=kept.dtype)
                if torchvision.ops.boxes.box_iou(kept, window).max() < min_jaccard_overlap:
                    continue
                kept[:, 0::2] -= left
                kept[:, 1::2] -= top
                kept[:, 0::2].clamp_(min=0, max=new_w)
                kept[:, 1::2].clamp_(min=0, max=new_h)
                st.target["boxes"] = kept
                st.target["labels"] = st.target["labels"][inside]
                st.ops.append((_C.YB_AUG_CROP, (top, left, new_h, new_w), None))
                st.h, st.w = new_h, new_w
                return

    def _sampler(self, s) -> Tuple[int, int]:
        if not 0 < len(self.options) <= _C.YB_AUG_MAX_OPTIONS:
            raise NotImplementedError(f"RandomIoUCrop with {len(self.options)} sampler options (the device sampler "
                                      f"takes 1 to {_C.YB_AUG_MAX_OPTIONS})")
        s.kind, s.trials, s.n_options = _C.YB_AUG_S_IOU_CROP, int(self.trials), len(self.options)
        s.lo[0], s.span[0] = self.min_scale, self.max_scale - self.min_scale
        s.min_aspect, s.max_aspect = self.min_aspect_ratio, self.max_aspect_ratio
        for j, o in enumerate(self.options):
            s.options[j] = o
        return 1, 0


class RandomZoomOut(_Transform):
    def __init__(self, fill: Optional[List[float]] = None, side_range: Tuple[float, float] = (1.0, 4.0), p: float = 0.5):
        super().__init__()
        if fill is None:
            fill = [0.0, 0.0, 0.0]
        self.fill = fill
        self.side_range = side_range
        if side_range[0] < 1.0 or side_range[0] > side_range[1]:
            raise ValueError(f"Invalid canvas side range provided {side_range}.")
        self.p = p

    def _draw(self, st: _State) -> None:
        if torch.rand(1) >= self.p:
            return
        orig_w, orig_h = st.w, st.h
        r = self.side_range[0] + torch.rand(1) * (self.side_range[1] - self.side_range[0])
        canvas_width, canvas_height = int(orig_w * r), int(orig_h * r)
        r = torch.rand(2)
        left = int((canvas_width - orig_w) * r[0])
        top = int((canvas_height - orig_h) * r[1])
        packed = self._packed_fill()
        st.ops.append((_C.YB_AUG_ZOOM_OUT, (top, left, orig_h, orig_w, canvas_height, canvas_width, packed), None))
        st.h, st.w = canvas_height, canvas_width
        if st.target is not None:
            b = st.target["boxes"].clone()
            b[:, 0::2] += left
            b[:, 1::2] += top
            st.target["boxes"] = b

    def _packed_fill(self) -> int:
        # the reference overwrites the border with torch.tensor(fill, dtype=uint8)
        f = torch.tensor(self.fill, dtype=torch.uint8).expand(3).tolist()
        return f[0] | (f[1] << 8) | (f[2] << 16)

    def _sampler(self, s) -> Tuple[int, int]:
        s.kind, s.p, s.fill = _C.YB_AUG_S_ZOOM_OUT, self.p, self._packed_fill()
        s.lo[0], s.span[0] = self.side_range[0], self.side_range[1] - self.side_range[0]
        return 1, 0


class RandomPhotometricDistort(_Transform):
    def __init__(self, contrast: Tuple[float] = (0.5, 1.5), saturation: Tuple[float] = (0.5, 1.5),
                 hue: Tuple[float] = (-0.05, 0.05), brightness: Tuple[float] = (0.875, 1.125), p: float = 0.5):
        super().__init__()
        # torchvision's ColorJitter keeps a range unless it is the identity (ColorJitter._check_input)
        self.brightness = _jitter_range(brightness, 1.0)
        self.contrast = _jitter_range(contrast, 1.0)
        self.hue = _jitter_range(hue, 0.0)
        self.saturation = _jitter_range(saturation, 1.0)
        self.p = p

    @staticmethod
    def _jitter(st: _State, kind: int, rng) -> None:
        # one single-factor ColorJitter call: randperm(4), then one uniform_ draw (ColorJitter.get_params)
        torch.randperm(4)
        if rng is None:
            return
        factor = float(torch.empty(1).uniform_(rng[0], rng[1]))
        st.ops.append((kind, (0, st.h, st.w) if kind == _C.YB_AUG_CONTRAST else (), factor))

    def _draw(self, st: _State) -> None:
        r = torch.rand(7)
        if r[0] < self.p:
            self._jitter(st, _C.YB_AUG_BRIGHTNESS, self.brightness)
        contrast_before = r[1] < 0.5
        if contrast_before and r[2] < self.p:
            self._jitter(st, _C.YB_AUG_CONTRAST, self.contrast)
        if r[3] < self.p:
            self._jitter(st, _C.YB_AUG_SATURATION, self.saturation)
        if r[4] < self.p:
            self._jitter(st, _C.YB_AUG_HUE, self.hue)
        if not contrast_before and r[5] < self.p:
            self._jitter(st, _C.YB_AUG_CONTRAST, self.contrast)
        if r[6] < self.p:
            st.ops.append((_C.YB_AUG_PERMUTE, tuple(torch.randperm(3).tolist()), None))

    def _sampler(self, s) -> Tuple[int, int]:
        s.kind, s.p = _C.YB_AUG_S_PHOTOMETRIC, self.p
        for j, rng in enumerate((self.brightness, self.contrast, self.saturation, self.hue)):
            if rng is not None:
                s.jitter |= 1 << j
                s.lo[j], s.span[j] = rng[0], rng[1] - rng[0]
        return bin(s.jitter).count("1") + 1, int(self.contrast is not None)


def _jitter_range(value, center: float):
    lo, hi = float(value[0]), float(value[1])
    return None if lo == hi == center else (lo, hi)


def recipe_of(st: _State) -> List[tuple]:
    """The recipe of a planned image in oracle/restate_augment.py's notation (for tests and debugging)."""
    names = {_C.YB_AUG_BRIGHTNESS: "brightness", _C.YB_AUG_CONTRAST: "contrast", _C.YB_AUG_SATURATION: "saturation",
             _C.YB_AUG_HUE: "hue"}
    out = []
    for kind, args, factor in st.ops:
        if kind in names:
            out.append((names[kind], factor))
        elif kind == _C.YB_AUG_PERMUTE:
            out.append(("permute", tuple(args)))
        elif kind == _C.YB_AUG_ZOOM_OUT:
            top, left, _, _, ch, cw, f = args
            out.append(("zoom", ch, cw, top, left, (f & 255, (f >> 8) & 255, (f >> 16) & 255)))
        elif kind == _C.YB_AUG_CROP:
            out.append(("crop",) + tuple(args))
        else:
            out.append(("hflip",))
    if st.float_out:
        out.append(("float",))
    return out
