"""`YOLOTransform`: the letterbox front-end, backed by the native kernel.

Same constructor and call contract as the reference class (yolort/models/transform.py:100-351):
`forward(images, targets=None)` returns a `NestedTensor` (padded batch + resized sizes) and the target batch.  The
resize/pad arithmetic is `yb_letterbox_geometry` (host, csrc/letterbox.cu) + `yb_letterbox` (device).  Extension:
images may be uint8 [3,H,W] tensors, in which case the `/255` of the default loader (yolov5.py:228) is fused.
"""
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
from torch import nn, Tensor

from .. import _C


class NestedTensor(NamedTuple):
    tensors: Tensor
    image_sizes: List[Tuple[int, int]]


class YOLOTransform(nn.Module):
    def __init__(self, min_size: int, max_size: int, *, size_divisible: int = 32,
                 fixed_shape: Optional[Tuple[int, int]] = None, fill_color: int = 114) -> None:
        super().__init__()
        self.min_size = min_size
        self.max_size = max_size
        self.size_divisible = size_divisible
        self.fixed_shape = fixed_shape
        self.fill_color = fill_color / 255

    # -- geometry --------------------------------------------------------------------------------
    def geometry(self, images: List[Tensor], batch_hw: Optional[Tuple[int, int]] = None):
        for im in images:
            if im.dim() != 3:
                raise ValueError(
                    f"images is expected to be a list of 3d tensors of shape [C, H, W], but got '{im.shape}'.")
        sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in images]
        fixed = batch_hw if batch_hw is not None else self.fixed_shape
        return _C.letterbox_geometry(sizes, float(self.min_size), float(self.max_size), self.size_divisible, fixed)

    def letterbox_into(self, images: List[Tensor], geoms, Hb: int, Wb: int, out: Tensor, layout: int) -> Tensor:
        return _C.letterbox(images, geoms, Hb, Wb, self.fill_color, out, layout)

    # -- reference call contract -------------------------------------------------------------------
    def forward(self, images: List[Tensor], targets: Optional[List[Dict[str, Tensor]]] = None):
        images = list(images)
        geoms, (Hb, Wb) = self.geometry(images)
        dt = images[0].dtype if images[0].is_floating_point() else torch.float32
        out = torch.empty((len(images), 3, Hb, Wb), dtype=dt, device=images[0].device)
        self.letterbox_into(images, geoms, Hb, Wb, out, _C.YB_LAYOUT_NCHW)
        sizes = [(int(g.new_h), int(g.new_w)) for g in geoms]
        if targets is None:
            return NestedTensor(out, sizes), None
        return NestedTensor(out, sizes), self.batch_targets(images, targets)

    def batch_targets(self, images: List[Tensor], targets: List[Dict[str, Tensor]]) -> Tensor:
        """The reference's target batch (transform.py:205-219 with normalize_boxes :370-381): each image's xyxy boxes
        divided by its PRE-resize (h, w) in fp32 (IEEE division, as the reference's tensor-by-tensor division), then
        cx = (x0 + x1) / 2, cy = (y0 + y1) / 2, w = x1 - x0, h = y1 - y0; rows (image, label, cx, cy, w, h) on the
        images' device, [0, 6] when there are no boxes.  As in the reference the boxes ignore the letterbox's
        padding offset.  No host synchronisation: the per-row image index and divisors cross in one copy."""
        if len(targets) != len(images):
            raise ValueError(f"{len(images)} images and {len(targets)} targets")
        dev = images[0].device
        counts = [int(t["labels"].shape[0]) for t in targets]
        if sum(counts) == 0:
            return torch.zeros((0, 6), dtype=torch.float32, device=dev)
        host = torch.empty((sum(counts), 5), dtype=torch.float32)
        row = 0
        for i, (im, c) in enumerate(zip(images, counts)):
            h, w = float(im.shape[-2]), float(im.shape[-1])
            host[row:row + c] = torch.tensor([i, w, h, w, h], dtype=torch.float32)
            row += c
        host = host.pin_memory().to(dev, non_blocking=True) if dev.type == "cuda" else host.to(dev)
        boxes = torch.cat([t["boxes"].to(dev, torch.float32) for t, c in zip(targets, counts) if c])
        labels = torch.cat([t["labels"].to(dev) for t, c in zip(targets, counts) if c]).to(torch.float32)
        b = boxes / host[:, 1:]
        x0, y0, x1, y1 = b.unbind(1)
        return torch.stack([host[:, 0], labels, (x0 + x1) / 2, (y0 + y1) / 2, x1 - x0, y1 - y0], 1)

    def batch_images(self, images: List[Tensor]) -> Tensor:
        """Pad already-resized images into one batch (transform.py:297-330): run the kernel with an
        identity resize per image."""
        sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in images]
        mh, mw = max(s[0] for s in sizes), max(s[1] for s in sizes)
        if self.fixed_shape is not None:
            Hb, Wb = self.fixed_shape
        else:
            d = self.size_divisible
            Hb, Wb = -(-mh // d) * d, -(-mw // d) * d
        geoms = (_C.LetterboxGeom * len(images))()
        for g, (h, w) in zip(geoms, sizes):
            g.src_h, g.src_w, g.new_h, g.new_w = h, w, h, w
            g.top, g.left = int(round((Hb - h) / 2 - 0.1)), int(round((Wb - w) / 2 - 0.1))
            g.ratio_h = g.ratio_w = 1.0
        dt = images[0].dtype if images[0].is_floating_point() else torch.float32
        out = torch.empty((len(images), 3, Hb, Wb), dtype=dt, device=images[0].device)
        return self.letterbox_into(list(images), geoms, Hb, Wb, out, _C.YB_LAYOUT_NCHW)

    def rescale_params(self, batch_hw: Tuple[int, int], original_image_sizes: List[Tuple[int, int]]) -> Tensor:
        """[n,3] fp32 (gain, pad_x, pad_y) of scale_coords (transform.py:354-367), host tensor."""
        rows = [_C.scale_coords_params(batch_hw[0], batch_hw[1], h, w) for h, w in original_image_sizes]
        return torch.tensor(rows, dtype=torch.float32)

    def rescale_params_device(self, batch_hw: Tuple[int, int], original_image_sizes: List[Tuple[int, int]], device) -> Tensor:
        """The same table on `device`, cached per (canvas, image sizes): a serving loop sees the same few size patterns,
        and the per-image host arithmetic plus a small pageable H2D copy cost ~0.1 ms of an otherwise idle GPU per call."""
        cache = self.__dict__.setdefault("_rescale_cache", {})
        key = (str(device), int(batch_hw[0]), int(batch_hw[1]), tuple(original_image_sizes))
        t = cache.get(key)
        if t is None:
            if len(cache) >= 256:
                cache.clear()
            t = self.rescale_params(batch_hw, original_image_sizes).to(device)
            cache[key] = t
        return t

    def postprocess(self, result: List[Dict[str, Tensor]], image_shapes, original_image_sizes: List[Tuple[int, int]]):
        """Stand-alone box rescale for callers that run their own detector between `forward` and
        `postprocess` (the fused path applies it inside the NMS kernel).  Elementwise affine only."""
        Hb, Wb = int(image_shapes[0]), int(image_shapes[1])
        for pred, (h, w) in zip(result, original_image_sizes):
            gain, px, py = _C.scale_coords_params(Hb, Wb, int(h), int(w))
            b = pred["boxes"]
            pad = torch.tensor([px, py, px, py], dtype=b.dtype, device=b.device)
            pred["boxes"] = (b - pad) / torch.tensor(gain, dtype=b.dtype, device=b.device)
        return result

    def __repr__(self):
        return f"{self.__class__.__name__}(\n    Resize(min_size={self.min_size}, max_size={self.max_size})\n)"
