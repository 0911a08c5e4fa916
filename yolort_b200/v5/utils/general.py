"""val.py's box helpers (yolort/v5/utils/general.py:404-515) on CUDA float32 tensors: `xywh2xyxy`, `scale_coords`,
`clip_coords` with torch's own arithmetic (python scalars are rounded to float32), in the reference's order: `-= pad`,
`/= gain`, clamp.  On CUDA tensors torch divides by a python scalar as a product with its float reciprocal, which can
differ from the correctly rounded quotient in the last place.

`scale_coords_padded` is the same rescale for a whole batch in one launch (csrc/v5_augment.cu, v5_rescale_kernel), in
torch's CPU float32 arithmetic (a correctly rounded division by gain, as the reference computes it on CPU tensors):
padded detections [n, D, 4] with their counts, and optionally the batch's targets, which it also takes through val.py's
`targets[:, 2:] *= [W, H, W, H]` and `xywh2xyxy`.  oracle/restate_v5val.py restates both.
"""
from typing import Optional, Sequence

import torch
from torch import Tensor

from ... import _C

__all__ = ["xywh2xyxy", "scale_coords", "clip_coords", "scale_coords_padded", "rescale_params"]


def xywh2xyxy(x: Tensor) -> Tensor:
    """nx4 boxes from [x, y, w, h] to [x1, y1, x2, y2] (xy1 top left, xy2 bottom right)."""
    y = x.clone()
    y[:, 0] = x[:, 0] - x[:, 2] / 2  # top left x
    y[:, 1] = x[:, 1] - x[:, 3] / 2  # top left y
    y[:, 2] = x[:, 0] + x[:, 2] / 2  # bottom right x
    y[:, 3] = x[:, 1] + x[:, 3] / 2  # bottom right y
    return y


def clip_coords(boxes: Tensor, shape) -> None:
    """Clips xyxy boxes to the image shape (height, width), in place."""
    boxes[:, 0].clamp_(0, shape[1])  # x1
    boxes[:, 1].clamp_(0, shape[0])  # y1
    boxes[:, 2].clamp_(0, shape[1])  # x2
    boxes[:, 3].clamp_(0, shape[0])  # y2


def scale_coords(img1_shape, coords: Tensor, img0_shape, ratio_pad=None) -> Tensor:
    """Rescales xyxy coords from img1_shape to img0_shape in place and returns them; ratio_pad ((gain, _), (padw,
    padh)) as letterbox returned them, else letterbox's centred geometry."""
    if ratio_pad is None:  # calculate from img0_shape
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])  # gain  = old / new
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2  # wh padding
    else:
        gain = ratio_pad[0][0]
        pad = ratio_pad[1]
    coords[:, [0, 2]] -= float(pad[0])  # x padding
    coords[:, [1, 3]] -= float(pad[1])  # y padding
    coords[:, :4] /= float(gain)
    clip_coords(coords, img0_shape)
    return coords


def rescale_params(shapes: Sequence, device) -> Tensor:
    """float32 [n, 5] (gain, padw, padh, h0, w0) per image from val_batch's shapes ((h0, w0), ((gain, _), (padw,
    padh)))."""
    rows = [[float(r[0]), float(p[0]), float(p[1]), float(s[0]), float(s[1])] for s, (r, p) in shapes]
    return torch.tensor(rows, dtype=torch.float32).reshape(-1, 5).pin_memory().to(device, non_blocking=True)


def scale_coords_padded(boxes: Tensor, counts: Tensor, params: Tensor, targets: Optional[Tensor] = None,
                        canvas_hw=None) -> Optional[Tensor]:
    """scale_coords(..., ratio_pad) and clip_coords of padded detections boxes [n, D, 4] float32 (slots d <
    counts[i]), in place, with params [n, 5] (gain, padw, padh, h0, w0) per image (rescale_params).  With `targets`
    [T, 6] (image, cls, x, y, w, h) normalised to the canvas canvas_hw (H, W), returns new targets (image, cls, x1, y1,
    x2, y2) in native pixels, as val.py makes them.  One launch; nothing synchronises."""
    dev = params.device
    _C.require_cuda(params, "scale_coords_padded")
    if params.dtype != torch.float32 or params.dim() != 2 or params.shape[1] != 5:
        raise ValueError(f"params: expected float32 [n, 5], got {params.dtype} {tuple(params.shape)}")
    n = int(params.shape[0])
    if boxes.dtype != torch.float32 or tuple(boxes.shape[::2]) != (n, 4) or boxes.dim() != 3 or boxes.device != dev:
        raise ValueError(f"boxes: expected float32 [{n}, D, 4] on {dev}, got {boxes.dtype} {tuple(boxes.shape)}")
    if not boxes.is_contiguous():
        raise ValueError("boxes: must be contiguous (rescaled in place)")
    counts = counts.to(device=dev, dtype=torch.int32).contiguous().reshape(-1)
    if counts.numel() != n:
        raise ValueError(f"counts: expected {n} values, got {counts.numel()}")
    params = params.contiguous()
    out = None
    if targets is not None:
        if targets.dim() != 2 or targets.shape[1] != 6:
            raise ValueError(f"targets: expected [T, 6], got {tuple(targets.shape)}")
        if canvas_hw is None:
            raise ValueError("targets need canvas_hw (H, W)")
        targets = targets.to(device=dev, dtype=torch.float32).contiguous()
        out = torch.empty_like(targets)
    _C.v5_rescale_coords(boxes, counts, targets if targets is not None and targets.shape[0] else None, out, params,
                         canvas_hw or (0, 0))
    return out
