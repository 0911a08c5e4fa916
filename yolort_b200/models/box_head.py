"""Detection head and post-processing front-ends.

`YOLOHead` keeps the reference parameter layout (yolort/models/box_head.py:14-82: one 1x1 conv with
bias per level, 3*(nc+5) outputs, bias initialised as `:40-46`).  `PostProcess` has the reference
constructor (box_head.py:363-386) and runs anchor-decode + multi-label threshold + batched NMS +
top-k as ONE native call (`yb_decode_nms`, csrc/decode_nms.cu) instead of the per-image Python loop
at box_head.py:414-427.  `SetCriterion` has the reference constructor (box_head.py:103-149) and computes
the training loss and its gradient in csrc/yolo_loss.cu.
"""
import math
from typing import Dict, List, Optional, Sequence

import torch
from torch import nn, Tensor

from .. import _C
from .common import _PlanOnly

# NMS semantics selector (see include/yolort_b200.h).  torchvision.ops.batched_nms switches between the
# coordinate-offset trick and exact per-class NMS on numel (SURVEY.md appendix C.2).
NMS_TV_AUTO = 0
NMS_EXACT_PER_CLASS = 1
NMS_OFFSET_TRICK = 2


class YOLOHead(_PlanOnly):
    def __init__(self, in_channels: List[int], num_anchors: int, strides: List[int], num_classes: int):
        super().__init__()
        if not isinstance(in_channels, list):
            in_channels = [in_channels] * len(strides)
        self.num_anchors = num_anchors
        self.num_classes = num_classes
        self.num_outputs = num_classes + 5
        self.strides = strides
        blocks = nn.ModuleList(nn.Conv2d(ch, self.num_outputs * num_anchors, 1) for ch in in_channels)
        for conv, s in zip(blocks, strides):
            with torch.no_grad():
                b = conv.bias.view(num_anchors, -1)
                b[:, 4] += math.log(8 / (640 / float(s)) ** 2)  # ~8 objects per 640 image
                b[:, 5:] += math.log(0.6 / (num_classes - 0.999999))
        self.head = blocks

    def forward(self, x: List[Tensor]) -> List[Tensor]:
        """`head(features)` (box_head.py:68-82): per level [N, A, H, W, nc+5] raw logits -- the training-mode output
        of the detector as well -- executed as the head launch range of the owning YOLO's plan."""
        owner = self.__dict__.get("_yb_owner")
        if not owner:
            return super().forward(x)
        return owner[0].run_head(list(x))


class PostProcess(nn.Module):
    """Decode + threshold + batched NMS + top-k on the device.

    forward() accepts the reference argument list (head_outputs [N,A,H,W,K] per level, grids, shifts);
    grids/shifts are accepted for signature compatibility -- the kernel recomputes them from
    `strides`/`anchors_px` (they are pure functions of the level shape).
    """

    def __init__(self, strides: List[int], score_thresh: float, nms_thresh: float, detections_per_img: int,
                 anchors_px: Optional[Sequence[Sequence[float]]] = None, nms_semantics: int = NMS_TV_AUTO):
        super().__init__()
        self.strides = strides
        self.score_thresh = score_thresh
        self.nms_thresh = nms_thresh
        self.detections_per_img = detections_per_img
        self.anchors_px = anchors_px
        self.nms_semantics = nms_semantics

    def forward(self, head_outputs: List[Tensor], grids: Optional[List[Tensor]] = None,
                shifts: Optional[List[Tensor]] = None) -> List[Dict[str, Tensor]]:
        if self.anchors_px is None:
            if shifts is None:
                raise ValueError("PostProcess needs anchors_px (or reference-style shifts)")
            anchors_px = [s[0, :, 0, 0, :].reshape(-1).float().tolist() for s in shifts]
        else:
            anchors_px = self.anchors_px
        return _C.decode_nms(
            head_outputs, layout="nahwk", strides=self.strides, anchors_px=anchors_px,
            score_thresh=self.score_thresh, nms_thresh=self.nms_thresh,
            detections_per_img=self.detections_per_img, semantics=self.nms_semantics,
        )


_LOSS_DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_LOSS_KEYS = ("cls_logits", "bbox_regression", "objectness")


class _LossCall:
    """What one loss call hands to the native library: parameters, level descriptors and the target count."""

    def __init__(self, params, levels, n_targets: int, device: torch.device):
        self.params, self.levels, self.n_targets, self.device = params, levels, n_targets, device


class _YoloLoss(torch.autograd.Function):
    """Forward: yb_yolo_loss_forward.  Backward: yb_yolo_loss_backward from the forward's workspace, with the incoming
    gradients of the three losses read on the device."""

    @staticmethod
    def forward(ctx, call: _LossCall, targets: Tensor, *heads: Tensor):
        out, status, ws = _C.yolo_loss_forward(call.params, call.levels, targets, call.device)
        ctx.call, ctx.ws = call, ws
        ctx.save_for_backward(*heads)       # the backward kernels read the logits again
        ctx.mark_non_differentiable(status)
        return out, status

    @staticmethod
    def backward(ctx, grad_out: Tensor, grad_status: Optional[Tensor]):
        heads = ctx.saved_tensors
        call = ctx.call
        grad_losses = grad_out[:3].to(torch.float32).contiguous()
        grads = [torch.empty_like(h, memory_format=torch.contiguous_format) for h in heads]
        _C.yolo_loss_backward(call.params, call.levels, call.n_targets, grad_losses, ctx.ws, grads)
        return (None, None, *grads)


class SetCriterion(nn.Module):
    """YOLOv5's training loss (yolort/models/box_head.py:85-325) on the device: target assignment, CIoU box loss, class
    and objectness BCE, and the gradient with respect to the head outputs, in the kernels of csrc/yolo_loss.cu.

    The constructor and the attributes are the reference's.  `strides` may be a Tensor (normalised to ints);
    `fl_gamma` is accepted and ignored, as in the reference.  `forward(targets, head_outputs)` returns
    {"cls_logits", "bbox_regression", "objectness"} as shape-[1] fp32 tensors, differentiable with respect to the head
    outputs ([N, A, H, W, nc + 5] per level, fp32 / fp16 / bf16).  Host targets are validated before their copy to the
    device; device targets are validated by the kernels and read back once.  With `auto_balance` the per-level
    objectness means are read back to update `balance`, after the call's loss has used the previous values.
    """

    def __init__(self, strides: List[int], anchor_grids: List[List[float]], num_classes: int, fl_gamma: float = 0.0,
                 box_gain: float = 0.05, cls_gain: float = 0.5, cls_pos: float = 1.0, obj_gain: float = 1.0,
                 obj_pos: float = 1.0, anchor_thresh: float = 4.0, label_smoothing: float = 0.0,
                 auto_balance: bool = False) -> None:
        super().__init__()
        if isinstance(strides, Tensor):
            strides = strides.tolist()
        strides = [int(s) for s in strides]
        if len(strides) != len(anchor_grids):
            raise ValueError("strides and anchor_grids must have one entry per level")
        if not 1 <= len(strides) <= _C.YB_MAX_LEVELS:
            raise ValueError(f"SetCriterion supports 1 to {_C.YB_MAX_LEVELS} levels, got {len(strides)}")
        self.num_classes = num_classes
        self.strides = strides
        self.anchor_grids = anchor_grids
        self.num_anchors = len(anchor_grids[0]) // 2
        if not 1 <= self.num_anchors <= _C.YB_MAX_ANCHORS or any(len(a) != 2 * self.num_anchors for a in anchor_grids):
            raise ValueError("every level needs the same 1 to 4 (w, h) anchors")
        balance_defaults = [4.0, 1.0, 0.4, 0.1]
        self.balance = balance_defaults[: len(strides)]
        self.ssi = strides.index(16) if 16 in strides else 0
        self.sort_obj_iou = False
        self.cls_pos = cls_pos
        self.obj_pos = obj_pos
        self.smooth_pos = 1.0 - 0.5 * label_smoothing
        self.smooth_neg = 0.5 * label_smoothing
        self.gr = 1.0
        self.auto_balance = auto_balance
        self.box_gain = box_gain
        self.cls_gain = cls_gain
        self.obj_gain = obj_gain
        self.anchor_thresh = anchor_thresh

    def _check_heads(self, head_outputs: Sequence[Tensor]) -> None:
        if len(head_outputs) != len(self.strides):
            raise ValueError(f"expected {len(self.strides)} head outputs, got {len(head_outputs)}")
        h0 = head_outputs[0]
        for i, h in enumerate(head_outputs):
            if (h.dim() != 5 or h.shape[0] != h0.shape[0] or h.shape[1] != self.num_anchors
                    or h.shape[4] != self.num_classes + 5 or h.shape[2] < 1 or h.shape[3] < 1):
                raise ValueError(f"head output {i}: expected [N, {self.num_anchors}, H, W, {self.num_classes + 5}], got "
                                 f"{tuple(h.shape)}")
            if h.dtype not in _LOSS_DTYPES or h.dtype != h0.dtype or h.device != h0.device:
                raise ValueError("head outputs must share one device and one dtype of fp32 / fp16 / bf16")

    def _check_host_targets(self, targets: Tensor, n_images: int) -> None:
        t = targets.to(torch.float64)
        bad = ~torch.isfinite(t[:, 2:6]).all(1)
        if bool(bad.any()):
            raise ValueError(f"target row {int(bad.nonzero()[0])}: cx, cy, w, h must be finite")
        bad = ~((t[:, 0] >= 0) & (t[:, 0] < n_images))
        if bool(bad.any()):
            r = int(bad.nonzero()[0])
            raise ValueError(f"target row {r}: image index {float(t[r, 0])} is outside [0, {n_images})")
        bad = ~((t[:, 1] >= 0) & (t[:, 1] < self.num_classes))
        if bool(bad.any()):
            r = int(bad.nonzero()[0])
            raise ValueError(f"target row {r}: class {float(t[r, 1])} is outside [0, {self.num_classes})")

    def _params(self, n_images: int):
        p = _C.YoloLossParams()
        p.n_images, p.n_levels, p.n_anchors, p.n_classes = n_images, len(self.strides), self.num_anchors, self.num_classes
        p.box_gain, p.cls_gain, p.obj_gain = self.box_gain, self.cls_gain, self.obj_gain
        p.cls_pos, p.obj_pos, p.anchor_thresh = self.cls_pos, self.obj_pos, self.anchor_thresh
        p.smooth_pos, p.smooth_neg, p.gr = self.smooth_pos, self.smooth_neg, self.gr
        for i, b in enumerate(self.balance):
            p.balance[i] = float(b)
        return p

    def forward(self, targets: Tensor, head_outputs: List[Tensor]) -> Dict[str, Tensor]:
        if self.sort_obj_iou:
            raise NotImplementedError("sort_obj_iou=True is not supported by the device loss")
        self._check_heads(head_outputs)
        if not isinstance(targets, Tensor) or targets.dim() != 2 or targets.shape[1] != 6 \
                or not targets.is_floating_point():
            raise ValueError("targets must be a floating-point [T, 6] tensor of (image, class, cx, cy, w, h)")
        n_images = int(head_outputs[0].shape[0])
        on_host = not targets.is_cuda
        if on_host:
            self._check_host_targets(targets, n_images)
        heads = [h.contiguous() for h in head_outputs]
        _C.require_cuda(heads[0], "SetCriterion")
        dev = heads[0].device
        tdev = targets.to(device=dev, dtype=torch.float32).contiguous()
        params = self._params(n_images)
        levels = _C.yolo_loss_levels(heads, self.strides, self.anchor_grids)
        call = _LossCall(params, levels, int(tdev.shape[0]), dev)
        if torch.is_grad_enabled() and any(h.requires_grad for h in heads):
            out, status = _YoloLoss.apply(call, tdev, *heads)
        else:
            out, status, _ = _C.yolo_loss_forward(params, levels, tdev, dev)
        if not on_host:
            bits = int(status.item())       # the call's one synchronisation
            if bits:
                why = [w for b, w in ((_C.YB_LOSS_ST_IMAGE, "an image index outside [0, N)"),
                                      (_C.YB_LOSS_ST_CLASS, "a class outside [0, num_classes)"),
                                      (_C.YB_LOSS_ST_NONFINITE, "a non-finite cx, cy, w or h")) if bits & b]
                raise ValueError("targets hold " + " and ".join(why))
        if self.auto_balance:
            objs = out[3:].detach().tolist()
            self.balance = [b * 0.9999 + 0.0001 / o for b, o in zip(self.balance, objs)]
            self.balance = [x / self.balance[self.ssi] for x in self.balance]
        return {key: out[i: i + 1] for i, key in enumerate(_LOSS_KEYS)}
