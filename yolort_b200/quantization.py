"""FP8 (e4m3) post-training calibration of the YOLOv5 detection models.

The reference deploys 8-bit inference through TensorRT (deployment/ppq/: per-channel weights, per-tensor activations,
calibrated on images).  On an H100 the 8-bit tensor-core type is FP8; this module provides the same recipe for the
native plan:

    calib = calibrate_fp8(model, batches)     # model: YOLOv5 or YOLO, batches: what model.forward takes
    model.set_fp8(calib)                      # every later forward / predict runs the FP8 plan
    torch.save(calib.state_dict(), path)      # next to the weights; model.state_dict() does not change

Calibration runs the existing fp16 / bf16 plan with every activation kept and records max|x| per arena buffer.  Scales
are powers of two (engine.e4m3_scale), weights are scaled per output channel, activations per tensor (DESIGN.md, "FP8
inference").
"""
import hashlib
import math
from typing import Dict, Iterable

import torch
from torch import nn

from . import _C

__all__ = ["Fp8Calibration", "calibrate_fp8"]


def arch_fingerprint(model: nn.Module) -> str:
    """Digest of the state-dict layout (names and shapes): a calibration only applies to the architecture it was made
    for."""
    h = hashlib.sha1()
    for k, v in model.state_dict().items():
        h.update(f"{k}:{tuple(v.shape)};".encode())
    return h.hexdigest()


class Fp8Calibration:
    """Calibrated activation ranges of one model: max|x| per buffer of the fp16 / bf16 plan (`amax`), and the
    architecture fingerprint they belong to."""

    def __init__(self, amax: Dict[str, float], fingerprint: str):
        self.amax = {str(k): float(v) for k, v in amax.items()}
        self.fingerprint = str(fingerprint)

    def state_dict(self) -> dict:
        return {"amax": dict(self.amax), "fingerprint": self.fingerprint}

    def load_state_dict(self, state_dict: dict) -> None:
        self.amax = {str(k): float(v) for k, v in state_dict["amax"].items()}
        self.fingerprint = str(state_dict["fingerprint"])

    def __repr__(self) -> str:
        return f"Fp8Calibration({len(self.amax)} buffers, fingerprint {self.fingerprint[:12]})"


def _yolo_of(model: nn.Module):
    from .engine import fp8_unsupported
    from .models.yolo import YOLO
    from .models.yolov5 import YOLOv5

    yolo = model.model if isinstance(model, YOLOv5) else model
    why = fp8_unsupported(yolo)
    if why is not None:
        raise NotImplementedError(f"FP8 inference is not implemented for {why}")
    if not isinstance(yolo, YOLO):
        raise TypeError(f"calibrate_fp8 takes a YOLOv5 or a YOLO, got {type(model).__name__}")
    return yolo


@torch.no_grad()
def calibrate_fp8(model: nn.Module, batches: Iterable) -> Fp8Calibration:
    """Runs `batches` through the fp16 / bf16 plan of `model` (a YOLOv5 or a YOLO; each batch is what that model's
    forward takes) with every activation kept and chains off, and returns the max|x| of every buffer over all
    batches.  Raises NotImplementedError for model families without an FP8 plan."""
    from .engine import PlanInstance
    from .models.yolov5 import YOLOv5

    yolo = _yolo_of(model)
    if yolo.training:
        raise NotImplementedError("calibrate_fp8 runs the inference plan; call .eval()")
    low = yolo.engine().lowered(fp8=False)
    amax: Dict[str, float] = {}
    n = 0
    for batch in batches:
        if isinstance(model, YOLOv5):
            images = model.collate_images(batch, model.default_loader)
            geoms, (Hb, Wb) = model.transform.geometry(images, None)
            plan = PlanInstance(low, len(images), Hb, Wb, keep_intermediates=True, fuse_chains=False)
            model.transform.letterbox_into(images, geoms, Hb, Wb, plan.input, _C.YB_LAYOUT_S2D16)
        else:
            if batch.dim() != 4 or batch.shape[1] != 3:
                raise ValueError(f"a YOLO batch must be [N,3,H,W], got {tuple(batch.shape)}")
            N, _, H, W = (int(v) for v in batch.shape)
            plan = PlanInstance(low, N, H, W, keep_intermediates=True, fuse_chains=False)
            yolo._write_samples(plan, batch)
        plan.run()
        names = list(plan.buffers)
        vals = torch.stack([plan.buffers[k].abs().amax().float() for k in names]).tolist()
        for k, v in zip(names, vals):
            if not math.isfinite(v):
                raise ValueError(f"calibrate_fp8: buffer {k} holds non-finite values")
            amax[k] = max(amax.get(k, 0.0), v)
        n += 1
    if n == 0:
        raise ValueError("calibrate_fp8 needs at least one batch")
    return Fp8Calibration(amax, arch_fingerprint(yolo))
