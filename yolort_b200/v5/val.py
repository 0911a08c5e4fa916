"""YOLOv5's validation loop (val.py, v6.0) on the GPU: `run(model, data, labels)` returns the metrics YOLOv5 prints
after every epoch, measured on upstream's protocol: rect batches sorted by aspect ratio, each with its own minimum
canvas (LoadImagesAndLabels(augment=False, rect=True, pad=0.5)), INTER_AREA shrinks centred by letterbox, and every
prediction and label mapped back to the original image (scale_coords with ratio_pad) before matching.
"""
from typing import Optional

import torch

from .. import _C
from .utils import datasets as _ds
from .utils.general import rescale_params, scale_coords_padded
from .utils.metrics import DetectionMetrics

__all__ = ["run"]


def _yolo(model):
    from ..models.yolov5 import YOLOv5

    return model.model if isinstance(model, YOLOv5) else model


def _image_sizes(paths):
    """(h, w) of each file as stored, read from its header; a file no header reader takes is decoded."""
    from PIL import Image
    from torchvision.io import ImageReadMode, read_image

    sizes = []
    for p in paths:
        try:
            with Image.open(p) as im:
                w, h = im.size
        except Exception:
            _, h, w = read_image(p, mode=ImageReadMode.RGB).shape
        sizes.append((int(h), int(w)))
    return sizes


def _detect(yolo, imgs: torch.Tensor, conf_thres: float, iou_thres: float, max_det: int):
    """The model's detections on a uint8 [N, 3, H, W] RGB batch at val's thresholds, in canvas pixels: the plan for
    (N, H, W) fed through the identity path, its stored logits decoded and NMS'd with the model's own post-processing
    semantics, nothing dropped (_C.decode_nms_complete).  (boxes [N, D, 4], scores, labels, counts)."""
    N, _, H, W = (int(v) for v in imgs.shape)
    plan = yolo.engine().plan(N, H, W)             # stored logits: no fused decode epilogue
    yolo._write_samples(plan, imgs)
    heads = yolo.run_plan(plan)
    pc = yolo.post_config()
    return _C.decode_nms_complete(heads, "nhwc", pc["strides"], pc["anchors_px"], pc["num_classes"], float(conf_thres),
                                  float(iou_thres), int(max_det), pc["semantics"])[:4]


@torch.no_grad()
def run(model, data, labels, batch_size: int = 32, img_size: int = 640, conf_thres: float = 0.001,
        iou_thres: float = 0.6, max_det: int = 300, pad: float = 0.5, channel_order: Optional[str] = None) -> dict:
    """val.py's loop over a whole set; returns DetectionMetrics.compute()'s dict (mp, mr, map50, map, maps, ...,
    fitness).

    model: a YOLOv5 or a YOLO in eval mode on a CUDA device.
    data: CUDA uint8 [H, W, 3] images (cv2's layout, any strides), or file paths.  Files are decoded as stored by the
        ingest path of YOLOv5.predict (baseline JPEGs on the device, everything else and corrupt files on the CPU), to
        the RGB bytes of torchvision's read_image; no EXIF orientation is applied (cv2.imread would apply one other
        than 1).
    labels: per image float32 [n, 5] (cls, x, y, w, h normalised) arrays, or None.
    channel_order: "bgr" or "rgb" of the images; paths are always "rgb"; tensors default to "bgr".

    Per rect batch, in upstream's order: load_image(augment=False) and letterbox into the batch canvas (val_batch),
    the model's plan for (N, H, W), decode + NMS at conf_thres / iou_thres / max_det with the model's own
    post-processing (the reference's PostProcess semantics, not upstream's non_max_suppression; the model's own
    thresholds are not touched), scale_coords of predictions and targets to native pixels, DetectionMetrics.
    update_padded.  Batch canvases are multiples of the model's largest stride."""
    yolo = _yolo(model)
    if yolo.training:
        raise NotImplementedError("val.run: call .eval() first")
    data = list(data)
    labels = list(labels)
    if not data:
        raise ValueError("val.run: no images")
    if len(labels) != len(data):
        raise ValueError(f"val.run: {len(data)} images and {len(labels)} label arrays")
    dev = next(yolo.parameters()).device
    if dev.type != "cuda":
        raise _C.NativeLibraryError("val.run: the model must live on a CUDA device (no CPU fallback)")
    paths = all(isinstance(d, str) for d in data)
    if paths:
        if channel_order not in (None, "rgb"):
            raise ValueError("val.run: decoded files are RGB")
        channel_order = "rgb"
        sizes = _image_sizes(data)
        from ..models.yolov5 import YOLOv5

        ingest = model if isinstance(model, YOLOv5) else YOLOv5(model=yolo)
    else:
        channel_order = channel_order or "bgr"
        sizes = [(int(im.shape[0]), int(im.shape[1])) for im in data]
    stride = int(max(yolo.anchor_generator.strides))
    irect, bi, batch_shapes = _ds.rect_batches(sizes, img_size, batch_size, stride, pad)
    metrics = DetectionMetrics(yolo.num_classes, device=dev)
    with _C.device_guard(dev):
        for k in range(len(batch_shapes)):
            idx = [int(i) for i in irect[bi == k]]
            if paths:
                images = [t.permute(1, 2, 0) for t in ingest._ingest_files([data[i] for i in idx], dev)]
            else:
                images = [data[i] for i in idx]
            H, W = (int(v) for v in batch_shapes[k])
            imgs, targets, shapes = _ds.val_batch(images, [labels[i] for i in idx], range(len(idx)), (H, W),
                                                  img_size, channel_order)
            boxes, scores, cls, counts = _detect(yolo, imgs, conf_thres, iou_thres, max_det)
            native = scale_coords_padded(boxes, counts, rescale_params(shapes, dev), targets, (H, W))
            metrics.update_padded(boxes, scores, cls, counts, native)
    return metrics.compute()
