"""`YOLOv5`: letterbox -> backbone/PAN/head -> decode+NMS -> rescale, end to end on the GPU.

Keeps the public surface of the reference wrapper (yolort/models/yolov5.py:19-297): constructor kwargs,
`forward(List[Tensor[3,H,W]]) -> List[Dict]` with keys (scores, labels, boxes), `predict`,
`collate_images`, `default_loader`, `load_from_yolov5`.  Differences, all additive: uint8 images are
accepted (the /255 is fused into the letterbox kernel), and `forward_padded` exposes the fixed-shape
device outputs for callers that gather across ranks.
"""
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
from torch import nn, Tensor

from .. import _C
from . import yolo
from .transform import YOLOTransform
from .yolo import YOLO

__all__ = ["YOLOv5"]


class YOLOv5(nn.Module):
    def __init__(
        self,
        arch: Optional[str] = None,
        model: Optional[nn.Module] = None,
        num_classes: int = 80,
        pretrained: bool = False,
        progress: bool = True,
        size: Tuple[int, int] = (640, 640),
        size_divisible: int = 32,
        fixed_shape: Optional[Tuple[int, int]] = None,
        fill_color: int = 114,
        **kwargs: Any,
    ) -> None:
        super().__init__()
        self.arch = arch
        self.num_classes = num_classes
        if model is None:
            if arch is None or not hasattr(yolo, arch):
                raise ValueError(f"unknown architecture {arch!r}; available: {yolo.__all__[1:]}")
            model = getattr(yolo, arch)(pretrained=pretrained, progress=progress, num_classes=num_classes, **kwargs)
        self.model = model
        self.transform = YOLOTransform(size[0], size[1], size_divisible=size_divisible, fixed_shape=fixed_shape,
                                       fill_color=fill_color)

    # ---------------------------------------------------------------------------------------------
    @property
    def precision(self) -> str:
        """"fp8", "fp16" or "bf16": what the plans compute in (YOLO.precision)."""
        return self.model.precision

    def set_fp8(self, calib) -> None:
        """FP8 inference with the scales of `calib` (quantization.calibrate_fp8), or None for fp16 / bf16 again
        (YOLO.set_fp8)."""
        self.model.set_fp8(calib)

    def _prepare(self, inputs: List[Tensor], batch_hw: Optional[Tuple[int, int]] = None):
        """Letterbox `inputs` straight into the plan's input canvas; returns (plan, rescale[n,3] on device)."""
        if self.training:
            raise NotImplementedError("the training path is out of scope of this build; call .eval()")
        inputs = list(inputs)
        if len(inputs) == 0:
            raise ValueError("empty image list")
        original_image_sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in inputs]
        geoms, (Hb, Wb) = self.transform.geometry(inputs, batch_hw)
        plan = self.model.get_plan(len(inputs), Hb, Wb)
        self.transform.letterbox_into(inputs, geoms, Hb, Wb, plan.input, _C.YB_LAYOUT_S2D16)
        rescale = self.transform.rescale_params_device((Hb, Wb), original_image_sizes, plan.device)
        return plan, rescale

    def forward(self, inputs: List[Tensor], targets: Optional[List[Dict[str, Tensor]]] = None, augment: bool = False):
        """`augment=True`: YOLOv5's test-time augmentation (upstream `--augment`, yolort/v5/models/yolo.py:152-208): the
        letterboxed canvas, its 0.83x mirrored and its 0.67x copies through the network, their predictions descaled and
        merged into one NMS per image (YOLO.detect_augmented).  About twice the inference time."""
        if augment:
            return self._forward_augment(inputs, targets)
        if self.training or self.model.has_hooks():
            # The reference's own staging (yolov5.py:155-189): transform -> model (backbone -> head -> post-process
            # through the callable sub-modules, so forward hooks fire) -> rescale.  Training mode letterboxes the
            # images, batches the normalised targets (transform.py:205-250) and returns what the model's criterion
            # returns (YOLO(..., criterion=SetCriterion(...)); without one YOLO.forward raises).
            inputs = list(inputs)
            original_image_sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in inputs]
            samples, targets_batched = self.transform(inputs, targets if self.training else None)
            outputs = self.model(samples.tensors, targets_batched)
            if self.training:
                return outputs
            hb, wb = int(samples.tensors.shape[-2]), int(samples.tensors.shape[-1])
            return self.transform.postprocess(outputs, (hb, wb), original_image_sizes)
        if targets is not None:
            raise NotImplementedError("targets are only used by the training path")
        plan, rescale = self._prepare(inputs)
        return self.model.detect(plan, rescale)

    def _forward_augment(self, inputs: List[Tensor], targets=None) -> List[Dict[str, Tensor]]:
        if self.training:
            raise NotImplementedError("test-time augmentation is not implemented for training mode (an inference path; "
                                      "call .eval())")
        if targets is not None:
            raise NotImplementedError("targets are only used by the training path")
        inputs = list(inputs)
        if len(inputs) == 0:
            raise ValueError("empty image list")
        original_image_sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in inputs]
        geoms, (Hb, Wb) = self.transform.geometry(inputs)

        def write(canvas: Tensor) -> None:
            self.transform.letterbox_into(inputs, geoms, Hb, Wb, canvas, _C.YB_LAYOUT_S2D16)

        dev = next(self.parameters()).device
        with _C.device_guard(dev):
            rescale = self.transform.rescale_params_device((Hb, Wb), original_image_sizes, dev)
            return self.model.detect_augmented(len(inputs), Hb, Wb, write, rescale)

    def forward_padded(self, inputs: List[Tensor], batch_hw: Optional[Tuple[int, int]] = None):
        """Same computation, fixed-shape device outputs and no host synchronisation:
        (boxes [n,D,4], scores [n,D], labels [n,D] int64, counts [n] int32, status [4] int64).
        `batch_hw` pins the canvas (multi-GPU shards must letterbox to the GLOBAL batch shape to
        reproduce single-GPU boxes: SURVEY.md section 8e)."""
        plan, rescale = self._prepare(inputs, batch_hw)
        return self.model.detect_padded(plan, rescale)

    @torch.no_grad()
    def predict(self, x: Any, image_loader: Optional[Callable] = None, augment: bool = False) -> List[Dict[str, Tensor]]:
        image_loader = image_loader or self.default_loader
        if not augment:
            piped = self._predict_pipelined(x)
            if piped is not None:
                return piped
        images = self.collate_images(x, image_loader)
        return self.forward(images, augment=augment)

    # -- throughput API ---------------------------------------------------------------------------------------
    @torch.no_grad()
    def predict_stream(self, batches, depth: int = 2):
        """Serving loop over an iterable of HOST batches (each what `predict` accepts: a list of [3,H,W] tensors,
        ideally slices of one pinned buffer, or a list of paths).  Yields, in order, the reference's
        `List[Dict{scores, labels, boxes}]` per batch with the tensors on the HOST.

        Same kernels and same results as `predict`; what changes is the schedule: the PCIe copy of batch i+1 runs on
        a copy stream while batch i computes, and the results of batch i-1 come back as one asynchronous D2H of the
        padded `[n, D, 6]` block instead of a synchronous read per call, so the host never idles the GPU.  `depth`
        batches are in flight; a caller-owned host batch must stay unmodified until its results have been yielded.
        """
        import collections

        p = next(self.parameters())
        dev = p.device
        if dev.type != "cuda":
            raise _C.NativeLibraryError("predict_stream: the model must live on a CUDA device (no CPU fallback)")
        if self.training:
            raise NotImplementedError("the training path is out of scope of this build; call .eval()")
        compute = torch.cuda.current_stream(dev)
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream(dev)
        copy = self._copy_stream
        ring = self.__dict__.setdefault("_stream_ring", {})
        pending = collections.deque()
        seq = 0

        def finish(item):
            done, host_packed, host_meta, n, batch = item
            done.synchronize()
            meta = host_meta.tolist()
            if meta[n + 1] != 0:       # candidate arena overflow: the synchronous path grows it
                return [{k: v.cpu() for k, v in d.items()} for d in self.predict(batch)]
            out = []
            for i in range(n):
                c = meta[i]
                row = host_packed[i, :c]
                out.append({"scores": row[:, 4].clone(), "labels": row[:, 5].to(torch.int64), "boxes": row[:, :4].clone()})
            return out

        for batch in batches:
            batch = [batch] if isinstance(batch, (str, Tensor)) else list(batch)
            with torch.cuda.stream(copy):
                dev_imgs = self.collate_images(batch, self.default_loader)
                ev = torch.cuda.Event()
                ev.record(copy)
            compute.wait_event(ev)
            for t in dev_imgs:
                t.record_stream(compute)
            boxes, scores, labels, counts, status = self.forward_padded(dev_imgs)
            n, D = int(boxes.shape[0]), int(boxes.shape[1])
            packed = torch.cat([boxes, scores.unsqueeze(-1), labels.to(torch.float32).unsqueeze(-1)], dim=-1)
            meta = torch.cat([counts.to(torch.int64), status])
            key = (seq % (depth + 1), n, D)
            bufs = ring.get(key)
            if bufs is None:
                bufs = (torch.empty((n, D, 6), dtype=torch.float32, pin_memory=True),
                        torch.empty((n + 4,), dtype=torch.int64, pin_memory=True))
                ring[key] = bufs
            bufs[0].copy_(packed, non_blocking=True)
            bufs[1].copy_(meta, non_blocking=True)
            done = torch.cuda.Event()
            done.record(compute)
            pending.append((done, bufs[0], bufs[1], n, batch))
            seq += 1
            if len(pending) >= depth:
                yield finish(pending.popleft())
        while pending:
            yield finish(pending.popleft())

    # -- predict() on host tensors: the H2D copy hidden behind the front of the network ---------------------------------
    # A synchronous predict(list of host images) used to be  H2D (0.8 ms for 32 x 640^2 uint8)  ->  compute  ->  read
    # back, the PCIe copy fully exposed.  Now the batch crosses PCIe in four chunks on a copy stream; as soon as a chunk
    # has landed the compute stream letterboxes it and runs the front of the plan on those images only (stem ..
    # first tapped C3: the stride-2/4/8 levels, thousands of tiles even for 8 images), so the front of chunk k overlaps
    # the copy of chunk k+1; the rest of the plan, the decode and the NMS run once over the whole batch.  Same kernels
    # on the same per-image data: the detections are bit-identical to the device-resident call.
    _PIPELINE_MIN_IMAGES = 16

    def _predict_pipelined(self, x: Any) -> Optional[List[Dict[str, Tensor]]]:
        if self.training or self.model.has_hooks():
            return None
        if not (isinstance(x, (list, tuple)) and len(x) >= self._PIPELINE_MIN_IMAGES and len(x) % 4 == 0
                and all(isinstance(t, Tensor) and not t.is_cuda and t.dim() == 3 and t.dtype == x[0].dtype for t in x)):
            return None
        p = next(self.parameters())
        if p.device.type != "cuda":
            return None
        from ..relay.logits_decoder import LogitsDecoder

        if isinstance(self.model.post_process, LogitsDecoder):
            return None
        n = len(x)
        sizes = [(int(t.shape[-2]), int(t.shape[-1])) for t in x]
        tr = self.transform
        geoms, (Hb, Wb) = _C.letterbox_geometry(sizes, float(tr.min_size), float(tr.max_size), tr.size_divisible, tr.fixed_shape)
        plan = self.model.get_plan(n, Hb, Wb, chunked=True)
        if not plan.front_chunks or plan.fused_post is not None:
            return None
        dev = p.device
        with _C.device_guard(dev):
            compute = torch.cuda.current_stream(dev)
            if not hasattr(self, "_copy_stream"):
                self._copy_stream = torch.cuda.Stream(dev)
            copy = self._copy_stream
            copy.wait_stream(compute)          # the previous call's reads of recycled staging memory are done
            c = n // plan.front_chunks
            staged = []
            for k in range(plan.front_chunks):
                with torch.cuda.stream(copy):
                    part = self.collate_images(list(x[k * c:(k + 1) * c]), None)
                    ev = torch.cuda.Event()
                    ev.record(copy)
                staged.append((part, ev))
            GeomArr = _C.LetterboxGeom * c
            for k, (part, ev) in enumerate(staged):
                compute.wait_event(ev)
                for t in part:
                    t.record_stream(compute)
                gk = GeomArr(*[geoms[k * c + j] for j in range(c)])
                self.transform.letterbox_into(part, gk, Hb, Wb, plan.input[k * c:(k + 1) * c], _C.YB_LAYOUT_S2D16)
                plan.run_front_chunk(k)
            plan.run_rest()
            rescale = self.transform.rescale_params_device((Hb, Wb), sizes, dev)
            boxes, scores, labels, counts, status = self.model.post_padded(plan, rescale)
            host = torch.cat([counts.to(torch.int64), status]).tolist()
        if host[n + 1] != 0:
            return None       # candidate arena overflow: the plain path grows it
        return [{"scores": scores[i, :host[i]], "labels": labels[i, :host[i]], "boxes": boxes[i, :host[i]]} for i in range(n)]

    def default_loader(self, img_path: str) -> Tensor:
        """uint8 RGB [3,H,W]; the `/ 255.0` of the reference loader (yolov5.py:228) happens in the kernel."""
        from torchvision.io import ImageReadMode, read_image

        return read_image(img_path, mode=ImageReadMode.RGB)

    def collate_images(self, samples: Any, image_loader: Callable) -> List[Tensor]:
        p = next(self.parameters())

        def place(t: Tensor) -> Tensor:
            if t.dtype == torch.uint8:
                return t.to(p.device, non_blocking=True)
            return t.to(p.device).type_as(p)

        if isinstance(samples, Tensor):
            return [place(samples)]
        if isinstance(samples, (list, tuple)) and len(samples) > 0 and all(isinstance(s, Tensor) for s in samples):
            packed = self._place_packed(samples, p)
            return packed if packed is not None else [place(s) for s in samples]
        if isinstance(samples, str):
            samples = [samples]
        if isinstance(samples, (list, tuple)) and all(isinstance(s, str) for s in samples):
            if image_loader == self.default_loader and p.device.type == "cuda":
                return self._ingest_files(samples, p.device)
            return [place(image_loader(s)) for s in samples]
        raise NotImplementedError(
            f"The type of the sample is {type(samples)}, we currently don't support it now, the "
            "samples should be either a tensor, list of tensors, a image path or list of image paths.")

    # -- file ingest (SURVEY.md section 8f row 1) -------------------------------------------------------------
    _DECODE_THREADS = 8

    def _ingest_files(self, paths: List[str], device: torch.device) -> List[Tensor]:
        """`predict(paths)` fast path.  The files are read (and their headers parsed) on a small thread pool.  JPEGs
        the device decoder takes (yolort_b200.io) cross PCIe compressed, in one copy, and decode on the GPU to the
        bytes torchvision's CPU decoder gives; every other file is decoded on the CPU as before.  An image whose
        device decode reports corrupt data is decoded again on the CPU, so it warns, fills or raises exactly as
        before.  YB_JPEG_DECODE=cpu decodes everything on the CPU (A/B runs)."""
        import os

        on_gpu = os.environ.get("YB_JPEG_DECODE", "").lower() != "cpu"

        def load(path):
            if on_gpu:
                with open(path, "rb") as f:
                    data = f.read()
                info = _C.jpeg_parse(data)
                if info.supported:
                    return data, info
            return self.default_loader(path)

        if len(paths) > 1:
            from concurrent.futures import ThreadPoolExecutor

            with ThreadPoolExecutor(max_workers=min(self._DECODE_THREADS, len(paths))) as pool:
                loaded = list(pool.map(load, paths))
        else:
            loaded = [load(paths[0])]
        out: List[Optional[Tensor]] = [None] * len(paths)
        jpeg = [i for i, t in enumerate(loaded) if not isinstance(t, Tensor)]
        if jpeg:
            images, status = _C.jpeg_decode([loaded[i][0] for i in jpeg], [loaded[i][1] for i in jpeg], device)
            bad = status.cpu().tolist()        # waits for this stream's decode only
            for k, i in enumerate(jpeg):
                if bad[k]:
                    loaded[i] = self.default_loader(paths[i])
                else:
                    out[i] = images[k]
        cpu = [i for i, t in enumerate(loaded) if isinstance(t, Tensor)]
        if cpu:
            for i, t in zip(cpu, self._stage_decoded([loaded[i] for i in cpu], device)):
                out[i] = t
        return out

    def _stage_decoded(self, decoded: List[Tensor], device: torch.device) -> List[Tensor]:
        """CPU-decoded images: the decoder's interleaved HWC bytes are packed into ONE pinned staging buffer and
        cross PCIe as a single asynchronous copy; the letterbox kernel reads HWC uint8 in place
        (`yb_letterbox_strided`), so there is no repacking pass on either side and `/255` stays in the kernel."""
        total = sum(t.numel() for t in decoded)
        slots = self.__dict__.setdefault("_ingest_slots", [None, None])   # double-buffered pinned staging
        k = self.__dict__.get("_ingest_next", 0)
        self.__dict__["_ingest_next"] = k ^ 1
        slot = slots[k]
        if slot is not None:
            slot[1].synchronize()            # the previous copy out of this buffer has finished
        if slot is None or slot[0].numel() < total:
            slot = [torch.empty((max(total, 1 << 20),), dtype=torch.uint8, pin_memory=True), None]
        host = slot[0]
        off = 0
        for t in decoded:
            hwc = t.permute(1, 2, 0)          # read_image returns a CHW view of HWC memory: this is contiguous
            host[off: off + t.numel()].view(hwc.shape).copy_(hwc)
            off += t.numel()
        dev = host[:total].to(device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        slot[1] = ev
        slots[k] = slot
        out, off = [], 0
        for t in decoded:
            _, h, w = t.shape
            out.append(dev[off: off + t.numel()].view(h, w, 3).permute(2, 0, 1))
            off += t.numel()
        return out

    @staticmethod
    def _place_packed(samples, p):
        """Host images that sit back to back in ONE buffer (e.g. slices of a pinned batch tensor) cross PCIe as a
        single asynchronous copy instead of one cudaMemcpy per image; returns None when that does not apply."""
        first = samples[0]
        if first.is_cuda or first.dtype != torch.uint8 and not first.is_floating_point():
            return None
        esz = first.element_size()
        nxt = first.data_ptr()
        for t in samples:
            if t.is_cuda or t.dtype != first.dtype or not t.is_contiguous() or t.data_ptr() != nxt:
                return None
            nxt += t.numel() * esz
        total = (nxt - first.data_ptr()) // esz
        flat = torch.empty(0, dtype=first.dtype).set_(first.untyped_storage(), first.storage_offset(), (total,))
        dev = flat.to(p.device, non_blocking=True)
        if first.dtype != torch.uint8:
            dev = dev.type_as(p)
        out, off = [], 0
        for t in samples:
            out.append(dev[off: off + t.numel()].view(t.shape))
            off += t.numel()
        return out

    @classmethod
    def load_from_yolov5(cls, checkpoint_path: str, *, size: Tuple[int, int] = (640, 640), size_divisible: int = 32,
                         fixed_shape: Optional[Tuple[int, int]] = None, fill_color: int = 114, **kwargs: Any):
        model = YOLO.load_from_yolov5(checkpoint_path, **kwargs)
        return cls(model=model, size=size, size_divisible=size_divisible, fixed_shape=fixed_shape,
                   fill_color=fill_color)
