"""`YOLO`: backbone + head + post-process on the native plan, and the r6.0 model zoo.

Mirrors the constructor / forward contract of the reference (yolort/models/yolo.py:38-183) and its
factories `yolov5_darknet_pan_{n,s,m,l,x}_r60` (`:468-619`).  `forward(samples[N,3,H,W])` converts the
batch to the plan's input layout with the letterbox kernel (identity geometry), runs the plan and the
decode+NMS kernels; nothing is computed by PyTorch ops.
"""
import os
from typing import Any, Callable, Dict, List, Optional

import torch
from torch import nn, Tensor

from .. import _C
from .anchor_utils import AnchorGenerator
from .backbone_utils import darknet_pan_backbone
from .box_head import PostProcess, YOLOHead

__all__ = [
    "YOLO",
    "yolov5_darknet_pan_s_r31",
    "yolov5_darknet_pan_m_r31",
    "yolov5_darknet_pan_l_r31",
    "yolov5_darknet_pan_s_r40",
    "yolov5_darknet_pan_m_r40",
    "yolov5_darknet_pan_l_r40",
    "yolov5_darknet_pan_n_r60",
    "yolov5_darknet_pan_s_r60",
    "yolov5_darknet_pan_m_r60",
    "yolov5_darknet_pan_l_r60",
    "yolov5_darknet_pan_x_r60",
    "yolov5_darknet_pan_n6_r60",
    "yolov5_darknet_pan_s6_r60",
    "yolov5_darknet_pan_m6_r60",
    "yolov5_darknet_pan_l6_r60",
    "yolov5_darknet_pan_x6_r60",
]

DEFAULT_STRIDES = [8, 16, 32]
DEFAULT_ANCHOR_GRIDS = [
    [10, 13, 16, 30, 33, 23],
    [30, 61, 62, 45, 59, 119],
    [116, 90, 156, 198, 373, 326],
]
# P6 variants (yolort/models/yolo.py:641-647; the same table in every *6 factory)
P6_STRIDES = [8, 16, 32, 64]
P6_ANCHOR_GRIDS = [
    [19, 27, 44, 40, 38, 94],
    [96, 68, 86, 152, 180, 137],
    [140, 301, 303, 264, 238, 542],
    [436, 615, 739, 380, 925, 792],
]


class YOLO(nn.Module):
    def __init__(
        self,
        backbone: nn.Module,
        num_classes: int,
        strides: Optional[List[int]] = None,
        anchor_grids: Optional[List[List[float]]] = None,
        anchor_generator: Optional[nn.Module] = None,
        head: Optional[nn.Module] = None,
        criterion: Optional[Callable[..., Dict[str, Tensor]]] = None,
        score_thresh: float = 0.005,
        nms_thresh: float = 0.45,
        detections_per_img: int = 300,
        post_process: Optional[nn.Module] = None,
    ):
        super().__init__()
        if not hasattr(backbone, "out_channels"):
            raise ValueError(
                "backbone should contain an attribute out_channels specifying the number of output "
                "channels (assumed to be the same for all the levels)")
        self.backbone = backbone
        # accept tensors too: the reference loader passes `model.stride` as a Tensor (SURVEY.md 0.10)
        strides = DEFAULT_STRIDES if strides is None else [int(s) for s in strides]
        anchor_grids = DEFAULT_ANCHOR_GRIDS if anchor_grids is None else anchor_grids
        if anchor_generator is None:
            anchor_generator = AnchorGenerator(strides, anchor_grids)
        self.anchor_generator = anchor_generator
        self.compute_loss = criterion  # training loss is out of scope (SURVEY.md section 2, row 6)
        self.num_classes = num_classes
        if head is None:
            head = YOLOHead(backbone.out_channels, anchor_generator.num_anchors, anchor_generator.strides, num_classes)
        self.head = head
        if post_process is None:
            post_process = PostProcess(anchor_generator.strides, score_thresh, nms_thresh, detections_per_img,
                                       anchors_px=anchor_generator.anchors_px())
        self.post_process = post_process
        self._engine = None
        # `backbone(x)` / `head(features)` are callable sub-modules like the reference's (yolo.py:163-166,
        # utils/hooks.py:7-26): they execute the corresponding launch range of this model's plan.  The owner is
        # reached through a list so that it is neither registered as a sub-module nor lost by deepcopy/pickle.
        self.backbone.__dict__["_yb_owner"] = [self]
        self.head.__dict__["_yb_owner"] = [self]
        # Prepared (BN-folded, packed) weights must follow the parameters.  nn.Module.load_state_dict on a PARENT
        # never calls child.load_state_dict -- it recurses through _load_from_state_dict and fires the post hooks
        # of every sub-module -- so the invalidation is a post hook; `.to()/.half()/.cuda()` reach `_apply`; in-place
        # edits are caught by the engine's parameter-version fingerprint.
        self.register_load_state_dict_post_hook(lambda module, incompatible_keys: module._drop_engine())

    # -- engine lifetime -----------------------------------------------------------------------------
    def _drop_engine(self) -> None:
        self._engine = None

    def _apply(self, fn, *a, **k):  # .to()/.half()/.cuda() invalidate prepared weights
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self):
        from ..engine import Engine

        if self._engine is None:
            p = next(self.parameters())
            dtype = torch.bfloat16 if p.dtype == torch.bfloat16 else torch.float16
            self._engine = Engine(self, dtype, p.device)
        return self._engine

    # -- stages --------------------------------------------------------------------------------------
    def post_config(self) -> dict:
        """Post-processing parameters baked into a plan's fused head epilogues / NMS arena."""
        pp = self.post_process
        ag = self.anchor_generator
        if not hasattr(pp, "score_thresh"):
            raise NotImplementedError(f"{type(pp).__name__} has no thresholded detections; call the model's forward")
        return {"strides": list(pp.strides), "anchors_px": ag.anchors_px(), "n_anchors": ag.num_anchors,
                "num_classes": self.num_classes, "score_thresh": float(pp.score_thresh),
                "nms_thresh": float(pp.nms_thresh), "detections_per_img": int(pp.detections_per_img),
                "semantics": int(getattr(pp, "nms_semantics", _C.NMS_TV_AUTO))}

    def get_plan(self, N: int, H: int, W: int, keep_intermediates: bool = False, chunked: bool = False):
        """Plan instance for a batch of N canvases of H x W.  `keep_intermediates=True` gives every activation its
        own bytes (inspection / stage-wise tests); the default arena reuses the bytes of dead activations.
        `chunked=True`: the variant `YOLOv5.predict` uses for host inputs (front ops runnable per image chunk)."""
        # The fused decode epilogue (heads emit NMS candidates instead of logits) is functional; opt-in until it is
        # shown to be faster than storing fp16 logits + the stand-alone decode kernel.
        fuse = os.environ.get("YB_FUSED_DECODE", "0") == "1"
        return self.engine().plan(N, H, W, self.post_config() if fuse else None, keep_intermediates, chunked and not fuse)

    def has_hooks(self) -> bool:
        """True when a forward (pre-)hook sits on backbone / head / post_process (yolort/utils/hooks.py:15-17): the
        forward then goes stage by stage through the sub-modules' __call__ so that the hooks fire."""
        return any(m._forward_hooks or m._forward_pre_hooks for m in (self.backbone, self.head, self.post_process))

    def _write_samples(self, plan, samples: Tensor) -> None:
        """A pre-letterboxed NCHW batch -> the plan's space-to-depth input (identity geometry)."""
        N, _, H, W = (int(v) for v in samples.shape)
        geoms = (_C.LetterboxGeom * N)()
        for g in geoms:
            g.src_h, g.src_w, g.new_h, g.new_w, g.top, g.left = H, W, H, W, 0, 0
            g.ratio_h = g.ratio_w = 1.0
        samples = samples.contiguous()
        _C.letterbox([samples[i] for i in range(N)], geoms, H, W, 0.0, plan.input, _C.YB_LAYOUT_S2D16)

    def run_backbone(self, samples: Tensor) -> List[Tensor]:
        """`backbone(samples)`: body + PAN; NCHW feature maps (yolort/models/backbone_utils.py:54-57)."""
        if samples.dim() != 4 or samples.shape[1] != 3:
            raise ValueError(f"samples must be [N,3,H,W], got {tuple(samples.shape)}")
        N, _, H, W = (int(v) for v in samples.shape)
        plan = self.get_plan(N, H, W)
        self._write_samples(plan, samples)
        plan.run_backbone()
        return [plan.features[k].permute(0, 3, 1, 2).clone() for k in sorted(plan.features)]

    def run_head(self, features: List[Tensor]) -> List[Tensor]:
        """`head(features)`: the raw per-level logits [N, A, H, W, nc+5] (yolort/models/box_head.py:68-82); the same
        list in training and eval mode."""
        s0 = int(self.anchor_generator.strides[0])
        N, _, h0, w0 = (int(v) for v in features[0].shape)
        plan = self.get_plan(N, h0 * s0, w0 * s0)
        keys = sorted(plan.features)
        if len(features) != len(keys):
            raise ValueError(f"head expects {len(keys)} feature maps, got {len(features)}")
        for k, f in zip(keys, features):
            dst = plan.features[k]
            if tuple(f.shape) != (dst.shape[0], dst.shape[3], dst.shape[1], dst.shape[2]):
                raise ValueError(f"feature {k}: expected [N,{dst.shape[3]},{dst.shape[1]},{dst.shape[2]}], got {tuple(f.shape)}")
            _C.require_cuda(f, "head")
            dst.copy_(f.permute(0, 2, 3, 1))       # layout change only (NCHW caller tensor -> plan NHWC buffer)
        plan.run_heads()
        A, K = self.anchor_generator.num_anchors, self.num_classes + 5
        outs = []
        for hbuf in plan.heads:
            n, h, w, _ = hbuf.shape
            outs.append(hbuf[..., : A * K].view(n, h, w, A, K).permute(0, 3, 1, 2, 4).contiguous())
        return outs

    def run_plan(self, plan) -> List[Tensor]:
        """backbone + PAN + head on the prepared input canvas; returns the raw head logits (NHWC)."""
        plan.run()
        return plan.heads

    def post_padded(self, plan, rescale: Optional[Tensor] = None):
        """Post-processing over the head logits a plan has already produced; padded device outputs."""
        pc = self.post_config()
        return _C.decode_nms_padded(plan.heads, "nhwc", pc["strides"], pc["anchors_px"], pc["num_classes"],
                                    pc["score_thresh"], pc["nms_thresh"], pc["detections_per_img"], pc["semantics"],
                                    rescale)

    def detect_padded(self, plan, rescale: Optional[Tensor] = None):
        """Runs the plan and the post-processing; padded device outputs, no host synchronisation."""
        if plan.fused_post is not None:
            fp = plan.fused_post
            fp.begin()
            plan.run_fused()
            return fp.finish(rescale)
        heads = self.run_plan(plan)
        pc = self.post_config()
        return _C.decode_nms_padded(heads, "nhwc", pc["strides"], pc["anchors_px"], pc["num_classes"],
                                    pc["score_thresh"], pc["nms_thresh"], pc["detections_per_img"], pc["semantics"],
                                    rescale)

    def detect(self, plan, rescale: Optional[Tensor] = None):
        from ..relay.logits_decoder import LogitsDecoder

        if isinstance(self.post_process, LogitsDecoder):
            # relay/trt_inference.py:43: post_process=LogitsDecoder(strides) -> dense (boxes, scores), canvas coordinates
            heads = self.run_plan(plan)
            return self.post_process.decode_plan_heads(heads, self.anchor_generator.anchors_px(), self.num_classes)
        pc = self.post_config()
        if plan.fused_post is not None:
            boxes, scores, labels, counts, status = self.detect_padded(plan, rescale)
            n = counts.numel()
            host = torch.cat([counts.to(torch.int64), status]).tolist()     # one D2H + one conversion for the whole batch
            if host[n + 1] == 0:
                return [{"scores": scores[i, :host[i]], "labels": labels[i, :host[i]], "boxes": boxes[i, :host[i]]}
                        for i in range(n)]
            # an image overflowed its share of the fixed arena: redo the post-processing on stored logits with the
            # growable arena (never truncate)
        heads = self.run_plan(plan)
        return _C.decode_nms(heads, "nhwc", pc["strides"], pc["anchors_px"], pc["score_thresh"], pc["nms_thresh"],
                             pc["detections_per_img"], pc["semantics"], rescale=rescale, num_classes=self.num_classes)

    def forward(self, samples: Tensor, targets: Optional[Tensor] = None):
        if samples.dim() != 4 or samples.shape[1] != 3:
            raise ValueError(f"samples must be [N,3,H,W], got {tuple(samples.shape)}")
        if self.training or self.has_hooks():
            # stage by stage through the callable sub-modules, as the reference does (yolo.py:162-177)
            features = self.backbone(samples)
            head_outputs = self.head(features)
            if self.training:
                # the training-mode output of the head is the raw per-level list; the loss itself (SetCriterion,
                # box_head.py:85-325) is out of scope, a caller-supplied criterion receives what the reference passes
                if self.compute_loss is None:
                    raise NotImplementedError(
                        "training mode returns criterion(targets, head_outputs); SetCriterion is out of scope of this "
                        "build -- construct YOLO(..., criterion=...) or call model.head(model.backbone(x)) directly")
                return self.compute_loss(targets, head_outputs)
            return self.post_process(head_outputs, None, None)
        if targets is not None:
            raise NotImplementedError("targets are only used by the training path; call .train() with a criterion")
        N, _, H, W = (int(v) for v in samples.shape)
        plan = self.get_plan(N, H, W)
        self._write_samples(plan, samples)
        return self.detect(plan)

    @classmethod
    def load_from_yolov5(cls, checkpoint_path: str, score_thresh: float = 0.25, nms_thresh: float = 0.45,
                         version: str = "r6.0", post_process: Optional[nn.Module] = None):
        from ._checkpoint import load_from_ultralytics

        info = load_from_ultralytics(checkpoint_path, version=version)
        backbone = darknet_pan_backbone(f"darknet_{info['size']}_{version.replace('.', '_')}", info["depth_multiple"],
                                        info["width_multiple"], version=version, use_p6=info["use_p6"])
        model = cls(backbone, info["num_classes"], strides=info["strides"], anchor_grids=info["anchor_grids"],
                    score_thresh=score_thresh, nms_thresh=nms_thresh, post_process=post_process)
        model.load_state_dict(info["state_dict"])
        return model


def build_model(backbone_name: str, depth_multiple: float, width_multiple: float, version: str,
                weights_name: Optional[str] = None, pretrained: bool = False, progress: bool = True,
                num_classes: int = 80, use_p6: bool = False, **kwargs: Any) -> YOLO:
    backbone = darknet_pan_backbone(backbone_name, depth_multiple, width_multiple, version=version, use_p6=use_p6)
    model = YOLO(backbone, num_classes, **kwargs)
    if pretrained:
        raise ValueError(
            f"No checkpoint is available offline for model {weights_name}; load a converted state_dict with "
            "model.load_state_dict(...) or an upstream .pt with YOLO.load_from_yolov5(...)")
    return model


def _factory(size: str, depth: float, width: float, use_p6: bool = False, version: str = "r6.0"):
    six = "6" if use_p6 else ""
    vtag, vname = version.replace(".", ""), version.replace(".", "_")

    def fn(pretrained: bool = False, progress: bool = True, num_classes: int = 80, **kwargs: Any) -> YOLO:
        if use_p6:   # yolo.py:640-661: the *6 factories pin strides and anchor grids
            kwargs = dict(kwargs, strides=P6_STRIDES, anchor_grids=P6_ANCHOR_GRIDS)
        return build_model(f"darknet_{size}_{vname}", depth, width, version, f"yolov5_darknet_pan_{size}{six}_{vtag}_coco",
                           pretrained, progress, num_classes, use_p6=use_p6, **kwargs)

    fn.__name__ = f"yolov5_darknet_pan_{size}{six}_{vtag}"
    fn.__doc__ = (f"yolov5 {size}{six} release {version[1:]} (depth_multiple={depth}, width_multiple={width}"
                  + (", P6: 4 levels, strides 8..64)." if use_p6 else ")."))
    return fn


# r3.1 / r4.0 (Focus stem; BottleneckCSP+Hardswish / C3+SiLU): yolort/models/yolo.py:292-469
yolov5_darknet_pan_s_r31 = _factory("s", 0.33, 0.5, version="r3.1")
yolov5_darknet_pan_m_r31 = _factory("m", 0.67, 0.75, version="r3.1")
yolov5_darknet_pan_l_r31 = _factory("l", 1.0, 1.0, version="r3.1")
yolov5_darknet_pan_s_r40 = _factory("s", 0.33, 0.5, version="r4.0")
yolov5_darknet_pan_m_r40 = _factory("m", 0.67, 0.75, version="r4.0")
yolov5_darknet_pan_l_r40 = _factory("l", 1.0, 1.0, version="r4.0")
# (depth, width) table: yolort/models/yolo.py:468-619
yolov5_darknet_pan_n_r60 = _factory("n", 0.33, 0.25)
yolov5_darknet_pan_s_r60 = _factory("s", 0.33, 0.5)
yolov5_darknet_pan_m_r60 = _factory("m", 0.67, 0.75)
yolov5_darknet_pan_l_r60 = _factory("l", 1.0, 1.0)
yolov5_darknet_pan_x_r60 = _factory("x", 1.33, 1.25)
# P6 table: yolort/models/yolo.py:622-834
yolov5_darknet_pan_n6_r60 = _factory("n", 0.33, 0.25, use_p6=True)
yolov5_darknet_pan_s6_r60 = _factory("s", 0.33, 0.5, use_p6=True)
yolov5_darknet_pan_m6_r60 = _factory("m", 0.67, 0.75, use_p6=True)
yolov5_darknet_pan_l6_r60 = _factory("l", 1.0, 1.0, use_p6=True)
yolov5_darknet_pan_x6_r60 = _factory("x", 1.33, 1.25, use_p6=True)
