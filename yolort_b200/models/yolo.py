"""`YOLO`: backbone + head + post-process on the native plan, and the r6.0 model zoo.

Mirrors the constructor / forward contract of the reference (yolort/models/yolo.py:38-183) and its
factories `yolov5_darknet_pan_{n,s,m,l,x}_r60` (`:468-619`).  `forward(samples[N,3,H,W])` converts the
batch to the plan's input layout with the letterbox kernel (identity geometry), runs the plan and the
decode+NMS kernels; nothing is computed by PyTorch ops.
"""
import math
import os
import warnings
from typing import Any, Callable, Dict, List, Optional

import torch
from torch import nn, Tensor

from .. import _C
from .anchor_utils import AnchorGenerator
from .backbone_utils import darknet_pan_backbone
from .box_head import PostProcess, YOLOHead
from .transformer import darknet_tan_backbone

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
    "yolov5_darknet_tan_s_r40",
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
        self._fp8 = None             # quantization.Fp8Calibration of the FP8 plan (set_fp8), None: fp16 / bf16
        self._fp8_stale = False
        self._fp8_versions = ()
        # `backbone(x)` / `head(features)` are callable sub-modules like the reference's (yolo.py:163-166,
        # utils/hooks.py:7-26): they execute the corresponding launch range of this model's plan.  The owner is
        # reached through a list so that it is neither registered as a sub-module nor lost by deepcopy/pickle.
        self.backbone.__dict__["_yb_owner"] = [self]
        self.head.__dict__["_yb_owner"] = [self]
        # Prepared (BN-folded, packed) weights must follow the parameters.  nn.Module.load_state_dict on a PARENT
        # never calls child.load_state_dict -- it recurses through _load_from_state_dict and fires the post hooks
        # of every sub-module -- so the invalidation is a post hook; `.to()/.half()/.cuda()` reach `_apply`; in-place
        # edits are caught by the engine's parameter-version fingerprint.
        # The same hook makes an FP8 calibration stale (new weights need new activation ranges).
        self.register_load_state_dict_post_hook(lambda module, incompatible_keys: module._drop_engine())

    # -- engine lifetime -----------------------------------------------------------------------------
    def _drop_engine(self) -> None:
        self._engine = None
        if self._fp8 is not None:
            self._fp8_stale = True

    def _apply(self, fn, *a, **k):  # .to()/.half()/.cuda() invalidate prepared weights, and keep an FP8 calibration
        self._engine = None
        if self._fp8 is not None and self._param_versions() != self._fp8_versions:
            self._fp8_stale = True       # edited in place before the move
        out = super()._apply(fn, *a, **k)
        self._fp8_versions = self._param_versions()
        return out

    def _param_versions(self):
        return tuple(t._version for t in list(self.parameters()) + list(self.buffers()))

    def engine(self):
        from ..engine import Engine

        if self._engine is None:
            p = next(self.parameters())
            dtype = torch.bfloat16 if p.dtype == torch.bfloat16 else torch.float16
            self._engine = Engine(self, dtype, p.device)
            self._engine.set_fp8(self._fp8)
        return self._engine

    # -- precision -----------------------------------------------------------------------------------
    @property
    def precision(self) -> str:
        """"fp8" when the plans run in FP8 (set_fp8), else the compute dtype of the parameters: "fp16" or "bf16"."""
        if self._fp8 is not None:
            return "fp8"
        return "bf16" if next(self.parameters()).dtype == torch.bfloat16 else "fp16"

    def set_fp8(self, calib) -> None:
        """Run every later forward on the FP8 (e4m3) plan with the activation ranges of `calib`
        (quantization.calibrate_fp8), or, with None, on the fp16 / bf16 plan again.  The calibration is not part of
        `state_dict()`; save `calib.state_dict()` next to the weights.  It goes stale when the weights change
        (load_state_dict, in-place edits): a forward then raises until set_fp8 is called with a new calibration."""
        if calib is not None:
            from ..engine import fp8_unsupported
            from ..quantization import arch_fingerprint

            why = fp8_unsupported(self)
            if why is not None:
                raise NotImplementedError(f"FP8 inference is not implemented for {why}")
            if calib.fingerprint != arch_fingerprint(self):
                raise ValueError("this FP8 calibration was made for a different architecture")
        self._fp8 = calib
        self._fp8_stale = False
        self._fp8_versions = self._param_versions()
        if self._engine is not None:
            self._engine.set_fp8(calib)

    def _check_fp8(self) -> None:
        if self._fp8 is not None and (self._fp8_stale or self._param_versions() != self._fp8_versions):
            self._fp8_stale = True
            raise RuntimeError("the FP8 calibration is stale: the weights changed after it was set; recalibrate with "
                               "quantization.calibrate_fp8 and call set_fp8 (or set_fp8(None) for fp16 / bf16)")

    # -- anchors -------------------------------------------------------------------------------------
    def set_anchor_grids(self, anchor_grids) -> None:
        """Replace the anchors, per level [aw0, ah0, aw1, ah1, ...] in pixels (float32 values, as upstream's Detect holds
        them in stride units: anchors_px() gives the bits it decodes with).  Every copy follows: the anchor generator,
        the post-process's (or LogitsDecoder's) anchors_px, the criterion's anchor_grids; plan instances, whose fused
        head epilogues bake the anchors, are dropped; the lowered weights are kept."""
        ag = self.anchor_generator
        grids = [[float(v) for v in a] for a in anchor_grids]
        if len(grids) != ag.num_layers or any(len(a) != 2 * ag.num_anchors for a in grids):
            raise ValueError(f"anchor_grids must hold {ag.num_layers} levels of {ag.num_anchors} (w, h) pairs")
        if not all(math.isfinite(v) and v > 0 for a in grids for v in a):
            raise ValueError("anchor sizes must be positive and finite")
        ag.anchor_grids = grids
        px = ag.anchors_px()
        if getattr(self.post_process, "anchors_px", None) is not None:
            self.post_process.anchors_px = px
        if getattr(self.compute_loss, "anchor_grids", None) is not None:
            self.compute_loss.anchor_grids = px
        if self._engine is not None:
            self._engine.drop_plans()

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
        if fuse and self._fp8 is not None:
            raise NotImplementedError("the fused decode epilogue (YB_FUSED_DECODE=1) has no FP8 variant")
        return self.engine().plan(N, H, W, self.post_config() if fuse else None, keep_intermediates, chunked and not fuse)

    def has_hooks(self) -> bool:
        """True when a forward (pre-)hook sits on backbone / head / post_process (yolort/utils/hooks.py:15-17): the
        forward then goes stage by stage through the sub-modules' __call__ so that the hooks fire."""
        return any(m._forward_hooks or m._forward_pre_hooks for m in (self.backbone, self.head, self.post_process))

    @staticmethod
    def _write_samples(plan, samples: Tensor) -> None:
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
        if self._fp8 is not None:       # e4m3 features, dequantised (exactly) into the model's dtype
            dt = next(self.parameters()).dtype
            return [plan.dequantized_feature(k, dt).permute(0, 3, 1, 2).contiguous() for k in sorted(plan.features)]
        return [plan.features[k].permute(0, 3, 1, 2).clone() for k in sorted(plan.features)]

    def run_head(self, features: List[Tensor]) -> List[Tensor]:
        """`head(features)`: the raw per-level logits [N, A, H, W, nc+5] (yolort/models/box_head.py:68-82); the same
        list in training and eval mode.  Differentiable like the reference's nn.Conv2d head when autograd records (grad
        enabled and a head parameter or a feature requires grad): the logits then carry a grad_fn whose backward
        computes the head's weight and bias gradients (csrc/conv_wgrad_sm90.cu) and, for features that require grad,
        the feature gradients.  FP8 plans (set_fp8) keep the logits non-differentiable."""
        features = list(features)
        params = self._head_params()
        if (torch.is_grad_enabled() and self._fp8 is None
                and (any(p.requires_grad for p in params) or any(f.requires_grad for f in features))):
            return list(_HeadFunction.apply(self, len(features), *features, *params))
        return self._run_head_plan(features)

    def _head_params(self) -> List[Tensor]:
        """weight, bias of every level's 1x1 convolution, in level order."""
        return [t for conv in self.head.head for t in (conv.weight, conv.bias)]

    def _run_head_plan(self, features: List[Tensor]) -> List[Tensor]:
        """The head launch range of the plan over `features`; the logits have no grad_fn."""
        # the canvas is the first feature map times its divisor in the lowering (not strides[0]: the lite model's first
        # map sits at stride 16 while its anchor generator says 8)
        self._check_fp8()
        low = self.engine().lowered()
        s0 = low.feats[min(low.feats)].buf.div
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
            if self._fp8 is not None:
                plan.quantize_feature(k, f.permute(0, 2, 3, 1))     # YB_OP_QUANTIZE into the e4m3 feature buffer
            else:
                dst.copy_(f.permute(0, 2, 3, 1))       # layout change only (NCHW caller tensor -> plan NHWC buffer)
        plan.run_heads()
        A, K = self.anchor_generator.num_anchors, self.num_classes + 5
        outs = []
        for hbuf in plan.heads:
            n, h, w, _ = hbuf.shape
            outs.append(hbuf[..., : A * K].view(n, h, w, A, K).permute(0, 3, 1, 2, 4).contiguous())
        return outs

    def _head_backward(self, features: List[Tensor], grads: List[Optional[Tensor]], need_params: bool,
                       need_features: List[bool]):
        """Gradients of the head launch range: (feature gradients, [dW, db] per level).  The incoming gradients go
        into zero-padded [P, C_pad] rows of the compute dtype; one yb_conv_wgrad call computes every level's weight and
        bias gradient in the parameters' dtype; a feature gradient is the 1x1 convolution dY . W on the plan's conv
        kernel (one-op plans cached per shape on the lowering)."""
        if any(p.requires_grad for p in self.backbone.parameters()) and not self.__dict__.get("_yb_warned_backbone"):
            self.__dict__["_yb_warned_backbone"] = True
            warnings.warn(
                "only the detection head is trained: the backbone and neck run on the native plan with their running "
                "BatchNorm statistics and receive no gradient (backward through them is not implemented).  Freeze them "
                "to state this: model.model.backbone.requires_grad_(False) (model.backbone on a YOLO)", UserWarning,
                stacklevel=3)
        from ..engine import head_dgrad

        low = self.engine().lowered()
        dt = low.L.dtype
        A, K = self.anchor_generator.num_anchors, self.num_classes + 5
        convs = list(self.head.head)
        dys, specs, gparams = [], [], []
        for lvl, (f, g, conv) in enumerate(zip(features, grads, convs)):
            n, c, h, w = (int(v) for v in f.shape)
            co = conv.out_channels
            dy = head_dgrad(low, lvl, n, h, w, conv.in_channels).dy if need_features[lvl] else \
                torch.empty((n, h, w, (co + 15) // 16 * 16), dtype=dt, device=f.device)
            if dy.shape[3] > co:
                dy[..., co:].zero_()        # pad channels: the dgrad multiplies them by zero weights, NaN must not reach it
            if g is None:
                dy[..., :co].zero_()
            else:
                dy[..., :co].view(n, h, w, A, K).copy_(g.permute(0, 2, 3, 1, 4))
            dys.append(dy)
            if need_params:
                x = f.permute(0, 2, 3, 1)
                if x.dtype != dt or not x.is_contiguous():
                    x = x.to(dt).contiguous()
                dw = torch.empty((co, c), dtype=conv.weight.dtype, device=f.device)
                db = torch.empty((co,), dtype=conv.bias.dtype, device=f.device)
                specs.append((dy.view(-1, dy.shape[3]), x.reshape(-1, c), dw, db))
                gparams += [dw.view(co, c, 1, 1), db]
        if need_params:
            _C.conv_wgrad(specs, features[0].device)
        gfeats = []
        for lvl, f in enumerate(features):
            if not need_features[lvl]:
                gfeats.append(None)
                continue
            n, c, h, w = (int(v) for v in f.shape)
            gfeats.append(head_dgrad(low, lvl, n, h, w, c).run().permute(0, 3, 1, 2))
        return gfeats, gparams

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

    # -- test-time augmentation (yolort/v5/models/yolo.py:147-208) ------------------------------------------------------
    def augment_unsupported(self) -> Optional[str]:
        """Why `augment=True` cannot run on this model as it stands, or None."""
        from ..relay.logits_decoder import LogitsDecoder

        if self.training:
            return "training mode (test-time augmentation is an inference path; call .eval())"
        if self.has_hooks():
            return ("forward hooks on backbone / head / post_process (the staged path that fires them runs one canvas; "
                    "remove the hooks)")
        if isinstance(self.post_process, LogitsDecoder):
            return "a LogitsDecoder post-process (dense outputs are not merged across passes)"
        bufs = self.engine().lowered().head_bufs
        divs = [b.div for b in bufs]
        if any(b != 2 * a for a, b in zip(divs, divs[1:])):
            return (f"head maps at strides {divs}: _clip_augmented's level arithmetic needs each map half the previous "
                    "one (the MobileNet FPN model's are not)")
        A, K = self.anchor_generator.num_anchors, self.num_classes + 5
        if max(b.C for b in bufs) * 2 > 512:
            return (f"{self.num_classes} classes with {A} anchors: the multi-pass decode reads head rows of at most 256 "
                    f"16-bit logits ({A} x {K} here; at most 80 classes with 3 anchors)")
        return None

    def tta_plans(self, N: int, Hb: int, Wb: int):
        """(pass geometry, plan instance per pass) of augmented inference on an N x Hb x Wb canvas: (nh, nw, Hp, Wp) of
        each pass (_C.tta_pass_geometry with gs = the largest stride); passes of equal canvas shape get distinct plan
        instances (`slot`), so a later pass never overwrites an earlier pass's head logits."""
        gs = int(max(self.anchor_generator.strides))
        geo = _C.tta_pass_geometry(Hb, Wb, gs)
        eng = self.engine()
        plans, seen = [], {}
        for (_, _, hp, wp) in geo:
            slot = seen.get((hp, wp), 0)
            seen[(hp, wp)] = slot + 1
            plans.append(eng.plan(N, hp, wp, slot=slot))
        return geo, plans

    def detect_augmented(self, N: int, Hb: int, Wb: int, write_canvas: Callable[[Tensor], Any],
                         rescale: Optional[Tensor] = None) -> List[Dict[str, Tensor]]:
        """YOLOv5's augmented inference (_forward_augment, yolo.py:152-163) on the plans: `write_canvas(t)` letterboxes
        the batch into the pass-0 canvas t; the pass-1 (0.83, mirrored) and pass-2 (0.67) canvases are rescaled from it
        on the device (yb_canvas_rescale), the three plans run on the current stream, and one multi-pass decode + NMS
        (yb_decode_nms_tta: descale, un-mirror, _clip_augmented, one candidate arena per image) gives the detections,
        with a single device->host read of counts and status.  Always decodes stored logits (no fused epilogue)."""
        why = self.augment_unsupported()
        if why is not None:
            raise NotImplementedError(f"test-time augmentation is not implemented for {why}")
        self._check_fp8()
        # the list holds all three plans for the whole call, so the plan cache's eviction cannot free one mid-call
        geo, plans = self.tta_plans(N, Hb, Wb)
        write_canvas(plans[0].input)
        for q in (1, 2):
            nh, nw, _, _ = geo[q]
            _C.canvas_rescale(plans[0].input, plans[q].input, nh, nw, _C.TTA_FLIPS[q])
        for pl in plans:
            pl.run()
        pc = self.post_config()
        nl = len(plans[0].heads)
        kept = [list(range(nl - 1)), list(range(nl)), list(range(1, nl))]     # _clip_augmented (yolo.py:197-205)
        passes = [(pl.heads, kept[q], _C.TTA_SCALES[q], _C.TTA_FLIPS[q]) for q, pl in enumerate(plans)]
        return _C.decode_nms_tta(passes, Wb, pc["strides"], pc["anchors_px"], pc["num_classes"], pc["score_thresh"],
                                 pc["nms_thresh"], pc["detections_per_img"], pc["semantics"], rescale=rescale)

    def forward(self, samples: Tensor, targets: Optional[Tensor] = None):
        if samples.dim() != 4 or samples.shape[1] != 3:
            raise ValueError(f"samples must be [N,3,H,W], got {tuple(samples.shape)}")
        if self.training or self.has_hooks():
            # stage by stage through the callable sub-modules, as the reference does (yolo.py:162-177)
            features = self.backbone(samples)
            head_outputs = self.head(features)
            if self.training:
                # the training-mode output of the head is the raw per-level list; the criterion (opt-in, e.g.
                # box_head.SetCriterion, box_head.py:85-325) receives what the reference passes
                if self.compute_loss is None:
                    raise NotImplementedError(
                        "training mode returns criterion(targets, head_outputs) and no criterion is set -- construct "
                        "YOLO(..., criterion=SetCriterion(strides, anchor_grids, num_classes)) or call "
                        "model.head(model.backbone(x)) directly")
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


class _HeadFunction(torch.autograd.Function):
    """The plan's head launch range as an autograd node.  Saves the feature tensors it received (never plan arena
    buffers, which the next forward overwrites)."""

    @staticmethod
    def forward(ctx, model: "YOLO", n_feats: int, *args: Tensor):
        feats = list(args[:n_feats])
        outs = model._run_head_plan(feats)
        ctx.model, ctx.n_feats = model, n_feats
        ctx.save_for_backward(*feats)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads: Optional[Tensor]):
        feats = list(ctx.saved_tensors)
        n = ctx.n_feats
        need = ctx.needs_input_grad
        need_features = [bool(need[2 + i]) for i in range(n)]
        need_params = any(need[2 + n:])
        gfeats, gparams = ctx.model._head_backward(feats, list(grads), need_params, need_features)
        if not need_params:
            gparams = [None] * (len(need) - 2 - n)
        return (None, None, *gfeats, *gparams)


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


def yolov5_darknet_tan_s_r40(pretrained: bool = False, progress: bool = True, num_classes: int = 80,
                             **kwargs: Any) -> YOLO:
    """yolov5 small r4.0 with a transformer block (C3TR) as the first block of the neck (yolort/models/yolo.py:837-862,
    yolort/models/transformer.py)."""
    backbone = darknet_tan_backbone("darknet_s_r4_0", 0.33, 0.5, version="r4.0")
    model = YOLO(backbone, num_classes, **kwargs)
    if pretrained:
        raise ValueError(
            "No checkpoint is available offline for model yolov5_darknet_tan_s_r40_coco; load a converted state_dict "
            "with model.load_state_dict(...)")
    return model
