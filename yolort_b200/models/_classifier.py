"""Plan plumbing shared by the DarkNet image classifiers (`DarkNetV4`, `DarkNetV6`).

`features → avgpool → flatten → classifier` of the reference (yolort/models/darknetv4.py:119-130,
darknetv6.py:116-127) runs as one native plan: the features launch range, one YB_OP_AVGPOOL launch and two 1x1
convolutions for the Linear layers (yolort_b200/engine.py, `lower_darknet`).  `features`, `avgpool` and `classifier`
stay callable sub-modules that execute their own launch range of the owner's plan, so forward hooks on them fire.
"""
import torch
from torch import nn, Tensor

_HEAD_LAUNCHES = 3         # avgpool, classifier.0 (+ Hardswish), classifier.3


def _owner(m: nn.Module) -> "DarkNetClassifier":
    owner = m.__dict__.get("_yb_owner")
    if not owner:
        raise RuntimeError(f"{type(m).__name__} is executed by the sm_90a plan of the DarkNet model that owns it; "
                           "it has no eager PyTorch forward")
    return owner[0]


class PlanFeatures(nn.Sequential):
    """`features`: [N,3,H,W] -> the final feature map [N,C,H/32,W/32] (the features launch range)."""

    def forward(self, x: Tensor) -> Tensor:
        return _owner(self).run_features(x)


class PlanAvgPool(nn.AdaptiveAvgPool2d):
    """`avgpool`: AdaptiveAvgPool2d(1) as the plan's YB_OP_AVGPOOL launch."""

    def __init__(self) -> None:
        super().__init__(1)

    def forward(self, x: Tensor) -> Tensor:
        return _owner(self).run_avgpool(x)


class PlanClassifier(nn.Sequential):
    """`classifier`: Linear -> Hardswish -> Dropout -> Linear as the plan's two 1x1 convolution launches."""

    def forward(self, x: Tensor) -> Tensor:
        return _owner(self).run_classifier(x)


class DarkNetClassifier(nn.Module):
    """Base of DarkNetV4 / DarkNetV6: owns the engine whose plans run the whole classifier."""

    features: PlanFeatures
    avgpool: PlanAvgPool
    classifier: PlanClassifier

    def _attach(self) -> None:
        self._engine = None
        self._last_plan = None
        for m in (self.features, self.avgpool, self.classifier):
            m.__dict__["_yb_owner"] = [self]
        # prepared weights follow the parameters (see YOLO.__init__)
        self.register_load_state_dict_post_hook(lambda module, incompatible_keys: module._drop_engine())

    def _drop_engine(self) -> None:
        self._engine = None
        self._last_plan = None

    def _apply(self, fn, *a, **k):
        self._drop_engine()
        return super()._apply(fn, *a, **k)

    def engine(self):
        from ..engine import Engine

        if self._engine is None:
            p = next(self.parameters())
            dtype = torch.bfloat16 if p.dtype == torch.bfloat16 else torch.float16
            self._engine = Engine(self, dtype, p.device)
        return self._engine

    @property
    def num_classes(self) -> int:
        return self.classifier[3].out_features

    def _out_dtype(self) -> torch.dtype:
        return next(self.parameters()).dtype

    def get_plan(self, N: int, H: int, W: int, keep_intermediates: bool = False):
        if H % 32 or W % 32:
            raise ValueError(f"the canvas must be a multiple of 32 in H and W, got {H}x{W}")
        plan = self.engine().plan(N, H, W, keep_intermediates=keep_intermediates)
        self._last_plan = plan
        return plan

    def _plan_for(self, x: Tensor):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"samples must be [N,3,H,W], got {tuple(x.shape)}")
        N, _, H, W = (int(v) for v in x.shape)
        from .yolo import YOLO

        plan = self.get_plan(N, H, W)
        YOLO._write_samples(plan, x)
        return plan

    def _head_plan(self, N: int):
        """A plan of batch N for the head launches, which do not depend on the canvas: the last one used, or the
        smallest canvas."""
        plan = self._last_plan
        if plan is None or plan.N != N:
            plan = self.get_plan(N, 32, 32)
        return plan

    # -- launch ranges -----------------------------------------------------------------------------------------
    def run_features(self, x: Tensor) -> Tensor:
        plan = self._plan_for(x)
        plan.run(0, plan.plan.n_ops - _HEAD_LAUNCHES)
        return plan.features["features"].permute(0, 3, 1, 2).clone().to(self._out_dtype())

    def run_avgpool(self, f: Tensor) -> Tensor:
        if f.dim() != 4:
            raise ValueError(f"avgpool expects [N,C,h,w], got {tuple(f.shape)}")
        N, _, h, w = (int(v) for v in f.shape)
        plan = self.get_plan(N, 32 * h, 32 * w)
        dst = plan.features["features"]
        if tuple(f.shape) != (N, dst.shape[3], h, w):
            raise ValueError(f"avgpool expects [N,{dst.shape[3]},h,w], got {tuple(f.shape)}")
        dst.copy_(f.permute(0, 2, 3, 1))       # layout change only
        plan.run(plan.plan.n_ops - _HEAD_LAUNCHES, 1)
        return plan.features["avgpool"].permute(0, 3, 1, 2).clone().to(self._out_dtype())

    def run_classifier(self, v: Tensor) -> Tensor:
        plan = self._head_plan(int(v.shape[0]))
        dst = plan.features["avgpool"]
        if v.dim() != 2 or v.shape[1] != dst.shape[3]:
            raise ValueError(f"classifier expects [N,{dst.shape[3]}], got {tuple(v.shape)}")
        dst.view(v.shape[0], -1).copy_(v)
        plan.run(plan.plan.n_ops - 2, 2)
        return self._logits(plan)

    def _logits(self, plan) -> Tensor:
        return plan.heads[0].view(plan.N, -1)[:, : self.num_classes].clone().to(self._out_dtype())

    def has_hooks(self) -> bool:
        return any(m._forward_hooks or m._forward_pre_hooks for m in (self.features, self.avgpool, self.classifier))

    def forward(self, x: Tensor) -> Tensor:
        """[N,3,H,W] (H, W multiples of 32) -> [N, num_classes] logits in the model's dtype."""
        if self.training:
            raise NotImplementedError("training mode is out of scope of this build (the plan implements inference): "
                                      "call .eval()")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"samples must be [N,3,H,W], got {tuple(x.shape)}")
        if x.shape[2] % 32 or x.shape[3] % 32:
            raise ValueError(f"the canvas must be a multiple of 32 in H and W, got {x.shape[2]}x{x.shape[3]}")
        if self.has_hooks():
            # stage by stage through the callable sub-modules, as the reference's _forward_impl does
            return self.classifier(torch.flatten(self.avgpool(self.features(x)), 1))
        plan = self._plan_for(x)
        plan.run()
        return self._logits(plan)


def init_like_reference(model: nn.Module) -> None:
    """BatchNorm eps 1e-3 / momentum 0.03 and in-place activations, as the reference constructors set them
    (darknetv6.py:107-114, darknetv4.py:110-117)."""
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps = 1e-3
            m.momentum = 0.03
        elif isinstance(m, (nn.Hardswish, nn.LeakyReLU, nn.ReLU, nn.ReLU6)):
            m.inplace = True


def pretrained_check(arch: str, pretrained: bool, model_urls: dict) -> None:
    if pretrained and model_urls.get(arch) is None:
        raise NotImplementedError(f"pretrained {arch} is not supported as of now")


def build_head(last_channel: int, num_classes: int) -> PlanClassifier:
    return PlanClassifier(nn.Linear(last_channel, last_channel), nn.Hardswish(inplace=True),
                          nn.Dropout(p=0.2, inplace=True), nn.Linear(last_channel, num_classes))
