"""`yolov5_mobilenet_v3_small_fpn`: YOLO with a MobileNetV3-Small + FPN backbone (yolort/models/yolo_lite.py).

torchvision's MobileNetV3 features, `FrozenBatchNorm2d`, `IntermediateLayerGetter` and `FeaturePyramidNetwork` are
used as parameter containers only, so that state-dict keys, order and shapes match the reference by construction.  Their
PyTorch forward never runs: `BackboneWithFPN.forward` executes the backbone launch range of the owning YOLO's plan,
which yolort_b200/engine.py (`lower_lite`) builds from these modules.

The feature maps sit at strides 16, 32, 32 and 64 while the anchor generator says 8, 16, 32 and 64; the heads are
decoded with the latter, as in the reference (yolo_lite.py:125-131).
"""
import os
from typing import Callable, Dict, List, Optional

import torch
from torch import nn
from torchvision.models import mobilenet
from torchvision.models._utils import IntermediateLayerGetter
from torchvision.models.detection.backbone_utils import _validate_trainable_layers
from torchvision.ops import misc as misc_nn_ops
from torchvision.ops.feature_pyramid_network import ExtraFPNBlock, FeaturePyramidNetwork, LastLevelMaxPool

from .anchor_utils import AnchorGenerator
from .box_head import YOLOHead
from .yolo import YOLO

__all__ = ["yolov5_mobilenet_v3_small_fpn"]

# torchvision's ImageNet weights of each backbone (what `pretrained=True` of torchvision's constructors downloads)
_BACKBONE_WEIGHTS = {
    "mobilenet_v3_small": "https://download.pytorch.org/models/mobilenet_v3_small-047dcff4.pth",
}


class BackboneWithFPN(nn.Module):
    """IntermediateLayerGetter over the MobileNetV3 features + FeaturePyramidNetwork (yolo_lite.py:18-63).

    Args:
        backbone (nn.Module)
        return_layers (Dict[name, new_name]): modules of `backbone` whose activations are returned
        in_channels_list (List[int]): channels of each returned feature map
        out_channels (int): channels of the FPN
    """

    def __init__(self, backbone: nn.Module, return_layers: Dict[str, str], in_channels_list: List[int],
                 out_channels: int, extra_blocks: Optional[ExtraFPNBlock] = None) -> None:
        super().__init__()
        if extra_blocks is None:
            extra_blocks = LastLevelMaxPool()
        self.body = IntermediateLayerGetter(backbone, return_layers=return_layers)
        self.fpn = FeaturePyramidNetwork(in_channels_list=in_channels_list, out_channels=out_channels,
                                         extra_blocks=extra_blocks)
        self.out_channels = out_channels

    def forward(self, x):
        """`backbone(x)`: [N,3,H,W] -> the FPN maps [N,256,H/s,W/s] for s = 16, 32, 32, 64, executed as the backbone
        launch range of the owning YOLO's plan (forward hooks fire)."""
        owner = self.__dict__.get("_yb_owner")
        if not owner:
            raise RuntimeError("BackboneWithFPN is executed by the sm_90a plan of the YOLO model that owns it; "
                               "it has no eager PyTorch forward")
        return owner[0].run_backbone(x)


def _load_backbone_weights(backbone_name: str, model: nn.Module) -> None:
    """Loads torchvision's ImageNet weights from the torch hub cache.  Never downloads: a missing file is an error."""
    url = _BACKBONE_WEIGHTS.get(backbone_name)
    if url is None:
        raise ValueError(f"no ImageNet weights are known for backbone {backbone_name}")
    path = os.path.join(torch.hub.get_dir(), "checkpoints", os.path.basename(url))
    if not os.path.isfile(path):
        raise ValueError(
            f"pretrained_backbone=True needs torchvision's ImageNet weights at {path}, and they are not there (this "
            "package does not download). Place the file there, or construct the model with pretrained_backbone=False "
            "and load weights with load_state_dict(...)")
    model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))


def mobilenet_backbone(
    backbone_name: str,
    pretrained: bool,
    norm_layer: Callable[..., nn.Module] = misc_nn_ops.FrozenBatchNorm2d,
    trainable_layers: int = 2,
    returned_layers: Optional[List[int]] = None,
) -> nn.Module:
    """yolo_lite.py:66-105: torchvision MobileNetV3 features, the stages before the last `trainable_layers` frozen,
    and the last three stages returned to an FPN of 256 channels."""
    net = mobilenet.__dict__[backbone_name](weights=None, norm_layer=norm_layer)
    if pretrained:
        _load_backbone_weights(backbone_name, net)
    backbone = net.features

    # the strided blocks start stages C1 .. Cn-1; the first and the last module are always stages
    stage_indices = [0] + [i for i, b in enumerate(backbone) if getattr(b, "_is_cn", False)] + [len(backbone) - 1]
    num_stages = len(stage_indices)
    if not 0 <= trainable_layers <= num_stages:
        raise ValueError(f"trainable_layers must be in [0, {num_stages}], got {trainable_layers}")
    freeze_before = len(backbone) if trainable_layers == 0 else stage_indices[num_stages - trainable_layers]
    for b in backbone[:freeze_before]:
        for parameter in b.parameters():
            parameter.requires_grad_(False)

    out_channels = 256
    if returned_layers is None:
        returned_layers = [num_stages - 3, num_stages - 2, num_stages - 1]
    if not (min(returned_layers) >= 0 and max(returned_layers) < num_stages):
        raise ValueError(f"returned_layers must lie in [0, {num_stages}), got {returned_layers}")
    return_layers = {f"{stage_indices[k]}": str(v) for v, k in enumerate(returned_layers)}
    in_channels_list = [backbone[stage_indices[i]].out_channels for i in returned_layers]
    return BackboneWithFPN(backbone, return_layers, in_channels_list, out_channels, extra_blocks=LastLevelMaxPool())


model_urls = {
    "yolov5_mobilenet_v3_small_fpn_coco": None,
}


def _yolov5_mobilenet_v3_small_fpn(
    weights_name: str,
    pretrained: bool = False,
    progress: bool = True,
    num_classes: int = 80,
    pretrained_backbone: bool = True,
    trainable_backbone_layers: Optional[int] = None,
    **kwargs,
):
    trainable_backbone_layers = _validate_trainable_layers(pretrained or pretrained_backbone, trainable_backbone_layers,
                                                           6, 3)
    if pretrained:
        pretrained_backbone = False
        if model_urls.get(weights_name, None) is None:   # checked before anything is built: nothing to download
            raise ValueError(f"No checkpoint is available for model {weights_name}")
    backbone = mobilenet_backbone("mobilenet_v3_small", pretrained_backbone, trainable_layers=trainable_backbone_layers)
    strides = [8, 16, 32, 64]
    anchor_grids = [
        [19, 27, 44, 40, 38, 94],
        [96, 68, 86, 152, 180, 137],
        [140, 301, 303, 264, 238, 542],
        [436, 615, 739, 380, 925, 792],
    ]
    anchor_generator = AnchorGenerator(strides, anchor_grids)
    head = YOLOHead(backbone.out_channels, anchor_generator.num_anchors, anchor_generator.strides, num_classes)
    return YOLO(backbone, num_classes, anchor_generator=anchor_generator, head=head, **kwargs)


def yolov5_mobilenet_v3_small_fpn(
    pretrained: bool = False,
    progress: bool = True,
    num_classes: int = 80,
    pretrained_backbone: bool = True,
    trainable_backbone_layers: Optional[int] = None,
    **kwargs,
):
    """YOLOv5 detector with a MobileNetV3-Small FPN backbone (yolo_lite.py:151-191).  There are no COCO weights.

    Args:
        pretrained (bool): COCO weights; none exist, so True raises ValueError
        progress (bool): accepted for signature compatibility
        num_classes (int): number of output classes
        pretrained_backbone (bool): load torchvision's ImageNet weights into the backbone.  They are read from the torch
            hub cache (`<hub dir>/checkpoints/mobilenet_v3_small-047dcff4.pth`) and never downloaded; a missing file
            raises ValueError
        trainable_backbone_layers (int): number of trainable stages counted from the last one, 0 to 6 (only with
            pretrained weights; otherwise all 6 stages stay trainable)
    """
    weights_name = "yolov5_mobilenet_v3_small_fpn_coco"
    return _yolov5_mobilenet_v3_small_fpn(weights_name, pretrained=pretrained, progress=progress,
                                          num_classes=num_classes, pretrained_backbone=pretrained_backbone,
                                          trainable_backbone_layers=trainable_backbone_layers, **kwargs)
