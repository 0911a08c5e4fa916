"""TAN neck of `yolov5ts` -- parameter container (yolort/models/transformer.py).

The r4.0 PAN with one difference: `inner_blocks[0]` is a C3TR (C3 with a transformer block, common.py:360-367)
instead of a C3 (transformer.py:85-100).  Only r4.0 without P6 exists in the reference (`:47-48`).  The data flow is
the PAN's; the transformer block is lowered by yolort_b200/engine.py (`_Lowering.c3tr`).
"""
from typing import List, Optional

from torch import nn

from ._utils import depth_gain
from .backbone_utils import BackboneWithPAN
from .common import C3TR
from .darknetv4 import darknet_v4_features
from .path_aggregation_network import PathAggregationNetwork


class TransformerAttentionNetwork(PathAggregationNetwork):
    def __init__(self, in_channels_list: List[int], depth_multiple: float, version: str = "r4.0"):
        if len(in_channels_list) != 3 or version != "r4.0":
            raise NotImplementedError("the transformer attention network exists for r4.0 with 3 levels only")
        super().__init__(in_channels_list, depth_multiple, version=version)
        ch = list(in_channels_list)
        self.inner_blocks[0] = C3TR(ch[2], ch[2], n=depth_gain(3, depth_multiple), shortcut=False)


class BackboneWithTAN(BackboneWithPAN):
    """BackboneWithPAN with the TAN as its neck (transformer.py:62-74)."""

    def __init__(self, body: nn.Sequential, returned_layers: List[int], in_channels_list: List[int],
                 depth_multiple: float):
        super().__init__(body, returned_layers, in_channels_list, depth_multiple, "r4.0")
        self.pan = TransformerAttentionNetwork(in_channels_list, depth_multiple, version="r4.0")


def darknet_tan_backbone(
    backbone_name: str,
    depth_multiple: float,
    width_multiple: float,
    pretrained: Optional[bool] = False,
    returned_layers: Optional[List[int]] = None,
    version: str = "r4.0",
    use_p6: bool = False,
) -> BackboneWithTAN:
    """transformer.py:13-59: r4.0 CSPDarknet body (SPP closing the body) + TAN."""
    if version != "r4.0":
        raise NotImplementedError("Currently only supports version r4.0.")
    if use_p6:
        raise NotImplementedError("Currently doesn't support the P6 structure.")
    if pretrained:
        raise ValueError("no backbone checkpoints exist offline")
    body = darknet_v4_features(depth_multiple, width_multiple, version=version)
    if returned_layers is None:
        returned_layers = [4, 6, 8]
    in_channels_list = [int(gw * width_multiple) for gw in [256, 512, 1024]]
    return BackboneWithTAN(body, returned_layers, in_channels_list, depth_multiple)
