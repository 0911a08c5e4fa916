"""CSPDarknet (r3.1 / r4.0): the detection body and the DarkNetV4 image classifier.

Layout and channel rules follow the reference (yolort/models/darknetv4.py:33-220): Focus stem, three [3x3/s2 Conv,
block] stages with repeats [3, 9, 9] and widths [128, 256, 512], a 3x3/s2 Conv and the SPP; block = BottleneckCSP
(r3.1) or C3 (r4.0).  Module indices 0..8 are what the PAN taps (4, 6, 8 -- the last one is the SPP output) and what
the state-dict keys are built from.  The classifier adds `avgpool` and `classifier` (Linear -> Hardswish -> Dropout ->
Linear) and runs on the native plan (models/_classifier.py).
"""
from typing import Any, Callable, List, Optional

from torch import nn

from ._classifier import DarkNetClassifier, PlanAvgPool, PlanFeatures, build_head, init_like_reference, pretrained_check
from ._utils import depth_gain, make_divisible
from .common import BottleneckCSP, C3, Conv, Focus, SPP

__all__ = [
    "DarkNetV4",
    "darknet_s_r3_1",
    "darknet_m_r3_1",
    "darknet_l_r3_1",
    "darknet_s_r4_0",
    "darknet_m_r4_0",
    "darknet_l_r4_0",
]

model_urls = {
    "darknet_s_r3.1": None,
    "darknet_m_r3.1": None,
    "darknet_l_r3.1": None,
    "darknet_s_r4.0": None,
    "darknet_m_r4.0": None,
    "darknet_l_r4.0": None,
}

BLOCKS = {"r3.1": BottleneckCSP, "r4.0": C3}


def darknet_v4_features(depth_multiple: float, width_multiple: float, version: str = "r4.0",
                        last_channel: int = 1024, block: Optional[Callable[..., nn.Module]] = None,
                        stages_repeats: Optional[List[int]] = None, stages_out_channels: Optional[List[int]] = None,
                        round_nearest: int = 8) -> nn.Sequential:
    if version not in BLOCKS:
        raise NotImplementedError("Currently the module version used in DarkNetV4 is r3.1 or r4.0")
    block = BLOCKS[version] if block is None else block
    stages_repeats = [3, 9, 9] if stages_repeats is None else stages_repeats
    stages_out_channels = [128, 256, 512] if stages_out_channels is None else stages_out_channels
    c_in = make_divisible(64 * width_multiple, round_nearest)
    layers: List[nn.Module] = [Focus(3, c_in, k=3, version=version)]
    for n, c in zip(stages_repeats, stages_out_channels):
        c_out = make_divisible(c * width_multiple, round_nearest)
        layers.append(Conv(c_in, c_out, k=3, s=2, version=version))
        layers.append(block(c_out, c_out, n=depth_gain(n, depth_multiple)))
        c_in = c_out
    last = make_divisible(last_channel * width_multiple, round_nearest)
    layers.append(Conv(c_in, last, k=3, s=2, version=version))
    layers.append(SPP(last, last, k=(5, 9, 13), version=version))
    return nn.Sequential(*layers)


class DarkNetV4(DarkNetClassifier):
    """
    DarkNetV4 main class

    Args:
        depth_multiple (float): Depth multiplier
        width_multiple (float): Width multiplier - adjusts number of channels in each layer by this amount
        version (str): Module version released by ultralytics: "r3.1" or "r4.0".
        block: Module specifying the building block of the stages (BottleneckCSP for r3.1, C3 for r4.0 by default;
            the plan lowers these two)
        stages_repeats (Optional[List[int]]): List of repeats number in the stages.
        stages_out_channels (Optional[List[int]]): List of channels number in the stages.
        num_classes (int): Number of classes
        round_nearest (int): Round the number of channels in each layer to be a multiple of this number.
            Set to 1 to turn off rounding
        last_channel (int): Number of the last channel
    """

    def __init__(
        self,
        depth_multiple: float,
        width_multiple: float,
        version: str = "r4.0",
        block: Optional[Callable[..., nn.Module]] = None,
        stages_repeats: Optional[List[int]] = None,
        stages_out_channels: Optional[List[int]] = None,
        num_classes: int = 1000,
        round_nearest: int = 8,
        last_channel: int = 1024,
    ) -> None:
        super().__init__()
        assert version in ["r3.1", "r4.0"], "Currently the module version used in DarkNetV4 is r3.1 or r4.0"
        self.features = PlanFeatures(*darknet_v4_features(depth_multiple, width_multiple, version, last_channel, block,
                                                          stages_repeats, stages_out_channels, round_nearest))
        last = make_divisible(last_channel * width_multiple, round_nearest)
        self.avgpool = PlanAvgPool()
        self.classifier = build_head(last, num_classes)
        init_like_reference(self)
        self._attach()


def _darknet_v4_conf(arch: str, pretrained: bool, progress: bool, *args: Any, **kwargs: Any) -> DarkNetV4:
    pretrained_check(arch, pretrained, model_urls)
    return DarkNetV4(*args, **kwargs)


def darknet_s_r3_1(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 3.1 with small channels (depth 0.33, width 0.5).  `pretrained=True` raises
    NotImplementedError: no weights exist."""
    return _darknet_v4_conf("darknet_s_r3.1", pretrained, progress, 0.33, 0.5, version="r3.1", **kwargs)


def darknet_m_r3_1(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 3.1 with medium channels (depth 0.67, width 0.75)."""
    return _darknet_v4_conf("darknet_m_r3.1", pretrained, progress, 0.67, 0.75, version="r3.1", **kwargs)


def darknet_l_r3_1(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 3.1 with large channels (depth 1.0, width 1.0)."""
    return _darknet_v4_conf("darknet_l_r3.1", pretrained, progress, 1.0, 1.0, version="r3.1", **kwargs)


def darknet_s_r4_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 4.0 with small channels (depth 0.33, width 0.5)."""
    return _darknet_v4_conf("darknet_s_r4.0", pretrained, progress, 0.33, 0.5, version="r4.0", **kwargs)


def darknet_m_r4_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 4.0 with medium channels (depth 0.67, width 0.75)."""
    return _darknet_v4_conf("darknet_m_r4.0", pretrained, progress, 0.67, 0.75, version="r4.0", **kwargs)


def darknet_l_r4_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV4:
    """DarkNet release 4.0 with large channels (depth 1.0, width 1.0)."""
    return _darknet_v4_conf("darknet_l_r4.0", pretrained, progress, 1.0, 1.0, version="r4.0", **kwargs)
