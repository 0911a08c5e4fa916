"""CSPDarknet (r6.0): the detection body and the DarkNetV6 image classifier.

Layout and channel rules follow the reference (yolort/models/darknetv6.py:31-200): a 6x6/s2 stem followed by four
[3x3/s2 Conv, C3] stages; module indices 0..8 are what the PAN taps (4, 6, 8) and what the state-dict keys are built
from.  The classifier adds `avgpool` and `classifier` (Linear -> Hardswish -> Dropout -> Linear) and runs on the
native plan (models/_classifier.py).
"""
from typing import Any, Callable, List, Optional

from torch import nn

from ._classifier import DarkNetClassifier, PlanAvgPool, PlanFeatures, build_head, init_like_reference, pretrained_check
from ._utils import depth_gain, make_divisible
from .common import C3, Conv

__all__ = [
    "DarkNetV6",
    "darknet_n_r6_0",
    "darknet_s_r6_0",
    "darknet_m_r6_0",
    "darknet_l_r6_0",
    "darknet_x_r6_0",
]

model_urls = {
    "darknet_n_r6.0": None,
    "darknet_s_r6.0": None,
    "darknet_m_r6.0": None,
    "darknet_l_r6.0": None,
    "darknet_x_r6.0": None,
}


def darknet_v6_features(depth_multiple: float, width_multiple: float, last_channel: int = 1024,
                        block: Optional[Callable[..., nn.Module]] = None, stages_repeats: Optional[List[int]] = None,
                        stages_out_channels: Optional[List[int]] = None, round_nearest: int = 8) -> nn.Sequential:
    block = C3 if block is None else block
    stages_repeats = [3, 6, 9] if stages_repeats is None else stages_repeats
    stages_out_channels = [128, 256, 512] if stages_out_channels is None else stages_out_channels
    c_in = make_divisible(64 * width_multiple, round_nearest)
    layers: List[nn.Module] = [Conv(3, c_in, k=6, s=2, p=2)]
    for n, c in zip(stages_repeats, stages_out_channels):
        c_out = make_divisible(c * width_multiple, round_nearest)
        layers.append(Conv(c_in, c_out, k=3, s=2))
        layers.append(block(c_out, c_out, n=depth_gain(n, depth_multiple)))
        c_in = c_out
    last = make_divisible(last_channel * width_multiple, round_nearest)
    layers.append(Conv(c_in, last, k=3, s=2))
    layers.append(block(last, last, n=depth_gain(3, depth_multiple)))
    return nn.Sequential(*layers)


class DarkNetV6(DarkNetClassifier):
    """
    DarkNetV6 main class.

    Args:
        depth_multiple (float): Depth multiplier
        width_multiple (float): Width multiplier - adjusts number of channels in each layer by this amount
        version (str): Module version released by ultralytics, set to r4.0.
        block: Module specifying the building block of the stages (C3 by default; the plan lowers C3 and
            BottleneckCSP)
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
        assert version == "r4.0", "Currently the module version used in DarkNetV6 is r4.0."
        self.features = PlanFeatures(*darknet_v6_features(depth_multiple, width_multiple, last_channel, block,
                                                          stages_repeats, stages_out_channels, round_nearest))
        last = make_divisible(last_channel * width_multiple, round_nearest)
        self.avgpool = PlanAvgPool()
        self.classifier = build_head(last, num_classes)
        init_like_reference(self)
        self._attach()


def _darknet_v6_conf(arch: str, pretrained: bool, progress: bool, *args: Any, **kwargs: Any) -> DarkNetV6:
    pretrained_check(arch, pretrained, model_urls)
    return DarkNetV6(*args, **kwargs)


def darknet_n_r6_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV6:
    """DarkNet release 6.0 with nano channels (depth 0.33, width 0.25).  `pretrained=True` raises
    NotImplementedError: no weights exist."""
    return _darknet_v6_conf("darknet_n_r6.0", pretrained, progress, 0.33, 0.25, **kwargs)


def darknet_s_r6_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV6:
    """DarkNet release 6.0 with small channels (depth 0.33, width 0.5)."""
    return _darknet_v6_conf("darknet_s_r6.0", pretrained, progress, 0.33, 0.5, **kwargs)


def darknet_m_r6_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV6:
    """DarkNet release 6.0 with medium channels (depth 0.67, width 0.75)."""
    return _darknet_v6_conf("darknet_m_r6.0", pretrained, progress, 0.67, 0.75, **kwargs)


def darknet_l_r6_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV6:
    """DarkNet release 6.0 with large channels (depth 1.0, width 1.0)."""
    return _darknet_v6_conf("darknet_l_r6.0", pretrained, progress, 1.0, 1.0, **kwargs)


def darknet_x_r6_0(pretrained: bool = False, progress: bool = True, **kwargs: Any) -> DarkNetV6:
    """DarkNet release 6.0 with extra-large channels (depth 1.33, width 1.25)."""
    return _darknet_v6_conf("darknet_x_r6.0", pretrained, progress, 1.33, 1.25, **kwargs)
