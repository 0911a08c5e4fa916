"""CPU restatement of `yolov5_mobilenet_v3_small_fpn` (yolort/models/yolo_lite.py) -- TEST INFRASTRUCTURE ONLY.

Computed module by module in fp32 from a state dict, with no folding, following:
  * the MobileNetV3-Small features (torchvision models/mobilenetv3.py:252-265, the `mobilenet_v3_small` table below):
    a 3x3/s2 stem conv + BN + Hardswish, eleven InvertedResidual blocks ([1x1 expand + BN + act] -> depthwise k x k / s
    + BN + act -> [SE] -> 1x1 project + BN, [+ input when stride 1 and in == out]) and a 1x1 conv 96 -> 576 + BN +
    Hardswish;
  * FrozenBatchNorm2d (torchvision ops/misc.py:54-62): scale = w * rsqrt(rv + eps), shift = b - rm * scale, eps 1e-5;
  * SqueezeExcitation (ops/misc.py:252-261): x * hardsigmoid(fc2(relu(fc1(mean_hw(x)))));
  * FeaturePyramidNetwork (ops/feature_pyramid_network.py:180-200) with LastLevelMaxPool (:220) over the returned
    layers 4, 9 and 12 (yolo_lite.py:92-105);
  * YOLOHead and PostProcess through oracle/restate.py with strides 8, 16, 32, 64 and the P6 anchors
    (yolo_lite.py:125-131), although the maps sit at strides 16, 32, 32 and 64.
"""
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from . import restate as R

STRIDES = [8, 16, 32, 64]
ANCHORS = [[19, 27, 44, 40, 38, 94], [96, 68, 86, 152, 180, 137], [140, 301, 303, 264, 238, 542],
           [436, 615, 739, 380, 925, 792]]
BN_EPS = 1e-5
# (kernel, use_se, activation, stride) of features.1 .. features.11 (mobilenetv3.py:254-264); the widths come from the
# state dict
SMALL_BLOCKS = [(3, True, "RE", 2), (3, False, "RE", 2), (3, False, "RE", 1), (5, True, "HS", 2), (5, True, "HS", 1),
                (5, True, "HS", 1), (5, True, "HS", 1), (5, True, "HS", 1), (5, True, "HS", 2), (5, True, "HS", 1),
                (5, True, "HS", 1)]
RETURN_LAYERS = (4, 9, 12)


class NetLite:
    def __init__(self, state_dict: Dict[str, torch.Tensor]):
        self.sd = {k: v.float() for k, v in state_dict.items()}
        self.se_gates: List[torch.Tensor] = []     # every SE gate of the last backbone() call

    def bn(self, x, p: str):
        sd = self.sd
        scale = sd[f"{p}.weight"] * (sd[f"{p}.running_var"] + BN_EPS).rsqrt()
        shift = sd[f"{p}.bias"] - sd[f"{p}.running_mean"] * scale
        return x * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)

    @staticmethod
    def act(x, kind: str):
        return F.relu(x) if kind == "RE" else F.hardswish(x) if kind == "HS" else x

    def conv_bn_act(self, x, p: str, stride: int, act: str, groups: int = 1):
        w = self.sd[f"{p}.0.weight"]
        k = w.shape[-1]
        return self.act(self.bn(F.conv2d(x, w, None, stride, (k - 1) // 2, 1, groups), f"{p}.1"), act)

    def se(self, x, p: str):
        sd = self.sd
        s = x.mean((2, 3), keepdim=True)
        s = F.relu(F.conv2d(s, sd[f"{p}.fc1.weight"], sd[f"{p}.fc1.bias"]))
        g = F.hardsigmoid(F.conv2d(s, sd[f"{p}.fc2.weight"], sd[f"{p}.fc2.bias"]))
        self.se_gates.append(g.flatten(1))
        return g * x

    def block(self, x, i: int):
        k, use_se, act, stride = SMALL_BLOCKS[i - 1]
        p = f"backbone.body.{i}.block"
        j = 0
        y = x
        c_in = x.shape[1]
        if self.sd[f"{p}.0.0.weight"].shape[1] != 1:      # expand (absent when expanded == input width)
            y = self.conv_bn_act(y, f"{p}.0", 1, act)
            j = 1
        y = self.conv_bn_act(y, f"{p}.{j}", stride, act, groups=y.shape[1])
        j += 1
        if use_se:
            y = self.se(y, f"{p}.{j}")
            j += 1
        y = self.conv_bn_act(y, f"{p}.{j}", 1, "")
        if stride == 1 and c_in == y.shape[1]:
            y = y + x
        return y

    def backbone(self, x) -> List[torch.Tensor]:
        """BackboneWithFPN.forward: the FPN outputs "0", "1", "2", "pool"."""
        self.se_gates = []
        y = self.conv_bn_act(x, "backbone.body.0", 2, "HS")
        taps = []
        for i in range(1, 12):
            y = self.block(y, i)
            if i in RETURN_LAYERS:
                taps.append(y)
        y = self.conv_bn_act(y, "backbone.body.12", 1, "HS")
        taps.append(y)
        sd = self.sd

        def inner(t, i):
            return F.conv2d(t, sd[f"backbone.fpn.inner_blocks.{i}.0.weight"], sd[f"backbone.fpn.inner_blocks.{i}.0.bias"])

        def layer(t, i):
            return F.conv2d(t, sd[f"backbone.fpn.layer_blocks.{i}.0.weight"], sd[f"backbone.fpn.layer_blocks.{i}.0.bias"],
                            1, 1)

        last = inner(taps[-1], len(taps) - 1)
        results = [layer(last, len(taps) - 1)]
        for idx in range(len(taps) - 2, -1, -1):
            lat = inner(taps[idx], idx)
            last = lat + F.interpolate(last, size=lat.shape[-2:], mode="nearest")
            results.insert(0, layer(last, idx))
        results.append(F.max_pool2d(results[-1], kernel_size=1, stride=2, padding=0))
        return results

    def head(self, feats: List[torch.Tensor]) -> List[torch.Tensor]:
        outs = []
        for i, f in enumerate(feats):
            y = F.conv2d(f, self.sd[f"head.head.{i}.weight"], self.sd[f"head.head.{i}.bias"])
            n, _, h, w = y.shape
            outs.append(y.view(n, 3, -1, h, w).permute(0, 1, 3, 4, 2).contiguous())
        return outs


def postprocess(heads, score_thresh: float, nms_thresh: float = 0.45, detections_per_img: int = 300):
    return R.postprocess(heads, score_thresh, nms_thresh, detections_per_img, strides=STRIDES, anchor_grids=ANCHORS)


def detect(state_dict, batch: torch.Tensor, score_thresh: float, nms_thresh: float = 0.45,
           detections_per_img: int = 300):
    """YOLO.forward (yolort/models/yolo.py:141-183) on a batched [N,3,H,W] tensor: no letterbox, boxes on the canvas."""
    net = NetLite(state_dict)
    with torch.no_grad():
        heads = net.head(net.backbone(batch.float()))
    return postprocess(heads, score_thresh, nms_thresh, detections_per_img)


def level_shapes(heads: Sequence[torch.Tensor]):
    """(H, W, stride) per level as decode sees them."""
    return [(int(h.shape[2]), int(h.shape[3]), s) for h, s in zip(heads, STRIDES)]
