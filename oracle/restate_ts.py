"""CPU restatement of `yolov5ts` (r4.0 with the C3TR transformer neck) -- TEST INFRASTRUCTURE ONLY.

Extends oracle/restate.py: `NetTS` is `restate.Net` whose C3 restatement becomes C3TR
(yolort/v5/models/common.py:360-367) wherever a block carries transformer parameters (`{p}.m.tr.0.q.weight`).
The transformer block is restated module by module in fp32, with no folding, following common.py:328-357 and
torch's nn.MultiheadAttention math.
"""
import math
from typing import Sequence

import torch
import torch.nn.functional as F

from . import restate as R


class NetTS(R.Net):
    def c3(self, x, p: str, shortcut: bool):
        if f"{p}.m.tr.0.q.weight" not in self.sd:
            return super().c3(x, p, shortcut)
        # C3TR.forward = C3.forward (common.py:172-173) with m = TransformerBlock
        y = self.transformer(self.conv(x, f"{p}.cv1"), f"{p}.m")
        return self.conv(torch.cat((y, self.conv(x, f"{p}.cv2")), 1), f"{p}.cv3")

    def transformer(self, x, p: str, num_heads: int = 4):
        """TransformerBlock.forward (common.py:352-357, conv is None since c1 == c2) and TransformerLayer.forward
        (:328-331); nn.MultiheadAttention (batch_first=False, eval: no dropout) restated as torch computes it:
        in-projection with bias, per-head softmax(q k^T / sqrt(d)) v, out_proj."""
        sd = self.sd
        b, c, h, w = x.shape
        t = x.flatten(2).unsqueeze(0).transpose(0, 3).squeeze(3)          # [L, N, E], token y*W + x
        t = t + F.linear(t, sd[f"{p}.linear.weight"], sd[f"{p}.linear.bias"])
        self.attention = []
        i = 0
        while self.has(f"{p}.tr.{i}"):
            q_ = f"{p}.tr.{i}"
            q = F.linear(t, sd[f"{q_}.q.weight"])
            k = F.linear(t, sd[f"{q_}.k.weight"])
            v = F.linear(t, sd[f"{q_}.v.weight"])
            w_in, b_in = sd[f"{q_}.ma.in_proj_weight"], sd[f"{q_}.ma.in_proj_bias"]
            q = F.linear(q, w_in[:c], b_in[:c])
            k = F.linear(k, w_in[c:2 * c], b_in[c:2 * c])
            v = F.linear(v, w_in[2 * c:], b_in[2 * c:])
            L, N, _ = q.shape
            d = c // num_heads

            def heads(z):
                return z.reshape(L, N * num_heads, d).transpose(0, 1)    # [N*heads, L, d]

            a = torch.softmax(torch.bmm(heads(q) * (1.0 / math.sqrt(d)), heads(k).transpose(1, 2)), dim=-1)
            self.attention.append(a)                                        # [N*heads, L, L] (tests inspect it)
            o = torch.bmm(a, heads(v)).transpose(0, 1).reshape(L, N, c)
            t = F.linear(o, sd[f"{q_}.ma.out_proj.weight"], sd[f"{q_}.ma.out_proj.bias"]) + t
            t = F.linear(F.linear(t, sd[f"{q_}.fc1.weight"]), sd[f"{q_}.fc2.weight"]) + t
            i += 1
        return t.unsqueeze(3).transpose(0, 3).reshape(b, c, h, w)


def detect(state_dict, images: Sequence[torch.Tensor], score_thresh: float = 0.005, nms_thresh: float = 0.45,
           detections_per_img: int = 300, size=(640, 640), size_divisible: int = 32):
    """restate.detect (YOLOv5.forward, yolov5.py:135-189) with the yolov5ts network."""
    batch, _, _ = R.letterbox(images, float(size[0]), float(size[1]), size_divisible)
    net = NetTS(state_dict)
    with torch.no_grad():
        heads = net.head(net.backbone(batch))
    dets = R.postprocess(heads, score_thresh, nms_thresh, detections_per_img)
    Hb, Wb = int(batch.shape[2]), int(batch.shape[3])
    for d, im in zip(dets, images):
        d["boxes"] = R.scale_coords(d["boxes"], Hb, Wb, int(im.shape[-2]), int(im.shape[-1]))
    return dets
