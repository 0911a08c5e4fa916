"""CPU fake-quant restatement of the FP8 (e4m3) YOLOv5 plan -- TEST INFRASTRUCTURE ONLY.

Extends oracle/restate.py the way restate_ts.py does: `NetFP8` walks the MODULES of the state dict (not the engine's op
list), so a lowering mistake (a wrong scale, multiplier, weight or scale group) shows as a difference.  With an
activation calibration (`amax`: max|x| per buffer of the fp16 / bf16 plan, `Fp8Calibration.amax`) it restates the
numerics of DESIGN.md "FP8 inference" in fp32:

  * weights: the BN-folded fp64 weight, one power-of-two scale per output channel, one rounding to e4m3;
  * activations: every module output is rounded to e4m3 (nearest even, saturating at +-448) with the scale of the
    buffer the plan writes it into; concat windows share their buffer's scale, and an upsample's source and
    destination share one scale (the SPP pools run inside one concat buffer);
  * the stem keeps full-precision weights and its output is rounded with the stem buffer's scale; a Bottleneck's
    shortcut is added before its output is rounded; the heads keep unrounded outputs (the plan writes fp16 logits).

With `amax=None` nothing is rounded and every step is restate.Net's own arithmetic: the result equals restate.Net
bit for bit, which ties this walk to the fixtures pinned against the reference.
"""
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import restate as R

E4M3_MAX = 448.0


def e4m3_scale(amax: float) -> float:
    """The smallest power of two s with amax / s <= 448 (1 for zero)."""
    if not amax > 0:
        return 1.0
    s = 1.0
    while amax / s > E4M3_MAX:
        s *= 2.0
    while amax / (0.5 * s) <= E4M3_MAX:
        s *= 0.5
    return s


def e4m3_round(x: torch.Tensor) -> torch.Tensor:
    """Nearest e4m3 value of x (ties to even), saturating at +-448; exact arithmetic in x's dtype.  The spacing in the
    binade [2^(e-1), 2^e) is 2^(e-4), and 2^-9 for the subnormals."""
    _, e = torch.frexp(x)
    q = torch.ldexp(torch.ones_like(x), torch.clamp(e - 4, min=-9))
    return torch.clamp(torch.round(x / q) * q, -E4M3_MAX, E4M3_MAX)


def quantize_weight(w: torch.Tensor) -> torch.Tensor:
    """fp64 [Co, ...] -> its e4m3 values times their per-output-channel scales, as fp32."""
    amax = w.abs().flatten(1).amax(1).tolist()
    s = torch.tensor([e4m3_scale(a) for a in amax], dtype=torch.float64).view(-1, *([1] * (w.dim() - 1)))
    return (e4m3_round(w / s) * s).float()


class NetFP8(R.Net):
    def __init__(self, state_dict: Dict[str, torch.Tensor], amax: Optional[Dict[str, float]] = None):
        super().__init__(state_dict)
        self.amax = amax
        nl = 4 if self.has("backbone.pan.intermediate_blocks.p6") else 3
        taps = (4, 6, 8)
        # the plan's concat buffers (engine.lower_yolo): cat_dn[l] = [up(lateral) | body tap], cat_up[l] = [down | lateral]
        self.cat_dn = {l: f"pan.cat{nl - 1 - l}[up(lat{nl - 1 - l})|f{taps[l]}]" for l in range(nl - 1)}
        self.cat_up = {l: f"pan.cat_p{l + 3}[down(p{l + 2})|lat{nl - l}]" for l in range(1, nl)}
        self.taps = {taps[l]: self.cat_dn[l] for l in range(min(nl - 1, 3))}
        # an upsample copies the lateral window of cat_up[l] into cat_dn[l - 1]: one scale for both buffers
        self.partner = {}
        for l in range(1, nl):
            self.partner[self.cat_up[l]] = self.cat_dn[l - 1]
            self.partner[self.cat_dn[l - 1]] = self.cat_up[l]

    # -- rounding ------------------------------------------------------------------------------------------------
    def scale(self, buf: str) -> float:
        names = [buf] + ([self.partner[buf]] if buf in self.partner else [])
        return e4m3_scale(max(self.amax[n] for n in names))

    def q(self, t: torch.Tensor, buf: str) -> torch.Tensor:
        """t rounded to e4m3 with the scale of plan buffer `buf` (identity without a calibration)."""
        if self.amax is None:
            return t
        s = self.scale(buf)
        return e4m3_round(t / s) * s

    def _geometry(self, p: str, k: int):
        stride, pad = 1, k // 2
        if k == 3 and p in self.stride2:
            stride = 2
        return stride, pad

    def fold(self, p: str, lo: int = 0, hi: Optional[int] = None, bn: Optional[str] = None):
        """BN-folded fp64 weight and bias of module p (channels [lo, hi) of BatchNorm `bn`, default p's own)."""
        w = self.sd[f"{p}.conv.weight" if bn is None else f"{p}.weight"].double()
        b_ = f"{p}.bn" if bn is None else bn
        hi = w.shape[0] + lo if hi is None else hi
        scale = self.sd[f"{b_}.weight"].double()[lo:hi] / torch.sqrt(self.sd[f"{b_}.running_var"].double()[lo:hi] + R.BN_EPS)
        shift = self.sd[f"{b_}.bias"].double()[lo:hi] - self.sd[f"{b_}.running_mean"].double()[lo:hi] * scale
        return w * scale.view(-1, 1, 1, 1), shift

    def conv_pre(self, x, p: str):
        """A Conv module's activation output before rounding: e4m3 folded weights (restate.Net.conv without a
        calibration)."""
        if self.amax is None:
            return self.conv(x, p)
        w, b = self.fold(p)
        stride, pad = self._geometry(p, w.shape[-1])
        return self.act(F.conv2d(x, quantize_weight(w), b.float(), stride, pad))

    def cq(self, x, p: str, buf: str):
        return self.q(self.conv_pre(x, p), buf)

    # -- blocks: they return the unrounded output, the caller rounds it into its destination -------------------
    def c3(self, x, p: str, shortcut: bool):
        if f"{p}.cv4.conv.weight" in self.sd:
            return self.csp(x, p, shortcut)
        n = p[len("backbone."):]
        y = self.cq(x, f"{p}.cv1", f"{n}.cat")
        i = 0
        while self.has(f"{p}.m.{i}"):
            last = not self.has(f"{p}.m.{i + 1}")
            z = self.conv_pre(self.cq(y, f"{p}.m.{i}.cv1", f"{n}.m{i}.t"), f"{p}.m.{i}.cv2")
            y = self.q(y + z if shortcut else z, f"{n}.cat" if last else f"{n}.m{i}.y")
            i += 1
        return self.conv_pre(torch.cat((y, self.cq(x, f"{p}.cv2", f"{n}.cat")), 1), f"{p}.cv3")

    def csp(self, x, p: str, shortcut: bool):
        n = p[len("backbone."):]
        y = self.cq(x, f"{p}.cv1", f"{n}.y")
        i = 0
        while self.has(f"{p}.m.{i}"):
            z = self.conv_pre(self.cq(y, f"{p}.m.{i}.cv1", f"{n}.m{i}.t"), f"{p}.m.{i}.cv2")
            y = self.q(y + z if shortcut else z, f"{n}.m{i}.y")
            i += 1
        if self.amax is None:
            y1 = F.conv2d(y, self.sd[f"{p}.cv3.weight"])
            y2 = F.conv2d(x, self.sd[f"{p}.cv2.weight"])
            t = F.batch_norm(torch.cat((y1, y2), 1), self.sd[f"{p}.bn.running_mean"], self.sd[f"{p}.bn.running_var"],
                             self.sd[f"{p}.bn.weight"], self.sd[f"{p}.bn.bias"], False, 0.0, R.BN_EPS)
            t = F.leaky_relu(t, 0.1)
        else:   # the concat's BatchNorm is per channel: its halves fold into cv3 and cv2
            c_ = self.sd[f"{p}.cv3.weight"].shape[0]
            w3, b3 = self.fold(f"{p}.cv3", 0, c_, bn=f"{p}.bn")
            w2, b2 = self.fold(f"{p}.cv2", c_, 2 * c_, bn=f"{p}.bn")
            y1 = F.leaky_relu(F.conv2d(y, quantize_weight(w3), b3.float()), 0.1)
            y2 = F.leaky_relu(F.conv2d(x, quantize_weight(w2), b2.float()), 0.1)
            t = self.q(torch.cat((y1, y2), 1), f"{n}.cat")
        return self.conv_pre(t, f"{p}.cv4")

    def spp(self, x, p: str):
        n = p[len("backbone."):]
        x = self.cq(x, f"{p}.cv1", f"{n}.cat")
        return self.conv_pre(torch.cat([x] + [F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)], 1), f"{p}.cv2")

    def backbone(self, x) -> List[torch.Tensor]:
        """restate.Net.backbone with every module output rounded into its plan buffer."""
        b = "backbone.body"
        feats = []
        for i in range(9):
            if i == 0 and self.focus:
                x = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)
                x = self.q(self.conv(x, f"{b}.0.conv"), "body.0")
            elif i == 0:
                x = self.q(self.conv(x, f"{b}.0"), "body.0")
            elif i == 8 and self.focus:
                x = self.q(self.spp(x, f"{b}.8"), "body.8")
            elif i in (1, 3, 5, 7):
                x = self.cq(x, f"{b}.{i}", f"body.{i}")
            else:
                x = self.q(self.c3(x, f"{b}.{i}", True), self.taps.get(i, f"body.{i}"))
            if i in (4, 6, 8):
                feats.append(x)
        x = feats
        inner, layer = "backbone.pan.inner_blocks", "backbone.pan.layer_blocks"
        p6 = "backbone.pan.intermediate_blocks.p6"
        if self.has(p6):
            x.append(self.q(self.c3(self.cq(x[-1], f"{p6}.0", "pan.p6.conv"), f"{p6}.1", True), "pan.p6.c3"))
        up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")
        nf = len(x)
        inners = []
        last = x[-1]
        for idx in range(nf - 1):
            l = nf - 1 - idx
            if idx == 0 and not self.focus:
                last = self.q(self.spp(last, f"{inner}.0"), "pan.spp")
            elif idx == 0:
                last = self.q(self.c3(last, f"{inner}.0", False), "pan.spp")
            else:
                last = self.q(self.c3(last, f"{inner}.{3 * idx}", False), f"pan.u{idx}")
            last = self.cq(last, f"{inner}.{3 * idx + 1}", self.cat_up[l])
            inners.insert(0, last)
            last = torch.cat([up(last), x[nf - idx - 2]], 1)
        inners.insert(0, last)
        last = self.q(self.c3(inners[0], f"{layer}.0", False), "pan.p3")
        results = [last]
        for idx in range(nf - 1):
            last = self.cq(last, f"{layer}.{2 * idx + 1}", self.cat_up[idx + 1])
            last = self.q(self.c3(torch.cat([last, inners[idx + 1]], 1), f"{layer}.{2 * idx + 2}", False),
                          f"pan.p{idx + 4}")
            results.append(last)
        return results

    def head(self, feats: List[torch.Tensor], num_anchors: int = 3) -> List[torch.Tensor]:
        """restate.Net.head with e4m3 weights (per output channel); the logits are not rounded."""
        if self.amax is None:
            return super().head(feats, num_anchors)
        outs = []
        for i, f in enumerate(feats):
            w = quantize_weight(self.sd[f"head.head.{i}.weight"].double())
            y = F.conv2d(f, w, self.sd[f"head.head.{i}.bias"])
            n, _, h, w_ = y.shape
            outs.append(y.view(n, num_anchors, -1, h, w_).permute(0, 1, 3, 4, 2).contiguous())
        return outs


def detect(state_dict, amax: Optional[Dict[str, float]], images: Sequence[torch.Tensor], score_thresh: float = 0.005,
           nms_thresh: float = 0.45, detections_per_img: int = 300, size=(640, 640), size_divisible: int = 32):
    """restate.detect (YOLOv5.forward, yolov5.py:135-189) with the fake-quant network."""
    batch, _, _ = R.letterbox(images, float(size[0]), float(size[1]), size_divisible)
    net = NetFP8(state_dict, amax)
    with torch.no_grad():
        heads = net.head(net.backbone(batch))
    dets = R.postprocess(heads, score_thresh, nms_thresh, detections_per_img)
    Hb, Wb = int(batch.shape[2]), int(batch.shape[3])
    for d, im in zip(dets, images):
        d["boxes"] = R.scale_coords(d["boxes"], Hb, Wb, int(im.shape[-2]), int(im.shape[-1]))
    return dets
