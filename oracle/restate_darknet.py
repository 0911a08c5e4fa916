"""CPU restatement of the DarkNet classifiers (yolort/models/darknetv4.py:33-136, darknetv6.py:31-127) -- TEST
INFRASTRUCTURE ONLY.

`features` reuses oracle/restate.py's Net (conv, c3 / csp, spp: the same fp32 torch CPU operators as the reference)
on the `features.` prefix; then AdaptiveAvgPool2d(1) as an fp32 mean over H x W, and the classifier Linear ->
Hardswish -> (Dropout: identity in eval) -> Linear in fp32."""
from typing import Dict, List

import torch
import torch.nn.functional as F

from . import restate as R


class NetDarknet(R.Net):
    # stride-2 3x3 convolutions: every odd module of the features (darknetv4.py:92,98, darknetv6.py:88,94)
    stride2 = {f"features.{i}" for i in range(1, 64, 2)}

    def __init__(self, state_dict: Dict[str, torch.Tensor]):
        self.sd = {k: v.detach().float().cpu() for k, v in state_dict.items()}
        self.focus = "features.0.conv.conv.weight" in self.sd
        self.r31 = "features.2.cv4.conv.weight" in self.sd
        self.n_features = 1 + max(int(k.split(".")[1]) for k in self.sd if k.startswith("features."))

    def features(self, x) -> torch.Tensor:
        """features (darknetv4.py:84-101 / darknetv6.py:80-98): stem, [Conv, block] stages, Conv, SPP (V4) or block
        (V6)."""
        p = "features"
        for i in range(self.n_features):
            if i == 0 and self.focus:      # Focus.forward (common.py:230-240): parity order (0,0),(1,0),(0,1),(1,1)
                x = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)
                x = self.conv(x, f"{p}.0.conv")
            elif i == self.n_features - 1 and self.focus:
                x = self.spp(x, f"{p}.{i}")
            elif i % 2 == 1 or i == 0:
                x = self.conv(x, f"{p}.{i}")
            else:
                x = self.c3(x, f"{p}.{i}", True)
        return x

    def avgpool(self, f) -> torch.Tensor:
        return f.mean((2, 3))

    def classifier(self, v) -> torch.Tensor:
        sd = self.sd
        h = F.hardswish(F.linear(v, sd["classifier.0.weight"], sd["classifier.0.bias"]))
        return F.linear(h, sd["classifier.3.weight"], sd["classifier.3.bias"])

    def forward(self, x) -> List[torch.Tensor]:
        """(final features [N,C,h,w], logits [N,num_classes]), fp32."""
        f = self.features(x.float())
        return f, self.classifier(self.avgpool(f))
