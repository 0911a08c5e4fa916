"""Building blocks of the r6.0 / r4.0 / r3.1 YOLOv5 graphs as *parameter containers*.

These modules reproduce the parameter/buffer names of the reference blocks
(yolort/v5/models/common.py:42-73 Conv, :94-116 Bottleneck, :119-146 BottleneckCSP, :149-173 C3, :176-187 SPP,
:210-234 Focus) so that a
reference `state_dict` loads unchanged.  They do not compute: the arithmetic of the whole
backbone is executed by the sm_90a execution plan (yolort_b200/engine.py -> libyolort_b200.so).
Calling `forward` on a block is an error by design -- there is no PyTorch/CPU fallback.
"""
from torch import nn

BN_EPS = 1e-3  # set by the reference constructors (darknetv6.py:107-114, path_aggregation_network.py:158-165)
BN_MOMENTUM = 0.03


class _PlanOnly(nn.Module):
    def forward(self, *args, **kwargs):  # pragma: no cover - guard
        raise RuntimeError(
            f"{type(self).__name__} is executed by the sm_90a plan (yolort_b200.engine); "
            "it has no eager PyTorch forward."
        )


def _act(version: str) -> nn.Module:
    """common.py:61-66: module version "r4.0" (also used by r6.0 graphs) -> SiLU, "r3.1" -> Hardswish."""
    if version == "r4.0":
        return nn.SiLU()
    if version == "r3.1":
        return nn.Hardswish()
    raise NotImplementedError(f"Currently doesn't support version {version}.")


class Conv(_PlanOnly):
    """conv(k, s, autopad, bias=False) -> BatchNorm(eps=1e-3) -> SiLU (r4.0/r6.0) or Hardswish (r3.1)."""

    def __init__(self, c1: int, c2: int, k: int = 1, s: int = 1, p=None, version: str = "r4.0"):
        super().__init__()
        pad = k // 2 if p is None else p
        self.conv = nn.Conv2d(c1, c2, k, s, pad, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=BN_EPS, momentum=BN_MOMENTUM)
        self.act = _act(version)


class Bottleneck(_PlanOnly):
    """x (+) cv2_3x3(cv1_1x1(x)); the add exists only when shortcut and c1 == c2."""

    def __init__(self, c1: int, c2: int, shortcut: bool = True, e: float = 0.5, version: str = "r4.0"):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1, version=version)
        self.cv2 = Conv(c_, c2, 3, 1, version=version)
        self.add = bool(shortcut and c1 == c2)


class BottleneckCSP(_PlanOnly):
    """r3.1 block (common.py:119-146): cv4(LeakyReLU0.1(BN(cat(cv3(m(cv1(x))), cv2(x))))); cv2/cv3 are bare
    convolutions, cv1/cv4 and the bottlenecks are Conv+BN+Hardswish."""

    def __init__(self, c1: int, c2: int, n: int = 1, shortcut: bool = True, e: float = 0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1, version="r3.1")
        self.cv2 = nn.Conv2d(c1, c_, 1, 1, bias=False)
        self.cv3 = nn.Conv2d(c_, c_, 1, 1, bias=False)
        self.cv4 = Conv(2 * c_, c2, 1, 1, version="r3.1")
        self.bn = nn.BatchNorm2d(2 * c_, eps=BN_EPS, momentum=BN_MOMENTUM)
        self.act = nn.LeakyReLU(0.1, inplace=True)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, e=1.0, version="r3.1") for _ in range(n)])


class C3(_PlanOnly):
    """cv3(cat(m(cv1(x)), cv2(x))) with n bottlenecks of expansion 1.0 at width c2/2."""

    def __init__(self, c1: int, c2: int, n: int = 1, shortcut: bool = True, e: float = 0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, e=1.0) for _ in range(n)])


class SPP(_PlanOnly):
    """cv2(cat(x', mp5(x'), mp9(x'), mp13(x'))) with x' = cv1(x); pools are stride 1, -inf padded."""

    def __init__(self, c1: int, c2: int, k=(5, 9, 13), version: str = "r4.0"):
        super().__init__()
        c_ = c1 // 2
        self.k = tuple(k)
        self.cv1 = Conv(c1, c_, 1, 1, version=version)
        self.cv2 = Conv(c_ * (len(k) + 1), c2, 1, 1, version=version)
        self.m = nn.ModuleList([nn.MaxPool2d(kernel_size=x, stride=1, padding=x // 2) for x in k])


class Focus(_PlanOnly):
    """r3.1/r4.0 stem (common.py:210-234): 2x2 space-to-depth in the order [(0,0), (1,0), (0,1), (1,1)] of
    (row, col) parity, then Conv(4*c1, c2, k)."""

    def __init__(self, c1: int, c2: int, k: int = 1, s: int = 1, p=None, version: str = "r4.0"):
        super().__init__()
        self.conv = Conv(c1 * 4, c2, k, s, p, version=version)
