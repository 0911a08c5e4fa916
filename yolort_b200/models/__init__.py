"""Model constructors with the reference's names and kwargs (yolort/models/__init__.py:24-185, `yolov5ts` at
:169-185), plus
`yolov5x`, which the reference defines as an architecture (yolo.py:592-619) but does not export."""
from typing import Any

from .yolo import YOLO
from .yolov5 import YOLOv5

__all__ = ["YOLO", "YOLOv5", "yolov5n", "yolov5s", "yolov5m", "yolov5l", "yolov5x", "yolov5n6", "yolov5s6", "yolov5m6",
           "yolov5ts"]


def _make(size: str, p6: bool = False):
    def ctor(upstream_version: str = "r6.0", export_friendly: bool = False, **kwargs: Any) -> YOLOv5:
        """Args:
            upstream_version (str): ultralytics release: "r6.0" (default), and "r4.0" / "r3.1" for s, m, l.
            export_friendly (bool): accepted for signature compatibility; there is no export path here
                (SiLU is evaluated inside the conv epilogue either way).
        """
        # models/__init__.py:24-110: s/m/l exist for r3.1, r4.0 and r6.0; n, x and the P6 variants only for r6.0
        allowed = ("r3.1", "r4.0", "r6.0") if (size in "sml" and not p6) else ("r6.0",)
        if upstream_version not in allowed:
            raise NotImplementedError(f"yolov5{size}{'6' if p6 else ''} supports upstream versions {allowed}")
        if upstream_version != "r6.0":
            return YOLOv5(arch=f"yolov5_darknet_pan_{size}_{upstream_version.replace('.', '')}", **kwargs)
        if p6:   # models/__init__.py:112-166: the P6 constructors letterbox to multiples of 64
            return YOLOv5(arch=f"yolov5_darknet_pan_{size}6_r60", size_divisible=64, **kwargs)
        return YOLOv5(arch=f"yolov5_darknet_pan_{size}_r60", **kwargs)

    ctor.__name__ = f"yolov5{size}" + ("6" if p6 else "")
    return ctor


yolov5n = _make("n")
yolov5s = _make("s")
yolov5m = _make("m")
yolov5l = _make("l")
yolov5x = _make("x")
yolov5n6 = _make("n", p6=True)
yolov5s6 = _make("s", p6=True)
yolov5m6 = _make("m", p6=True)


def yolov5ts(upstream_version: str = "r4.0", export_friendly: bool = False, **kwargs: Any) -> YOLOv5:
    """yolov5s r4.0 with a transformer block in the neck (models/__init__.py:169-185).

    Args:
        upstream_version (str): "r4.0", the only release the reference builds it for.
        export_friendly (bool): accepted for signature compatibility; there is no export path here.
    """
    if upstream_version != "r4.0":
        raise NotImplementedError("Currently only supports r4.0 versions")
    return YOLOv5(arch="yolov5_darknet_tan_s_r40", **kwargs)
