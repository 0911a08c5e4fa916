"""yolort_b200: the YOLOv5 inference path of zhiqwang/yolort rebuilt for H100 (sm_90a).

Python here mirrors the `yolort.models` surface; all arithmetic is in libyolort_b200.so
(yolort_b200/csrc/*.cu, C ABI in include/yolort_b200.h)."""
__version__ = "0.1.0"
