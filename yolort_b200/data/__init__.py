"""Dataset-side tools of the reference's `yolort.data` that the inference path needs: COCO box evaluation."""
from .coco_eval import COCOEvaluator

__all__ = ["COCOEvaluator"]
