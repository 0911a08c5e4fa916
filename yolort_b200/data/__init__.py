"""Dataset-side tools of the reference's `yolort.data`: COCO box evaluation and the training augmentations."""
from . import transforms
from .coco_eval import COCOEvaluator

__all__ = ["COCOEvaluator", "transforms"]
