"""yolort/v5/utils on the GPU: augmentations, the mosaic training and rect validation loaders (datasets), AutoAnchor
(autoanchor), val.py's box helpers (general) and the validation metrics (metrics: ap_per_class, ConfusionMatrix, val.py's
process_batch and DetectionMetrics)."""
