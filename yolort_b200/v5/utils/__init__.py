"""yolort/v5/utils on the GPU: augmentations, the mosaic training loader (datasets) and AutoAnchor (autoanchor)."""
