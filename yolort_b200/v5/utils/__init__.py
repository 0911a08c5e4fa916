"""yolort/v5/utils on the GPU: augmentations and the mosaic training loader (datasets)."""
