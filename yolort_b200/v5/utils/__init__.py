"""yolort/v5/utils on the GPU: augmentations."""
