"""YOLOv5 utilities of the reference (yolort/v5) on the GPU."""
