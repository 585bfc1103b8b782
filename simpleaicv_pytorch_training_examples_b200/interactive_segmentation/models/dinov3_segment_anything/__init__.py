"""DINOv3 SAM image encoder (SimpleAICV/interactive_segmentation/models/dinov3_segment_anything)."""
from .dinov3_image_encoder import DINOV3ViTImageEncoder  # noqa: F401
