"""`from vit_tensorflow.scalable_vit import ScalableViT` (reference scalable_vit.py:250: scalable self-attention and interactive
windowed self-attention) on the H100 engine."""
from vit_tensorflow_b200 import ScalableViT  # noqa: F401

__all__ = ["ScalableViT"]
