"""`from vit_tensorflow.levit import LeViT` (reference levit.py:164) on the H100 engine."""
from vit_tensorflow_b200 import LeViT  # noqa: F401

__all__ = ["LeViT"]
