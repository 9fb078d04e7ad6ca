"""`from vit_tensorflow.regionvit import RegionViT` (reference regionvit.py:184) on the H100 engine."""
from vit_tensorflow_b200 import RegionViT  # noqa: F401

__all__ = ["RegionViT"]
