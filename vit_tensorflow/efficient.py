"""`from vit_tensorflow.efficient import ViT` (reference efficient.py:12) on the H100 engine."""
from vit_tensorflow_b200 import EfficientViT as ViT  # noqa: F401
