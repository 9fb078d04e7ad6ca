"""`from vit_tensorflow.parallel_vit import ViT` (reference parallel_vit.py:120) on the H100 engine."""
from vit_tensorflow_b200 import ParallelViT as ViT  # noqa: F401
