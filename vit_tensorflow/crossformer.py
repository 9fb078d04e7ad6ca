"""`from vit_tensorflow.crossformer import CrossFormer` (reference crossformer.py:205) on the H100 engine."""
from vit_tensorflow_b200 import CrossFormer  # noqa: F401

__all__ = ["CrossFormer"]
