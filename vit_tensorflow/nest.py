"""`from vit_tensorflow.nest import NesT` (reference nest.py:150) on the H100 engine."""
from vit_tensorflow_b200 import NesT  # noqa: F401

__all__ = ["NesT"]
