"""`from vit_tensorflow.cvt import CvT` (reference cvt.py:149) on the H100 engine."""
from vit_tensorflow_b200 import CvT  # noqa: F401

__all__ = ["CvT"]
