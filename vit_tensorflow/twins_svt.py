"""`from vit_tensorflow.twins_svt import TwinsSVT` (reference twins_svt.py:215) on the H100 engine."""
from vit_tensorflow_b200 import TwinsSVT  # noqa: F401

__all__ = ["TwinsSVT"]
