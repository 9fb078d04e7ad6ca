"""`from vit_tensorflow.pit import PiT` (reference pit.py:158: the overlapping patch embedding and per-stage attention heads, run as
the reference runs it, with no pooling stage) on the H100 engine."""
from vit_tensorflow_b200 import PiT  # noqa: F401

__all__ = ["PiT"]
