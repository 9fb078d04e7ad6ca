"""`from vit_tensorflow.simmim import SimMIM` (reference simmim.py:72, simple masked image modelling) on the H100 engine; the
encoder is a `vit_tensorflow_b200.ViT`."""
from vit_tensorflow_b200 import SimMIM  # noqa: F401

__all__ = ["SimMIM"]
