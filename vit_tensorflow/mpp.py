"""`from vit_tensorflow.mpp import MPP` (reference mpp.py:133, masked patch prediction) on the H100 engine; the transformer is a
`vit_tensorflow_b200.ViT`."""
from vit_tensorflow_b200 import MPP  # noqa: F401

__all__ = ["MPP"]
