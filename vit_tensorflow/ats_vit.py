"""`from vit_tensorflow.ats_vit import ViT` (reference ats_vit.py:260, adaptive token sampling) on the H100 engine."""
from vit_tensorflow_b200 import ATSViT as ViT  # noqa: F401

__all__ = ["ViT"]
