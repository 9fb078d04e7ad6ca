"""`from vit_tensorflow.mobile_vit import MobileViT` (reference mobile_vit.py:209: MobileNetV2 blocks and MobileViT blocks) on the
H100 engine."""
from vit_tensorflow_b200 import MobileViT  # noqa: F401

__all__ = ["MobileViT"]
