"""`from vit_tensorflow.vit_for_small_dataset import ViT, SPT` (reference vit_for_small_dataset.py:142, 159: shifted patch tokens
and locality self-attention) on the H100 engine."""
from vit_tensorflow_b200 import SmallDatasetViT as ViT, SPT  # noqa: F401

__all__ = ["ViT", "SPT"]
