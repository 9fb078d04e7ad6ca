"""`from vit_tensorflow.vit_with_patch_merger import ViT, PatchMerger` (reference vit_with_patch_merger.py:42,134) on the H100 engine."""
from vit_tensorflow_b200 import PatchMergerViT as ViT, PatchMerger  # noqa: F401
