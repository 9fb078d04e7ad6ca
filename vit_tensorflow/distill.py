"""`from vit_tensorflow.distill import DistillableViT, DistillableT2TViT, DistillableEfficientViT` (reference distill.py:47, :61,
:74) -- forward path only, on the H100 engine."""
from vit_tensorflow_b200 import DistillableEfficientViT, DistillableT2TViT, DistillableViT  # noqa: F401
