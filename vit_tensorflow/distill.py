"""`from vit_tensorflow.distill import DistillableViT, DistillableT2TViT, DistillableEfficientViT, DistillWrapper` (reference
distill.py:47, :61, :74, :87) on the H100 engine; DistillWrapper takes any teacher callable."""
from vit_tensorflow_b200 import DistillableEfficientViT, DistillableT2TViT, DistillableViT, DistillWrapper  # noqa: F401
