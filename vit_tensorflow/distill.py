"""`from vit_tensorflow.distill import DistillableViT` (reference distill.py:47) -- forward path only, on the H100 engine."""
from vit_tensorflow_b200 import DistillableViT  # noqa: F401
