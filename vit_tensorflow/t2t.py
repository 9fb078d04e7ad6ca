"""`from vit_tensorflow.t2t import T2TViT` (reference t2t.py:50) on the H100 engine."""
from vit_tensorflow_b200 import T2TViT  # noqa: F401
