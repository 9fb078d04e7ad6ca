"""`from vit_tensorflow.mae import MAE` (reference mae.py:17, masked autoencoder) on the H100 engine; the encoder is a
`vit_tensorflow_b200.ViT`."""
from vit_tensorflow_b200 import MAE  # noqa: F401

__all__ = ["MAE"]
