"""`from vit_tensorflow.cct import CCT` (reference cct.py:307) and the cct_2 ... cct_16 factories (:16-48) on the H100 engine."""
from vit_tensorflow_b200 import CCT, cct_2, cct_4, cct_6, cct_7, cct_8, cct_14, cct_16  # noqa: F401

__all__ = ['cct_2', 'cct_4', 'cct_6', 'cct_7', 'cct_8', 'cct_14', 'cct_16']
