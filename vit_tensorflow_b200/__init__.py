"""vit_tensorflow_b200 -- H100-native forward engine behind the vit_tensorflow constructor/call API.

    from vit_tensorflow_b200 import ViT, DeepViT, CaiT, CrossViT

Python here is host code only (argument validation, weight dict, pointer marshalling over ctypes); the compute is
hand-written sm_90a CUDA in `libvitb200.so` (sources under `csrc/`, C-ABI in `include/vitb200.h`).
Importing the package does not load the library; constructing a model does, and fails loudly when the library
or an H100 is missing -- there is no CPU / PyTorch fallback.
"""
from .models import (ViT, DeepViT, CaiT, CrossViT, DistillableViT, ParallelViT, T2TViT, PatchMergerViT, PatchMerger,  # noqa: F401
                     EfficientViT, CCT, cct_2, cct_4, cct_6, cct_7, cct_8, cct_14, cct_16, LeViT, CvT, TwinsSVT,
                     CrossFormer, from_config, pair)

__all__ = ["ViT", "DeepViT", "CaiT", "CrossViT", "DistillableViT", "ParallelViT", "T2TViT", "PatchMergerViT", "PatchMerger",
           "EfficientViT", "CCT", "cct_2", "cct_4", "cct_6", "cct_7", "cct_8", "cct_14", "cct_16", "LeViT", "CvT", "TwinsSVT",
           "CrossFormer", "from_config"]
