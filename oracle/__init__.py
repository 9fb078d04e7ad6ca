"""CPU oracle for the ViT-family forward path of taki0112/vit-tensorflow.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it, and only as the checker / the timed CPU
arm, never as the thing shipped.  The product path (``vit_tensorflow_b200``) never
imports this package and fails loudly when its CUDA library is missing.

PARITY: pinned on the reference's own code, unpinned only at the TensorFlow-primitive boundary.  The reference
(TensorFlow/Keras + einops, un-vendored, version ">= 2.3.0") cannot be imported as shipped in this image (no
TensorFlow), and it ships no tests / golden vectors (SURVEY.md section 8c).  ``tf_shim`` therefore provides a numpy
stand-in for the ~35 TensorFlow / Keras entry points the reference calls; over it the UNMODIFIED reference modules
(imported from /root/reference, never copied) run here, ``ref_bind`` loads the oracle's named weights into their Keras
variables by attribute path, and their logits equal ``spec_numpy``'s to 2e-15 in float64 for every model class
(tests/test_reference_shim.py; committed as tests/golden/*__refshim.npz by tests/golden/make_ref_golden.py so that the
GPU box, which has no /root/reference, can compare the CUDA engine with them).  What stays assumed is the semantics
of those primitives (Dense, LayerNormalization epsilon 1e-3, extract_patches 'SAME', ...: listed in ``tf_shim``'s
docstring and SURVEY.md Appendix A) -- checked against PyTorch's operators, confirmable only by TensorFlow itself
(``tools/ref_tf_dump.py`` is the hook).  Further anchors: (1) two independent restatements -- a numpy-float64 "spec"
(``spec_numpy``) and a torch-CPU-float32 one (``ref_torch``) -- that must agree, (2) einops itself (installed here) used
as the ground truth for the patch ``Rearrange``, (3) ``tests/test_oracle_vs_hf_vit.py``: the ViT restatement reproduces
Hugging Face's independent PyTorch ``ViTForImageClassification`` on mapped weights, (4) ``tests/test_oracle_anchors.py``:
building blocks against PyTorch operators and plain-loop restatements.
"""
from .weights import (make_config, weight_specs, init_weights, stress_weights,  # noqa: F401
                      make_image, flops_per_image, t2t_token_grid)
from .spec_numpy import forward as forward_numpy  # noqa: F401
