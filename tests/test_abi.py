"""CPU tests of the boundary: the C-ABI library builds for sm_90a, loads, exports every symbol
include/vitb200.h declares, refuses to compute without a GPU, and the Python host classes validate kwargs with
the reference's assertion messages (vit.py:136,139; deepvit.py:117; cait.py:160; cross_vit.py:207)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    return sorted(set(re.findall(r"VB_API[^;(]*?\b(vb_\w+)\s*\(", src)))


def test_header_symbols_are_exported_and_bound_at_abi_7(lib):
    from vit_tensorflow_b200 import _lib
    declared = _declared_symbols()
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/vitb200.h but not exported"
    assert sorted(_lib.SIGNATURES) == declared, "ctypes SIGNATURES must cover exactly the declared ABI"
    # ABI 5 added vb_op_gemm / vb_op_attention_ex / vb_op_softmax_rows, ABI 6 vb_graph_stats, ABI 7 vb_last_attention_path:
    # header, library and ctypes binding agree on the version
    header = int(re.search(r"#define VB_ABI_VERSION (\d+)", open(os.path.join(ROOT, "include", "vitb200.h")).read()).group(1))
    assert lib.vb_abi_version() == header == _lib.ABI_VERSION == 7
    for name in ("vb_op_gemm", "vb_op_attention_ex", "vb_op_softmax_rows", "vb_graph_stats", "vb_last_attention_path"):
        assert name in declared


def test_attention_path_names_match_header_and_start_empty(lib):
    """The VB_ATTN_PATH_* values of the header are the ones the binding names; a thread that ran no attention reads NONE."""
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    values = {int(v): k.lower() for k, v in re.findall(r"#define VB_ATTN_PATH_(\w+) (\d+)", src)}
    assert values == {k: (v or "none") for k, v in _lib.ATTENTION_PATHS.items()}
    assert _lib.last_attention_path() is None and lib.vb_last_attention_path() == 0


def test_graph_stats_refuses_a_null_handle(lib):
    import ctypes as C
    n = C.c_int64(-1)
    assert lib.vb_graph_stats(None, C.byref(n), None, None, None) != 0 and n.value == -1
    assert b"null handle" in lib.vb_last_error(None)


def test_config_struct_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_config {"):src.index("} vb_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    assert [f for f, _ in _lib.VbConfig._fields_] == fields


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(lib):
    from vit_tensorflow_b200 import _lib, ViT
    with pytest.raises(_lib.VbError, match="no CUDA device"):
        _lib.op_linear(np.zeros((4, 8), np.float32), np.zeros((8, 64), np.float32))
    with pytest.raises(_lib.VbError, match="no CUDA device"):
        ViT(image_size=32, patch_size=16, num_classes=4, dim=32, depth=1, heads=2, mlp_dim=32, dim_head=16)


def test_reference_assertions(lib):
    from vit_tensorflow_b200 import ViT, DeepViT, CaiT, CrossViT
    kw = dict(num_classes=4, dim=32, depth=1, heads=2, mlp_dim=32)
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        ViT(image_size=30, patch_size=16, **kw)
    with pytest.raises(AssertionError, match="pool type must be either cls"):
        ViT(image_size=32, patch_size=16, pool="max", **kw)
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        DeepViT(image_size=30, patch_size=16, **kw)
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        CaiT(image_size=30, patch_size=16, cls_depth=1, **kw)
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        CrossViT(image_size=30, num_classes=4, sm_dim=32, lg_dim=32)
    with pytest.raises(NotImplementedError, match="layer_dropout"):
        CaiT(image_size=32, patch_size=16, cls_depth=1, layer_dropout=0.05, **kw)


def test_reference_assertions_of_the_8f_classes(lib):
    # t2t.py:56,84 ; vit_with_patch_merger.py:154 ; efficient.py:18-19 -- raised by the host classes before any engine call
    from vit_tensorflow_b200 import T2TViT, PatchMergerViT, EfficientViT
    with pytest.raises(AssertionError, match="pool type must be either cls"):
        T2TViT(image_size=32, num_classes=4, dim=32, depth=1, heads=2, mlp_dim=32, pool="max")
    with pytest.raises(AssertionError, match="depth, heads, and mlp_dim must be supplied"):
        T2TViT(image_size=32, num_classes=4, dim=32)
    with pytest.raises(AssertionError, match="Image dimensions must be divisible by the patch size."):
        PatchMergerViT(image_size=30, patch_size=16, num_classes=4, dim=32, depth=2, heads=2, mlp_dim=32)
    with pytest.raises(AssertionError, match="image dimensions must be divisible by the patch size"):
        EfficientViT(image_size=30, patch_size=16, num_classes=4, dim=32, transformer=lambda x, training=True: x)
    with pytest.raises(AssertionError, match="pool type must be either cls"):
        EfficientViT(image_size=32, patch_size=16, num_classes=4, dim=32, transformer=lambda x, training=True: x, pool="max")


def test_oracle_configs_of_the_8f_kinds():
    import oracle
    cfg = oracle.make_config("t2t_vit", image_size=224, num_classes=1000, dim=512, depth=5, heads=8, mlp_dim=512)
    assert cfg["t2t_dims"] == (147, 1323, 11907) and cfg["num_patches"] == 196            # t2t.py:63,66 at the default t2t_layers
    assert oracle.t2t_token_grid(cfg) == [(56, 56), (28, 28), (14, 14)]                   # SAME padding: ceil(size / stride)
    specs = oracle.weight_specs(cfg)
    assert specs["t2t.0.layers.0.to_qkv.kernel"][0] == (147, 441) and "t2t.0.layers.0.to_out.kernel" not in specs   # vit.py:53
    assert specs["patch.kernel"][0] == (11907, 512) and specs["pos_embedding"][0] == (1, 197, 512)
    pm = oracle.make_config("patch_merger_vit", image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=12, heads=8, mlp_dim=2048,
                            patch_merge_layer=6)
    assert pm["patch_merge_layer_index"] == 5 and oracle.weight_specs(pm)["patch_merger.queries"][0] == (8, 1024)
    assert oracle.make_config("patch_merger_vit", image_size=32, patch_size=16, num_classes=2, dim=8, depth=12, heads=1,
                              mlp_dim=8)["patch_merge_layer_index"] == 5                   # default(None, depth // 2) - 1


def test_dp_unique_id_through_dlopened_nccl(lib):
    """vb_dp_unique_id: the engine dlopens NCCL on demand (no load-time dependency) and calls ncclGetUniqueId through its own
    declarations of the NCCL C API -- works without a GPU, so the dlopen / dlsym / by-value-struct plumbing is checked here."""
    import ctypes as C
    from vit_tensorflow_b200 import _lib
    from vit_tensorflow_b200.runtime import default_nccl_library
    path = default_nccl_library()
    if not os.path.exists(path):
        pytest.skip("no NCCL library in this environment")
    os.environ["VB_NCCL_LIB"] = path
    a, b = (C.c_char * 128)(), (C.c_char * 128)()
    _lib.check(lib.vb_dp_unique_id(a))
    _lib.check(lib.vb_dp_unique_id(b))
    assert bytes(a) != bytes(128) and bytes(a) != bytes(b)
    # the collective entry points refuse a handle-less call instead of crashing
    assert lib.vb_dp_init(None, a, 0, 1) != 0 and b"null argument" in lib.vb_last_error(None)
    assert lib.vb_forward_allgather(None, None, 0, 1, 32, 32, None, None) != 0


def test_drop_in_import_names():
    # README.md:47,148,177,325 of the reference
    from vit_tensorflow import ViT
    from vit_tensorflow.deepvit import DeepViT
    from vit_tensorflow.cait import CaiT
    from vit_tensorflow.cross_vit import CrossViT
    import vit_tensorflow_b200 as vb
    assert (ViT, DeepViT, CaiT, CrossViT) == (vb.ViT, vb.DeepViT, vb.CaiT, vb.CrossViT)
    from vit_tensorflow.parallel_vit import ViT as PV
    from vit_tensorflow.distill import DistillableViT
    from vit_tensorflow.t2t import T2TViT
    from vit_tensorflow.vit_with_patch_merger import ViT as PMV, PatchMerger
    from vit_tensorflow.efficient import ViT as EV
    assert (PV, DistillableViT, T2TViT, PMV, PatchMerger, EV) == (vb.ParallelViT, vb.DistillableViT, vb.T2TViT, vb.PatchMergerViT,
                                                                   vb.PatchMerger, vb.EfficientViT)


def test_built_for_sm90a_with_wgmma(lib):
    """The shipped library contains sm_90a SASS with wgmma (HGMMA), TMA loads (UTMALDG) and tensor-core MMA (HMMA)."""
    import shutil
    import subprocess
    from vit_tensorflow_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG", "HMMA"):
        assert mnemonic in sass, mnemonic


def test_attribute_surface_supports_the_wrapper_expressions():
    """`model.pos_embedding` / `model.cls_token` as mae.py:54, simmim.py:95, mpp.py:204-208 use them (slicing, einops repeat,
    arithmetic).  They are properties over the model's weight dict, so a stub holding `_specs` / `_weights` is enough on a CPU
    box (constructing a real model needs an H100)."""
    import numpy as np
    from einops import repeat
    from vit_tensorflow_b200.models import _EngineModel

    class Stub(_EngineModel):
        def __init__(self):
            rng = np.random.default_rng(0)
            self._weights = {"pos_embedding": rng.standard_normal((1, 17, 8)).astype(np.float32),
                             "cls_token": rng.standard_normal((1, 1, 8)).astype(np.float32)}
            self._specs = {k: v.shape for k, v in self._weights.items()}

        def __del__(self):
            pass

    m = Stub()
    w = m._weights
    n, b = 9, 3
    tokens = np.ones((b, n, 8), np.float32)
    assert m.pos_embedding.shape == (1, 17, 8) and m.pos_embedding.shape[-2:] == (17, 8)                   # mae.py:33
    np.testing.assert_array_equal(tokens + m.pos_embedding[:, 1:(n + 1)], tokens + w["pos_embedding"][:, 1:n + 1])   # mae.py:54, simmim.py:95
    np.testing.assert_array_equal(m.pos_embedding[:, :(n + 1)], w["pos_embedding"][:, :n + 1])             # mpp.py:208
    c = repeat(m.cls_token, '() n d -> b n d', b=b)                                                        # mpp.py:204
    assert c.shape == (b, 1, 8)
    np.testing.assert_array_equal(np.concatenate([c, tokens], axis=1)[:, 0], np.broadcast_to(w["cls_token"][0], (b, 8)))
    np.testing.assert_array_equal(2.0 * m.pos_embedding + 1.0, 2.0 * w["pos_embedding"] + 1.0)
    w["pos_embedding"] = np.zeros((1, 17, 8), np.float32)                                                  # a newly set weight is seen
    assert float(np.abs(m.pos_embedding).max()) == 0.0
    del m._specs["cls_token"]                                                                              # CaiT-less models: AttributeError
    try:
        m.cls_token
        raise AssertionError("expected AttributeError")
    except AttributeError:
        pass
