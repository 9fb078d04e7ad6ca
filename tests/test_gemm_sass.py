"""CPU test of what ptxas made of the wgmma GEMM: in every GEMM kernel of the shipped library the wgmmas of a k-block are
chained.  A function call anywhere in the wgmma pipeline (a printf in the mbarrier watchdog, for example) makes ptxas
serialise every wgmma.mma_async (warning C7510): each HGMMA then carries the gsb0 scoreboard and is waited for before the
next one issues.  Chained, only the last HGMMA of a commit group carries it."""
import os
import re

import pytest


def test_gemm_wgmma_chain_is_not_serialised(lib):
    import shutil
    import subprocess
    from vit_tensorflow_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    kernels = 0
    for func in re.split(r"\n\s*Function : ", sass)[1:]:
        name = func.split("\n", 1)[0].strip()
        if "gemm_bf16_kernel" not in name:
            continue
        kernels += 1
        hgmma = re.findall(r"HGMMA\.[^\n]*", func)
        gsb0 = [line for line in hgmma if "gsb0" in line]
        assert hgmma, f"{name}: no HGMMA"
        assert len(gsb0) < len(hgmma), f"{name}: all {len(hgmma)} HGMMAs carry gsb0 (wgmmas serialised)"
    assert kernels > 0, "no wgmma GEMM kernel found in the library"
