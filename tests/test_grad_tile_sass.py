"""The built library carries the gradient kernel's 256-column instantiations: wgmma m64n256k16 (HGMMA.64x256x16 in
SASS) for clusters of 1, 2 and 4 CTAs, and nowhere else (the loss kernel keeps its 128-column tiles)."""
import os
import re
import shutil
import subprocess

import pytest

from distributed_sigmoid_loss_b200 import _capi


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


def test_gradient_kernel_has_256_column_instantiations():
    exe = _cuobjdump()
    if exe is None or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run([exe, "-sass", _capi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    wide = {}
    for block in sass.split("Function : ")[1:]:
        name = block.split("\n", 1)[0].strip()
        if "HGMMA.64x256x16" in block:
            wide[name] = block
    # siglip_gemm_kernel<kModeOut = 1, 4 stages, cluster size, ..., 256>
    clusters = sorted(int(m.group(1)) for n in wide for m in [re.search(r"siglip_gemm_kernelILi1ELi4ELi(\d)E.*ELi256E", n)] if m)
    assert clusters == [1, 2, 4], sorted(wide)
    assert len(wide) == 3, sorted(wide)
