"""Every loss-kernel instantiation of the built library (default, sample ids, metrics, weights and their combinations,
for every cluster size and stage count) keeps 168 registers per thread and spills nothing to local memory."""
import os
import re
import shutil
import subprocess

import pytest

from distributed_sigmoid_loss_b200 import _capi


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


def test_loss_kernels_keep_168_registers_and_no_spills():
    exe = _cuobjdump()
    if exe is None or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([exe, "-res-usage", _capi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    usage = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "REG:" in line:
            usage[name] = line
            name = None
    # siglip_gemm_kernel<kModeLoss = 0, stages, cluster, kF8, kIds, kMetrics, kWeights, 128>
    loss = {n: u for n, u in usage.items() if re.search(r"siglip_gemm_kernelILi0ELi\d", n)}
    assert len(loss) == 48, sorted(loss)   # 2 stage counts x 3 cluster sizes x 8 label / metric / weight variants
    for n, u in loss.items():
        assert re.search(r"\bREG:168\b", u), (n, u)
        assert re.search(r"\bLOCAL:0\b", u), (n, u)
