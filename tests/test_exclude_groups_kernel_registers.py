"""The six excluded-groups kernels of the built library (siglip_gemm_kernel<kModeGroups = 5, 4 or 6 stages, cluster
1 / 2 / 4>) use 168 registers per thread, like the other loss kernels, and spill nothing to local memory (DESIGN.md,
"Excluded groups")."""
import os
import re
import shutil
import subprocess

import pytest

from distributed_sigmoid_loss_b200 import _capi


def test_exclude_groups_kernels_use_168_registers_and_no_spills():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(_capi.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    out = subprocess.run([exe, "-res-usage", _capi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    usage, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "REG:" in line:
            usage[name] = line
            name = None
    kern = {n: u for n, u in usage.items() if re.search(r"siglip_gemm_kernelILi5ELi[46]ELi[124]E", n)}
    assert len(kern) == 6, sorted(kern)   # 2 stage counts x 3 cluster sizes
    for n, u in kern.items():
        assert re.search(r"\bREG:168\b", u), (n, u)
        assert re.search(r"\bLOCAL:0\b", u), (n, u)
        # the kernel's own 16-byte frame: a register spill goes to the stack and grows it (LOCAL stays 0)
        assert re.search(r"\bSTACK:16\b", u), (n, u)
