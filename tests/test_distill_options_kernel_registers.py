"""The three distillation-with-options kernels of the built library (siglip_gemm_kernel<kModeDistillOpts = 8,
kDistillStages = 4, cluster 1 / 2 / 4>) use at most 168 registers per thread, like the other loss kernels, and spill
nothing to local memory (DESIGN.md, "Distillation with the other options")."""
import os
import re
import shutil
import subprocess

import pytest

from distributed_sigmoid_loss_b200 import _capi


def test_distill_options_kernels_fit_168_registers_and_no_spills():
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
    kern = {n: u for n, u in usage.items() if re.search(r"siglip_gemm_kernelILi8ELi4ELi[124]E", n)}
    assert len(kern) == 3, sorted(kern)   # 3 cluster sizes at kDistillStages
    for n, u in kern.items():
        assert int(re.search(r"\bREG:(\d+)\b", u).group(1)) <= 168, (n, u)
        assert re.search(r"\bLOCAL:0\b", u), (n, u)
        # the kernel's own 16-byte frame: a register spill goes to the stack and grows it (LOCAL stays 0)
        assert re.search(r"\bSTACK:16\b", u), (n, u)
