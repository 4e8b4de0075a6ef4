"""Real-peer check under pytest: on a machine with two or more H100s, run tools/multi_gpu_check.py (one rank per GPU, NCCL
process group, CUDA-IPC peer mappings, in-kernel flags over NVSwitch) on two ranks and require every comparison to pass —
the float64 closed form over the global batch, fp32 autograd with the text gradient all-reduced (the reduce-scatter of
all_gather's backward, torch distributed/nn/functional.py:343-354), the reference's own acceptance test
(test_distributed_sigmoid_loss.py:122-141) on GPUs, uneven batches, the scalar-gradient mean and a late rank.
On a one-GPU box (the driver's GPU test box) it is skipped: the one-GPU loopback tests of test_gpu_parity.py cover the
W-rank schedules there, and bench.py's `parity` block covers real peers at every N of the scaling run."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_real_peers_pass_the_multi_gpu_check():
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")      # a hung peer fails the test instead of the 10 min default
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29677", os.path.join(ROOT, "tools", "multi_gpu_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = "\n".join((out.stdout + out.stderr).splitlines()[-30:])
    assert out.returncode == 0, tail
    assert "MULTI-GPU CHECK PASS" in out.stdout, tail
    assert " FAIL" not in out.stdout, tail
