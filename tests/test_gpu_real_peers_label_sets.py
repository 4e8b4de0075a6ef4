"""Real-peer check of multi-label positives: on a machine with two or more H100s, run tools/multi_gpu_check.py with
--label-sets on two ranks. Each rank's text label sets ride its ids publish and the peers' ids pulls (flag 0), and
each rank checks its loss and gradients against the float64 oracle of the label sets. Skipped on a one-GPU
machine, where the loopback tests of test_gpu_label_sets.py cover the W-rank schedule."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_real_peers_pass_the_label_sets_check():
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29703", os.path.join(ROOT, "tools", "multi_gpu_check.py"),
           "--label-sets", "--skip-parity"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = "\n".join((out.stdout + out.stderr).splitlines()[-30:])
    assert out.returncode == 0, tail
    assert "MULTI-GPU CHECK PASS" in out.stdout, tail
    assert "label sets" in out.stdout and " FAIL" not in out.stdout, tail
