"""Real-peer check of the focal pair loss: on a machine with two or more H100s, run tools/multi_gpu_check.py with
--focal on two ranks. gamma and alpha are kernel parameters, so the exchange is the one of the options the step uses
(positional, label sets with extras, weights and excluded groups); each rank checks its loss and gradients against the
float64 focal oracle. Skipped on a one-GPU machine, where the loopback tests of test_gpu_focal.py cover the W-rank
schedule."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_real_peers_pass_the_focal_check():
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29704", os.path.join(ROOT, "tools", "multi_gpu_check.py"),
           "--focal", "--skip-parity"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = "\n".join((out.stdout + out.stderr).splitlines()[-30:])
    assert out.returncode == 0, tail
    assert "MULTI-GPU CHECK PASS" in out.stdout, tail
    assert "focal" in out.stdout and " FAIL" not in out.stdout, tail
