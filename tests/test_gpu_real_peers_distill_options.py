"""Real-peer check of distillation with the other options: on a machine with two or more H100s, run
tools/multi_gpu_check.py with --distill-options on two ranks. The teacher's rows of the hard negatives and extra texts
travel with the text through the peer pulls; each rank checks its loss, gradients and per-sample losses against the
float64 composed oracle, with label sets, extras, weights and excluded groups, on both schedules. Skipped on a one-GPU
machine, where the loopback tests of test_gpu_distill_options.py cover the W-rank schedule."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_real_peers_pass_the_distill_options_check():
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29706", os.path.join(ROOT, "tools", "multi_gpu_check.py"),
           "--distill-options", "--skip-parity"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = "\n".join((out.stdout + out.stderr).splitlines()[-30:])
    assert out.returncode == 0, tail
    assert "MULTI-GPU CHECK PASS" in out.stdout, tail
    assert "distill-options" in out.stdout and " FAIL" not in out.stdout, tail
