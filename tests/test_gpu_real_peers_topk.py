"""Real-peer check of the top-K retrieval: on a machine with two or more H100s, run tools/multi_gpu_check.py with
--metrics-topk on two ranks. Each rank's t2i lists merge every rank's sorted column lists of its chunk (flag kind 5,
step-parity buffers, read over P2P), and each rank checks its lists and recall@k exactly against the float64 oracle.
Skipped on a one-GPU machine, where the loopback tests of test_gpu_retrieval_topk.py cover the W-rank merge."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_real_peers_pass_the_topk_check():
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29699", os.path.join(ROOT, "tools", "multi_gpu_check.py"),
           "--metrics-topk", "--skip-parity"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = "\n".join((out.stdout + out.stderr).splitlines()[-30:])
    assert out.returncode == 0, tail
    assert "MULTI-GPU CHECK PASS" in out.stdout, tail
    assert "top-K" in out.stdout and " FAIL" not in out.stdout, tail
