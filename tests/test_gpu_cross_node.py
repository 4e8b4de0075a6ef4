"""Groups that span nodes on H100s: tools/cross_node_check.py under torch.distributed.run compares every rank's loss,
gradients (extras included), t_prime / bias gradients and per-sample losses with the float64 global-batch oracle.

On one H100, 2 and then 3 processes share the device over gloo with ranks_per_node=1: every rank is a "node" of its
own, so every text of the other ranks reaches it through the all-to-all exchange. With two GPUs, NCCL with one rank
per "node" is also compared with the same data on one node (the in-kernel exchange alone); with four, two nodes of two
GPUs run the in-kernel node exchange and the all-to-all together. Every launch runs in its own session and is killed
with all its processes on timeout."""
import os
import signal
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _launch(nproc: int, port: int, *args: str, timeout: int = 600) -> None:
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tools", "cross_node_check.py"), *args]
    proc = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                            start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        out, _ = proc.communicate()
        pytest.fail("cross-node check timed out:\n" + "\n".join(out.splitlines()[-40:]))
    finally:
        if proc.poll() is None:
            os.killpg(proc.pid, signal.SIGKILL)
            proc.wait()
    tail = "\n".join(out.splitlines()[-60:])
    assert proc.returncode == 0, tail
    assert "CROSS-NODE CHECK PASS" in out and " FAIL" not in out, tail


def _gpus() -> int:
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.parametrize("nproc,port", [(2, 29711), (3, 29713)])
def test_one_rank_nodes_on_one_device_over_gloo(nproc, port):
    _launch(nproc, port, "--ranks-per-node", "1", "--backend", "gloo", "--same-device")


@pytest.mark.gpu
def test_two_one_gpu_nodes_over_nccl_match_one_node():
    if _gpus() < 2:
        pytest.skip("needs two GPUs with peer access on one host")
    _launch(2, 29715, "--ranks-per-node", "1", "--backend", "nccl", "--compare-single-node")


@pytest.mark.gpu
def test_two_nodes_of_two_gpus_over_nccl():
    if _gpus() < 4:
        pytest.skip("needs four GPUs with peer access on one host")
    _launch(4, 29717, "--ranks-per-node", "2", "--backend", "nccl")
