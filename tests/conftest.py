import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# A protocol bug in a (loopback) multi-chunk test must fail the test within seconds, not after the production default of
# ten minutes: every context created during the test session bounds its waits on "peers" at 30 s.
os.environ.setdefault("SIGLIP_PEER_TIMEOUT_MS", "30000")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a) device; run with -m gpu on the GPU box")


def _cuda_ok() -> bool:
    try:
        import torch

        return torch.cuda.is_available() and torch.cuda.get_device_capability(0)[0] == 9
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a machine without an H100 skips instead of erroring
    if _cuda_ok():
        return
    skip = pytest.mark.skip(reason="no sm_90 device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def golden_cases(f32=False):
    """Fixture names. f32=False: inputs are bf16-representable (what the bf16 path consumes exactly); f32=True: raw fp32
    inputs as the reference's own test feeds them (the module's fp32-input path); f32="all": both."""
    names = sorted(f[:-4] for f in os.listdir(GOLDEN_DIR) if f.endswith(".npz"))
    if f32 == "all":
        return names
    return [n for n in names if ("_f32" in n) == bool(f32)]


def load_golden(name):
    import numpy as np

    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    world, batch, dim = int(z["world"]), int(z["batch"]), int(z["dim"])
    case = dict(name=name, world=world, batch=batch, dim=dim, t_prime=float(z["t_prime"]), bias=float(z["bias"]),
                img_all=z["img_all"], txt_all=z["txt_all"], variants={})
    for variant in ("ddp", "rw_bidir", "rw_uni"):
        ranks = []
        for r in range(world):
            ranks.append({k: z[f"{variant}.r{r}.{k}"] for k in ("loss", "dimg", "dtxt", "dt_prime", "dbias")})
        case["variants"][variant] = ranks
    return case
