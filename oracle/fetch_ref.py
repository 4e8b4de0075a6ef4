#!/usr/bin/env python
"""Place the UNMODIFIED reference next to the package for the CPU arm of bench.py (`--impl reference`).

    python oracle/fetch_ref.py [--src DIR]

The reference (ahmdtaha/distributed_sigmoid_loss) is five pure-Python files with no setup.py, so there is nothing to
build: this recipe copies the *.py files verbatim from a checkout of it (--src, else $SIGLIP_REFERENCE_SRC, else a
`reference` directory beside this repository) into `oracle/_ref/`. That directory is git-ignored: it is never part of
the history, but a tree that build() has run in carries it. Nothing but `bench.py --impl reference` (and the test that
checks the copy) reads it: it imports `DDPSigmoidLoss` from there and runs it through its own public API
(distributed_sigmoid_loss.py:8-48) on the host cores. A manifest with the sha256 of every file is written beside the
copies; tests/golden/reference_sha256.json pins the upstream digests.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_SRC = os.environ.get("SIGLIP_REFERENCE_SRC", os.path.join(os.path.dirname(ROOT), "reference"))
FILES = ("distributed_sigmoid_loss.py", "distributed_utils.py", "rwightman_sigmoid_loss.py",
         "test_distributed_sigmoid_loss.py", "test_sigmoid_loss_variants.py")


def fetch(src: str = DEFAULT_SRC, quiet: bool = False, dest: str = DEST) -> bool:
    """Returns True if `dest` (oracle/_ref) holds the reference afterwards (False: no checkout of the reference at `src`
    and no earlier copy)."""
    if not os.path.isdir(src):
        return os.path.exists(os.path.join(dest, FILES[0]))
    os.makedirs(dest, exist_ok=True)
    manifest = {}
    for name in FILES:
        s = os.path.join(src, name)
        if not os.path.exists(s):
            continue
        d = os.path.join(dest, name)
        shutil.copyfile(s, d)
        with open(d, "rb") as f:
            manifest[name] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, "MANIFEST.json"), "w") as f:
        json.dump({"sha256": manifest}, f, indent=1)
    if not quiet:
        print(f"reference: {len(manifest)} files -> {dest}")
    return FILES[0] in manifest


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=DEFAULT_SRC)
    a = ap.parse_args()
    sys.exit(0 if fetch(a.src) else 1)
