import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # a fresh checkout has no built artefacts (they are git-ignored): build them once, in-tree
    lib = ROOT / "pbs_plus_b200" / "libpbsgpu.so"
    if not lib.exists() or not (ROOT / "tests" / "cxx" / "driver.bin").exists():
        try:
            from pbs_plus_b200 import build as b
            b.build()
            b.build_cxx_driver()
        except Exception as e:  # the tests that need the library will say so themselves
            print(f"[conftest] could not build libpbsgpu.so: {e}", file=sys.stderr)


def _has_gpu() -> bool:
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
