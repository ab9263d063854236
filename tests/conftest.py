import gzip
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "reference: needs the read-only reference tree (/root/reference)")


@pytest.fixture(scope="session")
def golden_env():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "env_playouts.json.gz"), "rt") as f:
        return json.load(f)


@pytest.fixture(scope="session")
def emul_lib():
    """Integer kernels compiled for the CPU SIMT emulator (test tier only, never the product)."""
    import importlib
    build = importlib.import_module("chinesechess-alphazero_b200.build")
    from cczero_b200.lib import CzLib
    return CzLib(build.build_emul())


@pytest.fixture(scope="session")
def emul_env(emul_lib):
    from cczero_b200.env import StaticEnv
    return StaticEnv(emul_lib, "cpu")


@pytest.fixture(scope="session")
def cuda_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from cczero_b200.lib import get_lib
    return get_lib()   # raises if the CUDA library is missing: no fallback


@pytest.fixture(scope="session")
def cuda_env(cuda_lib):
    from cczero_b200.env import StaticEnv
    return StaticEnv(cuda_lib, "cuda")
