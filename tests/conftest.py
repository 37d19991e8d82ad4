import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def kvb():
    """The product package (llm-d-kv-cache_b200); builds libkvb.so first if nvcc is present and it is stale."""
    try:
        import importlib.util
        spec = importlib.util.spec_from_file_location("kvb_build", os.path.join(ROOT, "llm-d-kv-cache_b200", "build.py"))
        build = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(build)
        build.build()
    except Exception as e:  # no nvcc on this box: use the prebuilt library that travelled with the repo
        print(f"[conftest] not rebuilding libkvb.so: {e}")
    return importlib.import_module("llm-d-kv-cache_b200")


@pytest.fixture(scope="session")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "gpu-marked test needs a CUDA device"
    torch.cuda.set_device(0)
    return torch


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "kvblock_golden.json")) as f:
        return json.load(f)
