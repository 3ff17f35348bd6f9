import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) CUDA device")
    config.addinivalue_line("markers", "slow: takes more than ~20 s on 8 host cores")


def _has_gpu():
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


@pytest.fixture(scope="session")
def w2x():
    """The product binding (ctypes over libw2x_b200.so); builds the library if it is missing."""
    import w2x_loader
    mod = w2x_loader.load()
    if not os.path.exists(mod.lib_path()):
        mod.build()
    return mod


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def oracle_models(oracle_mod):
    return {n: oracle_mod.OracleModel.golden(n) for n in oracle_mod.MODEL_NAMES}


@pytest.fixture(scope="session")
def json_models(oracle_models, tmp_path_factory):
    """The three models written back out in the reference's JSON format (values identical)."""
    d = tmp_path_factory.mktemp("models")
    paths = {}
    for name, om in oracle_models.items():
        p = os.path.join(d, f"{name}_model.json")
        om.write_json(p)
        paths[name] = p
    return paths


@pytest.fixture(scope="session")
def ncpu():
    return max(1, min(16, os.cpu_count() or 1))


def golden_path(*parts):
    return os.path.join(GOLDEN, *parts)
