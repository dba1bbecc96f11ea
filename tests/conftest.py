import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


def _has_gpu():
    if os.environ.get("LILIOM_ASSUME_GPU") == "1":      # e.g. under compute-sanitizer: skip the torch import, the library itself reports a missing device
        return True
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
def oracle():
    import oracle_lib
    oracle_lib.build()
    return oracle_lib


@pytest.fixture(scope="session")
def world_small():
    """100k-point map, Horizon + HDL sweeps from the default pose (seeded)."""
    from liliom_b200 import synth
    m, _ = synth.make_map(100_000)
    T = synth.default_true_pose()
    hz, q_hz = synth.make_horizon_sweep(T)
    hdl, q_hdl = synth.make_hdl64_sweep(T)
    return dict(map=m, T=T, guess=synth.perturbed_pose(T), hz=hz, q_hz=q_hz, hdl=hdl, q_hdl=q_hdl)


@pytest.fixture(scope="session")
def ctx48():
    import liliom_b200 as L
    c = L.Context(variant=0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def ctx32():
    import liliom_b200 as L
    c = L.Context(variant=1)
    yield c
    c.close()
