import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu on an H100)")


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


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the CUDA library (cross-compiles without a GPU) and the oracle once per session."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def small_world():
    """~180k-point map (80 m x 80 m of street grid) + a 4k-point Livox sweep; oracle map built once."""
    from oracle import oracle_py as O
    from sr_livo_b200 import synth
    pts = synth.sample_map_points(80.0, 60.0, seed=1)
    sw = synth.make_sweep(4000, seed=1000, yaw=0.5)
    om = O.OracleMap()
    om.add_points(pts)
    return dict(pts=pts, sweep=sw, omap=om)


@pytest.fixture(scope="session")
def cfg1_world():
    """BASELINE config 1 scale: ~200k-pt map, 20k-pt sweep."""
    from oracle import oracle_py as O
    from sr_livo_b200 import synth
    pts = synth.sample_map_points(84.0, 60.0, seed=11)
    sw = synth.make_sweep(20000, seed=1011, yaw=0.4)
    om = O.OracleMap()
    om.add_points(pts)
    return dict(pts=pts, sweep=sw, omap=om)
