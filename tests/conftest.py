import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a); select with -m gpu")


_cases = {}


def get_case(name, scan_index=0):
    """Session cache of synthetic cases (map generation is the slow part)."""
    from superodom_b200 import synth
    key = (name, scan_index)
    if key not in _cases:
        base = (name, "map")
        if base not in _cases:
            _cases[base] = synth.make_map_for(name)
        scene, map_xyzi = _cases[base]
        _cases[key] = synth.make_case_on(scene, map_xyzi, name, scan_index)
    return _cases[key]


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def gpu_api():
    from superodom_b200 import api
    lib = api.load_library()          # raises if the extension is missing: no silent fallback
    assert lib.so_device_available(), "no sm_90 device visible"
    return api


def quat_angle(qa, qb):
    """rotation angle between two unit quaternions (xyzw), sign-insensitive"""
    d = abs(float(np.dot(qa, qb)))
    return 2.0 * np.arccos(min(1.0, d))
