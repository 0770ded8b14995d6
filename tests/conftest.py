import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the CPU oracle (torch convs) gets slower, not faster, beyond ~16 threads on the many-core GPU hosts
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))


@pytest.fixture(scope="session")
def state():
    """Seeded synthetic weights shared by oracle and engine (weights.make_state)."""
    import torch
    from voicefixer_main_b200.weights import make_state
    return make_state(1234)


def load_golden(name):
    import numpy as np
    return np.load(os.path.join(GOLDEN, name))


@pytest.fixture(scope="session")
def golden_fingerprint_ok(state):
    """The golden files were generated with make_state(1234); verify the local
    generator reproduces the same weights before trusting any golden comparison."""
    import numpy as np
    from oracle.make_golden import state_fingerprint
    fp = state_fingerprint(state)
    ref = load_golden("stage_b_t101.npz")["fingerprint"]
    assert np.allclose(fp, ref, rtol=1e-12), "synthetic weight generator drifted from the golden files"
    return True
