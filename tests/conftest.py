import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def oracle_params64():
    """Oracle weights (float64 copies of the fp32 values) with perturbed biases / beta / gamma."""
    import torch
    from oracle import cyclegan_oracle as O
    return O.init_params(seed=1234, dtype=torch.float64, perturb_affine=True)
