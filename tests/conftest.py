import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def cb():
    import clarabel_jl_b200 as cb
    from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
    cb.register_kktsolver("qdldl", OracleDirectLDLKKTSolver)
    return cb


@pytest.fixture(scope="session")
def gpu_available():
    import torch
    return torch.cuda.is_available()
