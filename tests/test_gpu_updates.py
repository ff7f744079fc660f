"""GPU: the reference's data-updating scenarios (test/OptTests/data_updating.jl) through the B200
backend: Solver.update_P/A -> cb200_update_P/A, then a re-solve without a new symbolic analysis."""
import pytest

from test_caller_paths import SCENARIOS, run_scenario

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scenario", SCENARIOS)
def test_data_updating_b200_backend(cb, scenario):
    # 1e-6 on the GPU; the reference's 1e-7 is what the CPU variant in test_caller_paths.py asserts
    run_scenario(cb, "b200", scenario, tol=1e-6)
