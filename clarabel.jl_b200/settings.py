"""Solver settings: mirror of the reference `Settings{T}` kw-struct.

Reference: src/settings.jl:70-148.  Only the fields the KKT path and its caller
read are kept; names and defaults are the reference's.  The B200 backend is
selected exactly like a reference LDL backend, by `direct_solve_method`
(src/settings.jl:114, read at src/kktsolvers/kktsolver_directldl.jl:100).
"""
from dataclasses import dataclass, field
import numpy as np

_EPS = float(np.finfo(np.float64).eps)


@dataclass
class Settings:
    max_iter: int = 200
    time_limit: float = float("inf")
    verbose: bool = False
    max_step_fraction: float = 0.99

    tol_gap_abs: float = 1e-8
    tol_gap_rel: float = 1e-8
    tol_feas: float = 1e-8
    tol_infeas_abs: float = 1e-8
    tol_infeas_rel: float = 1e-8
    tol_ktratio: float = 1e-6

    reduced_tol_gap_abs: float = 5e-5
    reduced_tol_gap_rel: float = 5e-5
    reduced_tol_feas: float = 1e-4
    reduced_tol_infeas_abs: float = 5e-12
    reduced_tol_infeas_rel: float = 5e-5
    reduced_tol_ktratio: float = 1e-4

    equilibrate_enable: bool = True
    equilibrate_max_iter: int = 10
    equilibrate_min_scaling: float = 1e-4
    equilibrate_max_scaling: float = 1e4

    linesearch_backtrack_step: float = 0.8
    min_switch_step_length: float = 1e-1
    min_terminate_step_length: float = 1e-4

    max_threads: int = 0

    direct_kkt_solver: bool = True
    # reference: :auto | :qdldl | :cholmod | ... ; here "b200" is the new
    # backend symbol and "qdldl" the CPU oracle (injected by tests / bench).
    direct_solve_method: str = "b200"

    static_regularization_enable: bool = True
    static_regularization_constant: float = 1e-8
    static_regularization_proportional: float = _EPS * _EPS

    dynamic_regularization_enable: bool = True
    dynamic_regularization_eps: float = 1e-13
    dynamic_regularization_delta: float = 2e-7

    iterative_refinement_enable: bool = True
    iterative_refinement_reltol: float = 1e-13
    iterative_refinement_abstol: float = 1e-12
    iterative_refinement_max_iter: int = 10
    iterative_refinement_stop_ratio: float = 5.0

    presolve_enable: bool = True
    input_sparse_dropzeros: bool = False

    # B200 backend knobs (no reference counterpart)
    b200_devices: tuple = field(default_factory=tuple)   # () = current device only
    # compute the NT scaling of symmetric cones on the device (cb200_update_scaling) instead of on the host;
    # used with direct_solve_method="b200" when every cone is Zero / NN / SOC / PSD
    b200_device_cone_scaling: bool = False
