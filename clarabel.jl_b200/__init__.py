"""clarabel.jl_b200 — H100-native KKT linear-system path for Clarabel.jl's interior-point loop.

Scope (SURVEY.md section 8): cone-Hessian -> KKT value update, static regularisation, sparse
multifrontal LDL' factorisation, triangular solves + iterative refinement, behind the
reference's AbstractKKTSolver / AbstractDirectLDLSolver plugin interfaces.  The numerics live
in csrc/ (hand-written sm_90a CUDA + host C++ symbolic analysis) behind the C-ABI declared in
include/clarabel_b200.h; the Python modules here are the host-side mirror of the reference's
interface (the Julia toolchain is absent from this image) and the caller harness.
"""
from . import settings, cones, problemdata, kkt_assembly, kktsystem, solver, problems  # noqa: F401
from .settings import Settings  # noqa: F401
from .cones import (ZeroConeT, NonnegativeConeT, SecondOrderConeT, PSDTriangleConeT,  # noqa: F401
                    ExponentialConeT, PowerConeT, GenPowerConeT, CompositeCone)
from .solver import Solver, STATUS_NAMES  # noqa: F401
from .kktsystem import register_kktsolver  # noqa: F401
