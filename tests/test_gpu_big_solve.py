"""GPU tests of the big-front solves (k_big_tri_fwd / k_big_tri_bwd: one launch per level and
direction whatever the pivot width, the 64-blocks of L11 chained by ready flags) on designed fronts
longer than the front zoo's: a root of 18 blocks with a 12-column tail and, in one level below it,
children of 1 to 11 blocks with partial tails and L21 below each.  Checked against the
extended-precision multifrontal reference, for bitwise run-to-run reproducibility, and for a launch
count that does not grow with ns."""
import numpy as np
import pytest
import front_zoo as fz
from mf_numpy import MFNumpy

pytestmark = pytest.mark.gpu

CHILDREN = ((64, 960), (65, 960), (128, 400), (300, 50), (700, 20))     # (ns, nr): nf * ns >= 65536, ns > 32


def design_chains():
    d = fz.Design("big_chains", 21)
    root = d.node(1100)                                        # 17 full blocks + a 12-column tail, nr = 0
    for ns, nr in CHILDREN:
        d.node(ns, root, nr)
    return d


def design_root(ns):
    d = fz.Design("big_root%d" % ns, 22)
    d.node(ns)
    return d


def _setup(monkeypatch, design, env=None, **over):
    from clarabel_jl_b200 import lib
    from clarabel_jl_b200.kktsolver_b200 import B200DirectLDLSolver
    for k, v in {**fz.ZOO_ENV, **(env or {})}.items():
        monkeypatch.setenv(k, v)
    K, sg, _ = design.build()
    a = lib.Symbolic(K, ordering=2).arrays()
    fz.check_design(design, a)
    fronts, _, _ = fz.route(a, K)
    assert all(f["solve"] == "big" for f in fronts)
    h = B200DirectLDLSolver(K, sg, None, ordering=2, **over)
    assert h.refactor()
    return K, sg, a, h


@pytest.mark.parametrize("env", [{}, {"CB200_MULTISTREAM": "0"}, {"CB200_GRAPH": "0"}],
                         ids=["default", "single_stream", "no_graph"])
def test_big_chains_match_reference(monkeypatch, env):
    d = design_chains()
    K, sg, a, h = _setup(monkeypatch, d, env)
    levels = {int(a["sn_level"][s]) for s in range(len(a["sn_first"]) - 1)}
    assert len(levels) == 2                                    # all children in one level
    mf = MFNumpy(a, np.longdouble)
    mf.factor(K.data, sg)
    rng = np.random.default_rng(11)
    for b in (rng.standard_normal(K.shape[0]), np.ones(K.shape[0])):
        x = np.zeros_like(b); h.solve(x, b)
        xr = mf.solve(b).astype(float)
        assert np.abs(x - xr).max() <= 1e-12 * np.abs(xr).max()


def test_big_chains_bitwise_reproducible(monkeypatch):
    d = design_chains()
    K, sg, _, h = _setup(monkeypatch, d, use_cuda_graph=1)
    b = np.random.default_rng(12).standard_normal(K.shape[0])
    first = np.zeros_like(b); h.solve(first, b)                # captures the solve graph
    assert h.stats()["solve_graph"] == 1
    for _ in range(20):                                        # graph replays
        x = np.zeros_like(b); h.solve(x, b)
        assert np.array_equal(x, first)
    _, _, _, h2 = _setup(monkeypatch, d, use_cuda_graph=0)
    x = np.zeros_like(b); h2.solve(x, b)
    assert h2.stats()["solve_graph"] == 0
    assert np.array_equal(x, first)


def test_big_launches_do_not_grow_with_ns(monkeypatch):
    counts = []
    for ns in (256, 1100):
        _, _, _, h = _setup(monkeypatch, design_root(ns), {"CB200_GRAPH": "0"})
        b = np.ones(ns)
        n0 = h.timers()["nlaunch"]
        x = np.zeros_like(b); h.solve(x, b)
        counts.append(h.timers()["nlaunch"] - n0)
        assert np.all(np.isfinite(x))
    assert counts[0] == counts[1], counts
