"""CPU checks of the extended-precision references in kkt_reference.py against the CPU oracle
(oracle/kktsolver_oracle.py), so that the GPU comparisons of test_gpu_kkt_update.py rest on
checked references."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla
import kkt_reference as kr
from common import cone_table_problem, set_interior_scaling, set_synthetic_state, sym_full


def _tables(cb):
    Z, N, S, P = cb.ZeroConeT, cb.NonnegativeConeT, cb.SecondOrderConeT, cb.PSDTriangleConeT
    return {
        "mixed": [Z(3), N(7), S(2), S(3), S(4), S(5), P(1), P(8), N(1), S(4), P(3), S(6), P(8), S(300)],
        "nonsym": [N(2), cb.ExponentialConeT(), S(5), cb.PowerConeT(0.3), P(3), cb.GenPowerConeT([0.3, 0.7], 2),
                   S(3), Z(2), cb.ExponentialConeT()],
    }


def _oracle(cb, P, A, cones, **st):
    from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
    o = OracleDirectLDLKKTSolver(P, A, cones, cones.numel, P.shape[0], cb.Settings(**st))
    o.update(cones)
    return o


@pytest.mark.parametrize("table", ["mixed", "nonsym"])
@pytest.mark.parametrize("state", ["interior", "synthetic"])
def test_cone_entries_match_oracle(cb, table, state):
    P, A, cones = cone_table_problem(cb, _tables(cb)[table], n=8, seed=1)
    set_interior_scaling(cones, seed=3)
    if state == "synthetic":
        set_synthetic_state(cones, seed=4)
    o = _oracle(cb, P, A, cones)
    pos, ref = kr.cone_entries(cones, o.map)
    nz = o.KKT.data
    assert kr.within_ulps(nz[pos], ref, 8).all()
    # every Zero / NN / SOC entry of the maps is covered once
    C = cb.cones
    want = [o.map.Hsblocks[cones.rng_blocks[i]:cones.rng_blocks[i + 1]] for i, t in enumerate(cones.types)
            if t in (C.ZERO, C.NONNEG, C.SOC)]
    want = np.concatenate(want + [o.map.soc_u, o.map.soc_v, o.map.soc_D])
    assert np.array_equal(np.sort(pos), np.sort(want))
    for i, n, blk, R in kr.psd_cones(cones, o.map):
        off, v, bnd = kr.psd_columns(R, np.arange(n * (n + 1) // 2))
        assert np.array_equal(np.sort(off), np.arange(len(blk)))
        assert (np.abs(nz[blk[off]].astype(kr.LD) - v) <= bnd).all()
        if n > 1:       # an index error is far outside the bound
            assert not (np.abs(np.roll(nz[blk[off]], 1).astype(kr.LD) - v) <= bnd).all()


@pytest.mark.parametrize("n", [1, 2, 3, 5, 9])
def test_skron_columns_match_oracle(n):
    from oracle.kktsolver_oracle import skron_triu
    rng = np.random.default_rng(n)
    M = rng.standard_normal((n, n)); A = M @ M.T
    ne = n * (n + 1) // 2
    H = skron_triu(A)
    ti, tj = np.tril_indices(ne)
    packed = H[tj, ti]
    cols = np.arange(ne)[::2] if ne > 2 else np.arange(ne)
    off, v = kr.skron_columns(A.astype(kr.LD), cols)
    assert np.allclose(packed[off], v.astype(float), rtol=1e-14, atol=1e-14 * np.abs(H).max())


def test_psd_check_columns_cover_both_ends():
    rng = np.random.default_rng(0)
    assert np.array_equal(kr.psd_check_columns(1275, rng), np.arange(1275))
    c = kr.psd_check_columns(5050, rng)
    assert c[0] == 0 and c[-1] == 5049 and len(c) == 32 + 96 + 32 and np.all(np.diff(c) > 0)


def test_static_eps_matches_oracle(cb):
    P, A, cones = cone_table_problem(cb, _tables(cb)["mixed"], n=8, seed=1)
    set_interior_scaling(cones, seed=5)
    o = _oracle(cb, P, A, cones, static_regularization_constant=1e-3, static_regularization_proportional=1e-6)
    assert kr.static_eps(o.KKT.data, o.map.diag_full, 1e-3, 1e-6) == o.diagonal_regularizer


def test_residual_reference(cb):
    P, A, cones = cone_table_problem(cb, _tables(cb)["mixed"], n=8, seed=1)
    set_interior_scaling(cones, seed=6)
    o = _oracle(cb, P, A, cones)
    K = o.KKT
    N = K.shape[0]
    rng = np.random.default_rng(7)
    x, b = rng.standard_normal(N), rng.standard_normal(N)
    e, bnd = kr.residual(K, x, b)
    e64 = b - o._sym_mul(x)
    assert (np.abs(e64.astype(kr.LD) - e) <= bnd).all()
    # exact on integers: e == 0 for b = K x
    Ki = K.copy(); Ki.data = rng.integers(-5, 5, K.nnz).astype(float)
    xi = rng.integers(-5, 5, N).astype(float)
    e0, _ = kr.residual(Ki, xi, kr.sym_matvec(Ki, xi).astype(float))
    assert not e0.any()


@pytest.mark.parametrize("eps", [0.0, 1e-3])
def test_longdouble_solver(cb, eps):
    from clarabel_jl_b200 import lib
    # no Zero cone: K itself is quasidefinite, so no pivot needs the dynamic regularisation at eps = 0
    specs = [cb.NonnegativeConeT(7), cb.SecondOrderConeT(3), cb.SecondOrderConeT(6), cb.PSDTriangleConeT(3),
             cb.PSDTriangleConeT(8)]
    P, A, cones = cone_table_problem(cb, specs, n=8, seed=1)
    set_interior_scaling(cones, seed=8)
    o = _oracle(cb, P, A, cones)
    K, Ds = o.KKT, o.Dsigns
    perm = lib.Symbolic(K).arrays()["perm"]
    ref = kr.LDSolver(K, Ds, perm, eps=eps)
    assert ref.nreg == 0 and np.all(np.sign(ref.D.astype(float)) == Ds[perm])
    Ks = K.copy(); Ks.data = kr.shifted_values(K.data, o.map.diag_full, Ds, eps)
    b = np.random.default_rng(9).standard_normal(K.shape[0])
    x = ref.solve(b)
    r = np.asarray(b, dtype=kr.LD) - kr.sym_matvec(Ks, x)
    assert float(np.abs(r).max()) < 1e-15 * float(np.abs(x).max())
    xs = spla.spsolve(sym_full(Ks).tocsc(), b)
    assert np.abs(xs - x.astype(float)).max() < 1e-9 * np.abs(xs).max()
