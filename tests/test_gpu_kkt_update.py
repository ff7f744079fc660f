"""GPU tests (run with -m gpu on an H100) of what runs around the factorisation in every interior-point
iteration, against the extended-precision references of kkt_reference.py:

  * the cone-block kernels (G1 k_hs_diag / k_hs_soc_dense / k_soc_expansion / k_soc_D, G2 k_psd_rrt /
    k_psd_skron) on designed cone tables, with every cone-owned K entry poisoned with NaN before the
    update so that an entry a kernel fails to write cannot pass on the previous iteration's value;
  * the static regularisation (G3 k_diag_absmax / k_compute_eps / k_shift_diag) through eps (selector 4),
    the pivots D (selector 1) and unrefined solves against a longdouble LDL' of K + eps diag(Dsigns);
  * the refinement residual (G8 k_residual<RL>, k_residual_long and their multi-column forms) through
    selector 9, and each exit of the refinement loop.

Bounds.  Zero / NN / SOC entries: bitwise the oracle's and within 8 ulps of the longdouble formula.
PSD entries: 4 (n + 2) eps (|R||R|' (x)_s |R||R|') entrywise.  Residuals: (len_i + 2) eps (|b_i| +
sum_j |K_ij| |x_j|) per row."""
import numpy as np
import pytest
import kkt_reference as kr
from common import cone_table_problem, set_interior_scaling, set_synthetic_state

pytestmark = pytest.mark.gpu


def _table(cb, name):
    Z, N, S, P = cb.ZeroConeT, cb.NonnegativeConeT, cb.SecondOrderConeT, cb.PSDTriangleConeT
    return {
        # every G1 branch: Zero, NN, dense SOC 2/3/4, expanded SOC 5+, unsorted, repeated PSD sides apart
        "mixed": [Z(3), N(7), S(2), S(3), S(4), S(5), P(1), P(8), N(1), S(4), P(3), S(6), P(8), S(3000)],
        # exp / pow / genpow values arrive through cb200_update_values
        "nonsym": [N(2), cb.ExponentialConeT(), S(5), cb.PowerConeT(0.3), P(3), cb.GenPowerConeT([0.3, 0.7], 2),
                   S(3), Z(2), cb.ExponentialConeT()],
        # skron: side 1, the 512-entry grid-stride wrap (ne > 512 from side 32), the old 48 KB staging
        # boundary (78 / 79) and side 100
        "skron_sides": [P(1), P(2), P(3), P(31), P(32), P(33), P(50), P(78), P(79), P(100)],
        # one launch over ragged sides: the grid is sized by the largest cone
        "ragged": [P(1), P(50), P(2), P(33)],
    }[name]


def _owned(mp):
    return np.concatenate([mp.Hsblocks, mp.soc_u, mp.soc_v, mp.soc_D, mp.gp_q, mp.gp_r, mp.gp_p, mp.gp_D])


def _solver(cb, P, A, cones, **cs):
    from clarabel_jl_b200.kktsolver_b200 import B200KKTSolver
    return B200KKTSolver(P, A, cones, cones.numel, P.shape[0], cb.Settings(), **cs)


def _poisoned_update(gpu, cones):
    own = _owned(gpu.map)
    gpu.ldl.update_values(own, np.full(len(own), np.nan))
    assert np.isnan(gpu.device_nzval()[own]).all()
    gpu.update(cones)
    return gpu.device_nzval()


def _check_cone_blocks(cones, gpu, nz, rng, oracle_nz=None):
    from clarabel_jl_b200.kktsolver_b200 import nonsym_update_values
    mp = gpu.map
    own = np.zeros(len(nz), dtype=bool); own[_owned(mp)] = True
    assert not np.isnan(nz).any(), np.nonzero(np.isnan(nz))[0][:10]
    # P, A and the structural zeros: bitwise what the host assembled
    assert np.array_equal(nz[~own], gpu.KKT.data[~own])
    pos, ref = kr.cone_entries(cones, mp)
    ok = kr.within_ulps(nz[pos], ref, 8)
    assert ok.all(), (pos[~ok][:5], nz[pos][~ok][:5], ref[~ok][:5])
    if oracle_nz is not None:
        assert np.array_equal(nz[pos], oracle_nz[pos])
    if cones.nonsym:
        assert np.array_equal(nz[gpu._ns_idx], nonsym_update_values(mp, cones))
    for i, n, blk, R in kr.psd_cones(cones, mp):
        cols = kr.psd_check_columns(n * (n + 1) // 2, rng)
        off, ref, bnd = kr.psd_columns(R, cols)
        err = np.abs(nz[blk[off]].astype(kr.LD) - ref)
        bad = ~(err <= bnd)
        assert not bad.any(), (i, n, off[bad][:5], nz[blk[off]][bad][:5], ref[bad][:5])


@pytest.mark.parametrize("table", ["mixed", "nonsym", "skron_sides", "ragged"])
def test_cone_blocks_against_longdouble(cb, table):
    from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
    P, A, cones = cone_table_problem(cb, _table(cb, table), n=8, seed=1)
    gpu = _solver(cb, P, A, cones)
    rng = np.random.default_rng(2)
    # an interior-point state, then a synthetic one spanning 1e+-8 on the same handle
    for state in ("interior", "synthetic"):
        set_interior_scaling(cones, seed=3)
        if state == "synthetic":
            set_synthetic_state(cones, seed=4)
        nz = _poisoned_update(gpu, cones)
        oracle_nz = None
        if table in ("mixed", "nonsym"):
            oracle = OracleDirectLDLKKTSolver(P, A, cones, cones.numel, P.shape[0], cb.Settings())
            oracle.update(cones)
            oracle_nz = oracle.KKT.data
        _check_cone_blocks(cones, gpu, nz, rng, oracle_nz)


def test_psd_side_171(cb):
    """A PSD cone of side 171 needs 8 * 171^2 = 233,928 bytes for A = RR', more than one block's shared
    memory on an H100 (232,448): skron reads A through the cache, so the handle sets up and updates."""
    P, A, cones = cone_table_problem(cb, [cb.NonnegativeConeT(2), cb.PSDTriangleConeT(171)], n=8, seed=5)
    gpu = _solver(cb, P, A, cones)
    set_interior_scaling(cones, seed=6)
    nz = _poisoned_update(gpu, cones)
    _check_cone_blocks(cones, gpu, nz, np.random.default_rng(7))


# ------------------------------------------------------------------ static regularisation
def _reg_instance(cb, where):
    """[NN(3), SOC(6), PSD(3)] with n = 6 at an interior state, with max|diag K| moved onto `where`."""
    P, A, cones = cone_table_problem(cb, [cb.NonnegativeConeT(3), cb.SecondOrderConeT(6), cb.PSDTriangleConeT(3)],
                                     n=6, seed=8)
    set_interior_scaling(cones, seed=9)
    if where == "P":
        P = P.copy(); P.data[2] = 1e4
    elif where == "NN":
        cones.w[cones.nn_idx[1]] = 100.0
    elif where == "SOC_D":
        cones.soc_eta[0] = 100.0             # eta^2 on the SOC diagonal and on D = (-eta^2, +eta^2)
    elif where == "PSD":
        cones.psd_groups[0]["R"][0] *= 10.0
    return P, A, cones


def _check_factor(gpu, nz, eps, rng):
    """D (selector 1) and an unrefined cb200_solve against the longdouble factor of K + eps diag(Dsigns)
    in the device's elimination order."""
    N = gpu.KKT.shape[0]
    K = gpu.KKT.copy(); K.data = nz.copy()
    perm = gpu.ldl.download(3, N).astype(np.int64)
    ref = kr.LDSolver(K, gpu.Dsigns, perm, eps=eps)
    D = gpu.ldl.download(1, N)
    assert np.all(np.abs(D - ref.D.astype(float)) <= 1e-12 * np.abs(ref.D.astype(float)))
    b = rng.standard_normal(N)
    x = np.zeros(N); gpu.ldl.solve(x, b)
    xr = ref.solve(b)
    assert np.abs(x - xr).max() <= 1e-12 * float(np.abs(xr).max())


@pytest.mark.parametrize("where", ["P", "NN", "SOC_D", "PSD"])
def test_static_regularisation_against_longdouble(cb, where):
    c, p = 1e-3, 1e-6
    P, A, cones = _reg_instance(cb, where)
    gpu = _solver(cb, P, A, cones, static_regularization_constant=c, static_regularization_proportional=p)
    assert gpu.update(cones)
    nz = gpu.device_nzval()
    diag = gpu.map.diag_full
    loc = {"P": gpu.map.diagP, "NN": diag[P.shape[0] + cones.nn_idx], "SOC_D": gpu.map.soc_D,
           "PSD": diag[P.shape[0] + cones.psd_groups[0]["idx"][0]]}[where]
    assert np.abs(nz[loc]).max() == np.abs(nz[diag]).max()
    eps = gpu.ldl.download(4, 1)[0]
    assert eps == kr.static_eps(nz, diag, c, p)
    assert eps > 1e-3
    _check_factor(gpu, nz, eps, np.random.default_rng(10))


def test_static_regularisation_disabled(cb):
    P, A, cones = _reg_instance(cb, "NN")
    gpu = _solver(cb, P, A, cones, static_regularization_enable=0)
    assert gpu.update(cones)
    _check_factor(gpu, gpu.device_nzval(), 0.0, np.random.default_rng(11))


def test_regularised_and_plain_factor_graphs_on_one_handle(cb):
    """update_cones (shifted) -> refactor (unshifted) -> update_cones: two captured factorisation graphs,
    each call against its own reference."""
    c, p = 1e-3, 1e-6
    P, A, cones = _reg_instance(cb, "PSD")
    gpu = _solver(cb, P, A, cones, static_regularization_constant=c, static_regularization_proportional=p,
                  use_cuda_graph=3)
    rng = np.random.default_rng(12)
    for step in ("update", "refactor", "update"):
        if step == "update":
            assert gpu.update(cones)
            nz = gpu.device_nzval()
            eps = gpu.ldl.download(4, 1)[0]
            assert eps == kr.static_eps(nz, gpu.map.diag_full, c, p)
        else:
            assert gpu.ldl.refactor()
            nz, eps = gpu.device_nzval(), 0.0
        _check_factor(gpu, nz, eps, rng)
    assert gpu.ldl.stats()["factor_graphs"] == 2


# ------------------------------------------------------------------ residuals
def _mean_row(K):
    return 2.0 * K.nnz / K.shape[0]


def _residual_instance(cb, name):
    Nn, Pp = cb.NonnegativeConeT, cb.PSDTriangleConeT
    if name == "mean_row_below_48":                  # k_residual<4>
        return cone_table_problem(cb, [Pp(9)], n=5, seed=13)
    if name == "mean_row_above_48":                  # k_residual<32>
        return cone_table_problem(cb, [Pp(10)], n=5, seed=14)
    if name == "rows_2048_2049":                     # K rows of exactly 2048 and 2049 entries (CSC part)
        n, m = 2048, 37
        D = np.zeros((m, n)); D[0, :] = 1e-2; D[1, 1:] = -1e-2
        return cone_table_problem(cb, [Nn(m)], n=n, seed=15, extra_A=D)
    if name == "dense_column":                       # a K row of 2101+ entries held in the row-wise part
        n, m = 7, 2100
        D = np.zeros((m, n)); D[:, 0] = 1e-2
        return cone_table_problem(cb, [Nn(m)], n=n, seed=16, extra_A=D)


RESIDUAL_INSTANCES = ["mean_row_below_48", "mean_row_above_48", "rows_2048_2049", "dense_column"]


def _residual_solver(cb, name, **cs):
    P, A, cones = _residual_instance(cb, name)
    gpu = _solver(cb, P, A, cones, **cs)
    set_interior_scaling(cones, seed=17)
    assert gpu.update(cones)
    K = gpu.KKT.copy(); K.data = gpu.device_nzval()
    N = K.shape[0]
    lens = kr.row_lengths(K)
    if name == "mean_row_below_48":
        assert _mean_row(K) < 48 and N % 64
    elif name == "mean_row_above_48":
        assert _mean_row(K) > 48 and N % 8
    elif name == "rows_2048_2049":
        assert {2048, 2049} <= set(lens.tolist()) and N % 64
    else:
        assert lens.max() > 2048 and N % 64
    return gpu, K


@pytest.mark.parametrize("name", RESIDUAL_INSTANCES)
def test_residual_against_longdouble(cb, name):
    gpu, K = _residual_solver(cb, name, iterative_refinement_max_iter=0)
    N, n, m = K.shape[0], gpu.n, gpu.m
    rng = np.random.default_rng(18)
    for _ in range(2):
        rx, rz = rng.standard_normal(n), rng.standard_normal(m)
        gpu.setrhs(rx, rz)
        assert gpu.solve(np.zeros(n), np.zeros(m))
        x0, e = gpu.ldl.download(6, N), gpu.ldl.download(9, N)
        b = np.r_[rx, rz, np.zeros(N - n - m)]
        eref, bnd = kr.residual(K, x0, b)
        err = np.abs(e.astype(kr.LD) - eref)
        assert (err <= bnd).all(), (np.nonzero(err > bnd)[0][:5])
        assert np.abs(e).max() > 0


def _single(gpu, RX, RZ):
    k = RX.shape[1]
    LX, LZ = np.full_like(RX, 7.0), np.full_like(RZ, 7.0)
    ok, rounds = np.zeros(k, bool), np.zeros(k, np.int32)
    for j in range(k):
        x, z = np.zeros(gpu.n), np.zeros(gpu.m)
        gpu.setrhs(RX[:, j].copy(), RZ[:, j].copy())
        r0 = gpu.ir_rounds
        ok[j] = gpu.solve(x, z)
        rounds[j] = gpu.ir_rounds - r0
        LX[:, j], LZ[:, j] = x, z
        if not ok[j]:
            LX[:, j] = np.nan; LZ[:, j] = np.nan
    return LX, LZ, ok, rounds


@pytest.mark.parametrize("name", RESIDUAL_INSTANCES)
def test_residual_multi_matches_single(cb, name):
    gpu, _ = _residual_solver(cb, name)
    rng = np.random.default_rng(19)
    for k in (1, 2, 3, 4, 5, 9):
        RX = np.asfortranarray(rng.standard_normal((gpu.n, k)))
        RZ = np.asfortranarray(rng.standard_normal((gpu.m, k)))
        if k >= 3:
            RX[0, k - 2] = np.nan if k % 2 else np.inf
        LX, LZ, ok1, r1 = _single(gpu, RX, RZ)
        MX = np.zeros_like(RX, order="F"); MZ = np.zeros_like(RZ, order="F")
        ok, rounds = gpu.solve_multi(RX, RZ, MX, MZ)
        assert np.array_equal(ok, ok1) and np.array_equal(rounds, r1)
        bad = [k - 2] if k >= 3 else []
        assert [j for j in range(k) if not ok[j]] == bad
        for j in bad:
            assert np.isnan(MX[:, j]).all() and np.isnan(MZ[:, j]).all()
        good = [j for j in range(k) if j not in bad]
        assert np.array_equal(MX[:, good], LX[:, good]) and np.array_equal(MZ[:, good], LZ[:, good])


# ------------------------------------------------------------------ refinement loop exits
def _ir_instance(cb):
    return cone_table_problem(cb, [cb.NonnegativeConeT(20), cb.SecondOrderConeT(6), cb.PSDTriangleConeT(4)],
                              n=10, seed=20)


def _ir_solver(cb, **cs):
    P, A, cones = _ir_instance(cb)
    gpu = _solver(cb, P, A, cones, **cs)
    set_interior_scaling(cones, seed=21)
    assert gpu.update(cones)
    return gpu


def _full_solve(gpu, b):
    """setrhs + cb200_solve_ir on the full right-hand side b (zero on the expansion rows):
    (ok, rounds, x = selector 6, e = selector 9)."""
    n, m, N = gpu.n, gpu.m, gpu.KKT.shape[0]
    gpu.setrhs(b[:n].copy(), b[n:n + m].copy())
    r0 = gpu.ir_rounds
    ok = gpu.solve(np.zeros(n), np.zeros(m))
    return ok, gpu.ir_rounds - r0, gpu.ldl.download(6, N), gpu.ldl.download(9, N)


def _rhs(gpu, rng, k):
    N, n, m = gpu.KKT.shape[0], gpu.n, gpu.m
    out = []
    for j in range(k):
        b = np.zeros(N)
        b[:n + m] = rng.standard_normal(n + m) * 10.0 ** rng.uniform(-3, 3)
        out.append(b)
    return out


def test_refinement_exit_on_tolerance(cb):
    gpu = _ir_solver(cb, iterative_refinement_abstol=1e300)
    N = gpu.KKT.shape[0]
    for b in _rhs(gpu, np.random.default_rng(22), 3):
        ok, r, x, _ = _full_solve(gpu, b)
        assert ok and r == 0
        x1 = np.zeros(N); gpu.ldl.solve(x1, b)
        assert np.array_equal(x, x1)


def test_refinement_exit_on_max_iter(cb):
    gpu = _ir_solver(cb, iterative_refinement_abstol=0.0, iterative_refinement_reltol=0.0,
                     iterative_refinement_stop_ratio=0.0, iterative_refinement_max_iter=3)
    for b in _rhs(gpu, np.random.default_rng(23), 3):
        ok, r, _, e = _full_solve(gpu, b)
        assert ok and r == 3 and np.abs(e).max() > 0


def test_refinement_exit_on_stagnation_keeps_the_better_iterate(cb):
    """Tolerances 0 and the default stop ratio 5: each column refines until a round improves max|e| by
    less than 5x, at the rounding floor after r rounds.  The host replays that last decision from the
    residuals (selector 9) of x_{r-1} and x_r, which handles stopping after r - 1 and r rounds give:
    the returned x is bitwise x_r if the last round still reduced max|e| and x_{r-1} otherwise."""
    tol0 = dict(iterative_refinement_abstol=0.0, iterative_refinement_reltol=0.0)
    gpu = _ir_solver(cb, **tol0)
    fixed = {}

    def after(j, b):          # x_j and its residual: j rounds, every round accepted
        if j not in fixed:
            fixed[j] = _ir_solver(cb, **tol0, iterative_refinement_stop_ratio=0.0, iterative_refinement_max_iter=j)
        ok, r, x, e = _full_solve(fixed[j], b)
        assert ok and r == j
        return x, e

    branches = set()
    for b in _rhs(gpu, np.random.default_rng(24), 16):
        ok, r, x, e = _full_solve(gpu, b)
        assert ok and 1 <= r < 10
        x_prev, e_prev = after(r - 1, b)
        x_r, e_r = after(r, b)
        assert np.array_equal(e, e_r)
        ratio = np.abs(e_prev).max() / np.abs(e_r).max()
        assert ratio < 5.0
        assert np.array_equal(x, x_r if ratio > 1.0 else x_prev)
        branches.add(ratio > 1.0)
    assert branches == {True, False}


def test_refinement_disabled(cb):
    gpu = _ir_solver(cb, iterative_refinement_enable=0)
    N, n, m = gpu.KKT.shape[0], gpu.n, gpu.m
    b = _rhs(gpu, np.random.default_rng(25), 1)[0]
    ok, r, x, _ = _full_solve(gpu, b)
    x1 = np.zeros(N); gpu.ldl.solve(x1, b)
    assert ok and r == 0 and np.array_equal(x, x1)
    b[1] = np.nan
    lx, lz = np.zeros(n), np.zeros(m)
    gpu.setrhs(b[:n].copy(), b[n:n + m].copy())
    assert not gpu.solve(lx, lz)
    assert np.isnan(lx).all() and np.isnan(lz).all()


def test_refinement_removes_a_large_static_shift(cb):
    """static_regularization_constant = 1e-4: the unrefined solve is ~1e-4 off; the refined x meets the
    stop rule against the unshifted K in longdouble and matches the longdouble solve of K."""
    st = cb.Settings()
    gpu = _ir_solver(cb, static_regularization_constant=1e-4)
    K = gpu.KKT.copy(); K.data = gpu.device_nzval()
    N = K.shape[0]
    ref = kr.LDSolver(K, gpu.Dsigns, gpu.ldl.download(3, N).astype(np.int64), eps=0.0)
    for b in _rhs(gpu, np.random.default_rng(26), 3):
        ok, r, x, _ = _full_solve(gpu, b)
        assert ok and r >= 1
        xr = ref.solve(b).astype(float)
        x0 = np.zeros(N); gpu.ldl.solve(x0, b)
        scale = np.abs(xr).max()
        assert np.abs(x0 - xr).max() > 1e-7 * scale          # the shift is visible without refinement
        e, bnd = kr.residual(K, x, b)
        assert float(np.abs(e).max()) <= (st.iterative_refinement_abstol + st.iterative_refinement_reltol
                                          * np.abs(b).max() + float(bnd.max()))
        assert np.abs(x - xr).max() <= 1e-10 * scale
