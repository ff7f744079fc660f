"""GPU tests of the multi-right-hand-side entry points (cb200_solve_multi, cb200_solve_ir_multi): every column
bitwise equal to the single-RHS solve of that column, on every solve kernel path of the front zoo and on the
big-front chains, with refinement, in resident mode, and the usage errors."""
import ctypes as C
import numpy as np
import pytest
import scipy.sparse as sp
import front_zoo as fz
import test_gpu_big_solve as tbs
import test_gpu_kernels as tgk
from mf_numpy import MFNumpy

pytestmark = pytest.mark.gpu

SINGLE_GPU_VARIANTS = list(tgk.VARIANTS)          # every variant there runs on one GPU
NRHS = (1, 2, 3, 4, 5, 9)
SOLVE_CLASSES = {"fwd_leaf", "fwd_warp", "fwd_cta", "fwd_big_assemble", "fwd_big_tri", "fwd_big_gemv",
                 "bwd_leaf", "bwd_warp", "bwd_cta", "bwd_big_gemvT", "bwd_big_tri"}


def _columns(R, design, k):
    """k columns: the _rhs_set vectors (random, zero, unit vector at a 64-block edge, 1e+-8 spread) then random"""
    base = list(tgk._rhs_set(R, design).values())
    rng = np.random.default_rng(100 + k)
    N = len(R["sg"])
    cols = [base[i] if i < len(base) else rng.standard_normal(N) for i in range(k)]
    return np.asfortranarray(np.stack(cols, axis=1))


def _singles(h, B):
    X = np.zeros_like(B)
    for j in range(B.shape[1]):
        x = np.zeros(B.shape[0]); h.solve(x, np.ascontiguousarray(B[:, j])); X[:, j] = x
    return X


@pytest.mark.parametrize("part", list(tgk.PARTS))
@pytest.mark.parametrize("variant", SINGLE_GPU_VARIANTS)
def test_multi_solve_matches_single_bitwise(monkeypatch, variant, part):
    env = tgk.VARIANTS[variant]
    tgk._set_env(monkeypatch, env)
    d = tgk.PARTS[part]
    R = tgk.reference(d, env)
    h = tgk._handle(R["K"], R["sg"])
    assert h.refactor()
    subtree = env.get("CB200_SUBTREE") == "1"
    w = d.scale
    ncols = 0
    for k in NRHS:
        B = _columns(R, d, k)
        X = np.zeros_like(B)
        h.solve_multi(X, B)
        ncols += k
        assert np.array_equal(X, _singles(h, B)), k
        for j in range(k):
            xr = R["mf"].solve(B[:, j]).astype(float)
            if not np.any(B[:, j]):
                assert np.all(X[:, j] == 0)
            else:
                assert np.abs(w * (X[:, j] - xr)).max() <= 1e-12 * np.abs(w * xr).max(), (k, j)
    st = h.stats()
    if subtree:
        assert st["multi_percol"] == ncols and st["multi_sweeps"] == 0
    else:
        assert st["multi_sweeps"] > 0 and st["multi_percol"] == 0


def test_big_chains_multi(monkeypatch):
    d = tbs.design_chains()
    K, sg, a, h = tbs._setup(monkeypatch, d, use_cuda_graph=1)
    N = K.shape[0]
    rng = np.random.default_rng(31)
    B = np.asfortranarray(rng.standard_normal((N, 9)))
    X = np.zeros_like(B); h.solve_multi(X, B)                 # captures the width-4 and width-1 graphs
    assert np.array_equal(X, _singles(h, B))
    for _ in range(5):                                        # graph replays
        X2 = np.zeros_like(B); h.solve_multi(X2, B)
        assert np.array_equal(X2, X)
    _, _, _, h0 = tbs._setup(monkeypatch, d, use_cuda_graph=0)
    X0 = np.zeros_like(B); h0.solve_multi(X0, B)
    assert np.array_equal(X0, X)
    mf = MFNumpy(a, np.longdouble); mf.factor(K.data, sg)
    for j in range(B.shape[1]):
        xr = mf.solve(B[:, j]).astype(float)
        assert np.abs(X[:, j] - xr).max() <= 1e-12 * np.abs(xr).max()


def test_multi_launches_per_sweep(monkeypatch):
    d = tbs.design_chains()
    K, _, _, h = tbs._setup(monkeypatch, d, {"CB200_GRAPH": "0"})
    N = K.shape[0]
    counts = []
    for k in (1, 4):
        B = np.asfortranarray(np.ones((N, k)))
        n0 = h.timers()["nlaunch"]
        X = np.zeros_like(B); h.solve_multi(X, B)
        counts.append(h.timers()["nlaunch"] - n0)
    assert counts[0] == counts[1], counts
    s0 = h.stats()["multi_sweeps"]
    B = np.asfortranarray(np.ones((N, 9)))
    X = np.zeros_like(B); h.solve_multi(X, B)
    assert h.stats()["multi_sweeps"] - s0 == 3


def test_multi_reaches_every_solve_class(monkeypatch):
    env = tgk.VARIANTS["default"]
    tgk._set_env(monkeypatch, env)
    seen = set()
    for name in tgk.PARTS:
        R = tgk.reference(tgk.PARTS[name], env)
        h = tgk._handle(R["K"], R["sg"])
        h.set_detail(2)
        assert h.refactor()
        h.reset_timers()
        B = _columns(R, tgk.PARTS[name], 4)
        X = np.zeros_like(B); h.solve_multi(X, B)
        assert h.stats()["multi_sweeps"] == 1
        seen |= {k for k, v in h.fine_timers().items() if v > 0}
    assert SOLVE_CLASSES <= seen, sorted(SOLVE_CLASSES - seen)


def _cta_tail_parts():
    """zoo parts with CTA-class solve fronts whose last 64-block is partial (ns not a multiple of 64)"""
    env = tgk.VARIANTS["default"]
    out = []
    for name, d in tgk.PARTS.items():
        R = tgk.reference(d, env)
        if any(f["solve"] == "cta" and f["ns"] % 64 for f in R["fronts"]):
            out.append(name)
    return out


def test_nan_column_does_not_leak_into_later_chunks(monkeypatch):
    """A NaN column in the first 4-column sweep, valid columns in the later ones: every column equals its
    single solve (NaN where that is NaN), on the fronts whose CTA solve has a partial last block"""
    env = tgk.VARIANTS["default"]
    tgk._set_env(monkeypatch, env)
    parts = _cta_tail_parts()
    assert parts
    for name in parts:
        d = tgk.PARTS[name]
        R = tgk.reference(d, env)
        h = tgk._handle(R["K"], R["sg"])
        assert h.refactor()
        B = _columns(R, d, 9)
        B[::7, 0] = np.nan
        B[3, 2] = np.inf
        for _ in range(3):
            X = np.zeros_like(B); h.solve_multi(X, B)
            assert np.array_equal(X, _singles(h, B), equal_nan=True), name
            assert np.all(np.isfinite(X[:, [1] + list(range(3, 9))])), name


def _kkt_qp(cb, n, m, dense_row, iters, seed, **over):
    from clarabel_jl_b200.kktsolver_b200 import B200KKTSolver
    rng = np.random.default_rng(seed)
    P = sp.diags(1.0 + rng.random(n), format="csc")
    A = sp.random(m - 1, n, 0.05 if n < 500 else 0.01, random_state=np.random.RandomState(seed), format="csr")
    first = np.ones((1, n)) if dense_row else sp.random(1, n, 0.2, random_state=np.random.RandomState(seed + 1)).toarray()
    A = sp.vstack([sp.csr_matrix(first), A]).tocsc()
    q = rng.standard_normal(n); b = np.ones(m)
    s = cb.Solver(P, q, A, b, [cb.cones.NonnegativeConeT(m)], cb.Settings(direct_solve_method="qdldl"))
    s.solve(max_iter=iters)
    data, cones, st = s.data, s.cones, s.settings
    gpu = B200KKTSolver(data.P, data.A, cones, data.m, data.n, st, **over)
    assert gpu.update(cones)
    return gpu, cones, rng


def _ir_columns(gpu, rng, k):
    n, m = gpu.n, gpu.m
    RX = np.zeros((n, k), order="F"); RZ = np.zeros((m, k), order="F")
    for j in range(k):
        if j == 1:
            continue                                          # a zero system: no refinement round
        sc = 10.0 ** rng.uniform(-6, 6)
        RX[:, j] = sc * rng.standard_normal(n); RZ[:, j] = sc * rng.standard_normal(m)
    return RX, RZ


def _single_ir(gpu, RX, RZ):
    k = RX.shape[1]
    LX = np.zeros_like(RX); LZ = np.zeros_like(RZ); ok = np.zeros(k, bool); rounds = np.zeros(k, int)
    for j in range(k):
        x, z = np.zeros(gpu.n), np.zeros(gpu.m)
        r0 = gpu.ir_rounds
        gpu.setrhs(RX[:, j], RZ[:, j]); ok[j] = gpu.solve(x, z)
        rounds[j] = gpu.ir_rounds - r0
        LX[:, j] = x; LZ[:, j] = z
    return LX, LZ, ok, rounds


@pytest.mark.parametrize("instance", ["qp_late_iterate", "long_row"])
def test_refinement_multi_matches_single(cb, instance):
    if instance == "long_row":
        gpu, _, rng = _kkt_qp(cb, 2100, 40, True, 2, 17)
    else:
        gpu, _, rng = _kkt_qp(cb, 60, 40, False, 12, 5)
    for k in (2, 5, 9):
        RX, RZ = _ir_columns(gpu, rng, k)
        LX, LZ, ok1, r1 = _single_ir(gpu, RX, RZ)
        MX = np.zeros_like(RX, order="F"); MZ = np.zeros_like(RZ, order="F")
        ok, rounds = gpu.solve_multi(RX, RZ, MX, MZ)
        assert np.all(ok) and np.all(ok1)
        assert np.array_equal(rounds, r1), (rounds, r1)
        assert np.array_equal(MX, LX) and np.array_equal(MZ, LZ)
    # a NaN right-hand side fails alone, also for the columns of the later sweeps of the same call
    k = 9
    RX, RZ = _ir_columns(gpu, rng, k)
    RX[3, 2] = np.nan
    LX, LZ, _, r1 = _single_ir(gpu, RX, RZ)
    MX = np.zeros_like(RX, order="F"); MZ = np.zeros_like(RZ, order="F")
    rounds = np.zeros(k, np.int32); status = np.zeros(k, np.int32)
    rc = gpu.ldl._L.cb200_solve_ir_multi(gpu.ldl._h, k, RX.ctypes.data, RZ.ctypes.data, MX.ctypes.data,
                                         MZ.ctypes.data, rounds.ctypes.data, status.ctypes.data)
    assert rc == 1 and status.tolist() == [0, 0, 1] + [0] * (k - 3)
    assert np.all(np.isnan(MX[:, 2])) and np.all(np.isnan(MZ[:, 2]))
    for j in [0, 1] + list(range(3, k)):
        assert np.array_equal(MX[:, j], LX[:, j]) and np.array_equal(MZ[:, j], LZ[:, j]) and rounds[j] == r1[j]


def test_refinement_columns_stop_after_different_rounds(cb):
    """With the tolerances at zero and a stop ratio of 1 every column refines until its residual grows,
    which happens at the rounding-noise floor after a different number of rounds per column: the
    per-column keep / replace of the iterate (k_select_cols) is exercised between two active columns."""
    gpu, _, rng = _kkt_qp(cb, 60, 40, False, 12, 5, iterative_refinement_reltol=0.0,
                          iterative_refinement_abstol=0.0, iterative_refinement_stop_ratio=1.0)
    k = 16
    RX, RZ = _ir_columns(gpu, rng, k)
    RX[:, 1] = rng.standard_normal(gpu.n); RZ[:, 1] = rng.standard_normal(gpu.m)
    LX, LZ, ok1, r1 = _single_ir(gpu, RX, RZ)
    MX = np.zeros_like(RX, order="F"); MZ = np.zeros_like(RZ, order="F")
    ok, rounds = gpu.solve_multi(RX, RZ, MX, MZ)
    assert np.all(ok) and np.all(ok1)
    assert np.array_equal(rounds, r1), (rounds, r1)
    assert np.array_equal(MX, LX) and np.array_equal(MZ, LZ)
    nonzero = set(int(r) for r in rounds if r > 0)
    assert len(nonzero) > 1, rounds.tolist()


def test_resident_multi_and_single_state(cb):
    import torch
    gpu, _, rng = _kkt_qp(cb, 60, 40, False, 12, 7)
    n, m, N, k = gpu.n, gpu.m, gpu.KKT.shape[0], 5
    RX, RZ = _ir_columns(gpu, rng, k)
    MX = np.zeros_like(RX, order="F"); MZ = np.zeros_like(RZ, order="F")
    ok, rounds = gpu.solve_multi(RX, RZ, MX, MZ)
    assert np.all(ok)
    full = gpu.ldl.download(8, N * k).reshape(k, N).T
    assert np.array_equal(full[:n], MX) and np.array_equal(full[n:n + m], MZ)
    # a single-RHS solve after a multi call still solves what setrhs stored
    rx0, rz0 = rng.standard_normal(n), rng.standard_normal(m)
    gpu.setrhs(rx0, rz0)
    x0, z0 = np.zeros(n), np.zeros(m); assert gpu.solve(x0, z0)
    sol0 = gpu.ldl.download(6, N)
    gpu.solve_multi(RX, RZ, MX, MZ)
    assert np.array_equal(gpu.ldl.download(6, N), sol0)
    x1, z1 = np.zeros(n), np.zeros(m); assert gpu.solve(x1, z1)
    assert np.array_equal(x1, x0) and np.array_equal(z1, z0)
    # resident: device pointers in, results through selector 8
    gpu.ldl.set_resident(True)
    tx = torch.tensor(RX.T.copy(), device="cuda")             # C-order k x n == column-major n x k
    tz = torch.tensor(RZ.T.copy(), device="cuda")
    torch.cuda.synchronize()
    ok_r, rounds_r = gpu.solve_multi_staged(tx.data_ptr(), tz.data_ptr(), k)
    assert np.all(ok_r) and np.array_equal(rounds_r, rounds)
    assert np.array_equal(gpu.ldl.download(8, N * k).reshape(k, N).T, full)
    gpu.ldl.set_resident(False)


def test_multi_usage_errors(cb):
    from clarabel_jl_b200 import lib
    gpu, _, _ = _kkt_qp(cb, 60, 40, False, 3, 9)
    L, h, N = gpu.ldl._L, gpu.ldl._h, gpu.KKT.shape[0]
    B = np.ones((N, 2), order="F"); X = np.zeros_like(B)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_multi(h, -1, ptr(X), N, ptr(B), N), "cb200_solve_multi")
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_multi(h, 2, ptr(X), N - 1, ptr(B), N), "cb200_solve_multi")
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_multi(h, 2, ptr(X), N, ptr(B), N - 1), "cb200_solve_multi")
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_multi(h, 2, ptr(X), N, None, N), "cb200_solve_multi")
    assert lib.check(L.cb200_solve_multi(h, 0, None, N, None, N), "cb200_solve_multi")
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_ir_multi(h, -1, None, None, None, None, None, None), "cb200_solve_ir_multi")
    with pytest.raises(RuntimeError):
        lib.check(L.cb200_solve_ir_multi(h, 2, None, None, None, None, None, None), "cb200_solve_ir_multi")
    assert lib.check(L.cb200_solve_ir_multi(h, 0, None, None, None, None, None, None), "cb200_solve_ir_multi")
    d = tbs.design_root(64)
    K, sg, _ = d.build()
    from clarabel_jl_b200.kktsolver_b200 import B200DirectLDLSolver
    h2 = B200DirectLDLSolver(K, sg, None, ordering=2)
    rx = np.ones((K.shape[0], 1))
    with pytest.raises(RuntimeError):                         # cb200_set_maps not called
        lib.check(h2._L.cb200_solve_ir_multi(h2._h, 1, ptr(rx), ptr(rx), None, None, None, None), "cb200_solve_ir_multi")
