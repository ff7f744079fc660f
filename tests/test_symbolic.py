"""CPU: the product's host-side symbolic analysis (ordering, supernodes, a_map / rel maps, level
sets) checked by running a numpy emulation of the multifrontal numeric phase on those maps and
comparing with the QDLDL oracle and scipy's SuperLU; plus the C-ABI export check."""
import ctypes
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl
import pytest
from common import small_instances, kkt_fixture, sym_full, random_quasidefinite
from mf_numpy import MFNumpy


def test_cabi_library_exports_every_declared_symbol():
    import re, os
    from clarabel_jl_b200 import lib
    L = lib.lib()
    hdr = open(os.path.join(os.path.dirname(lib.LIB_PATH), "..", "include", "clarabel_b200.h")).read()
    declared = set(re.findall(r"\b(cb200_[a-z_A-Z0-9]+)\s*\(", hdr))
    assert declared == set(lib.EXPORTED)
    for s in declared:
        assert hasattr(L, s), s


def test_no_cuda_device_fails_loudly(cb, gpu_available):
    if gpu_available:
        pytest.skip("GPU present")
    from clarabel_jl_b200.kktsolver_b200 import B200DirectLDLSolver
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)["C1s"])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        B200DirectLDLSolver(KKT, Ds, cb.Settings())


@pytest.mark.parametrize("name", ["C1s", "C2s", "C3s", "C4s", "C5s"])
@pytest.mark.parametrize("ordering", [0, 1])
def test_symbolic_maps_via_numpy_multifrontal(cb, name, ordering):
    from clarabel_jl_b200 import lib
    from oracle import qdldl as oq
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)[name])
    N = KKT.shape[0]
    S = lib.Symbolic(KKT, ordering=ordering, nd_leaf=32)
    a = S.arrays()
    assert sorted(a["perm"].tolist()) == list(range(N))
    # supernode partition and tree sanity
    assert a["sn_first"][0] == 0 and a["sn_first"][-1] == N and np.all(np.diff(a["sn_first"]) > 0)
    par = a["sn_parent"]
    assert np.all((par == -1) | (par > np.arange(len(par))))
    assert np.all(a["sn_level"][par[par >= 0]] > a["sn_level"][par >= 0])
    mf = MFNumpy(a)
    D = mf.factor(KKT.data, Ds)
    assert np.all(np.sign(D) == Ds[a["perm"]])          # quasidefinite => signs as expected
    rng = np.random.default_rng(1)
    b = rng.standard_normal(N)
    x = mf.solve(b)
    Kf = sym_full(KKT)
    assert np.abs(Kf @ x - b).max() < 1e-9 * max(1.0, np.abs(x).max())
    # same system through the QDLDL oracle and SuperLU
    F = oq.QDLDLFactorisation(KKT, Ds)
    assert F.refactor()
    xo = b.copy(); F.solve(xo)
    xs = spl.splu(Kf).solve(b)
    scale = max(1.0, np.abs(xs).max())
    assert np.abs(x - xo).max() < 1e-8 * scale and np.abs(xo - xs).max() < 1e-8 * scale
    # the factorisation's inertia matches between engines (no dynamic regularisation fired)
    assert mf.nreg == 0 and F.regularize_count == 0


def test_amd_and_nd_are_permutations_and_reduce_fill(cb):
    from oracle import qdldl as oq
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)["C3s"])
    N = KKT.shape[0]
    nat = oq.QDLDLFactorisation(KKT, Ds, perm=np.arange(N))
    for perm in (oq.amd_order(KKT), oq.nd_order(KKT, 1.5, 32)):
        assert sorted(perm.tolist()) == list(range(N))
        F = oq.QDLDLFactorisation(KKT, Ds, perm=perm)
        assert F.nnzL < nat.nnzL


def test_ordering_arbitration_rejects_bad_dissection(cb):
    """ordering=1 keeps nested dissection only when its factor cost is within 3x of the AMD-class
    ordering; on a factor-model (expander-like) KKT graph it must not be worse than AMD."""
    from clarabel_jl_b200 import lib
    KKT, mp, Ds, data, cones = kkt_fixture(cb, lambda: cb.problems.c2_portfolio(n=6000))
    amd = lib.Symbolic(KKT, ordering=0).stats
    auto = lib.Symbolic(KKT, ordering=1).stats
    assert auto["flops"] <= 3.0 * amd["flops"] * (1 + 1e-12)


def test_block_hint_keeps_cone_blocks_contiguous(cb):
    """cb200_hint_blocks: rows of a dense cone block may not be split by a separator, i.e. in the
    elimination order every block is contiguous up to the interleaving the leaf AMD does inside a
    leaf; here we only require a valid permutation and that the hint is consumed (one-shot)."""
    from clarabel_jl_b200 import lib
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)["C4s"])
    N = KKT.shape[0]
    bid = lib.cone_block_ids(cones, data.n, N)
    assert bid is not None and bid.max() == int((cones.types == cb.cones.PSD).sum()) - 1
    S1 = lib.Symbolic(KKT, ordering=1, nd_leaf=32, block_id=bid)
    assert sorted(S1.arrays()["perm"].tolist()) == list(range(N))
    S2 = lib.Symbolic(KKT, ordering=1, nd_leaf=32)            # hint must not leak into this call
    S3 = lib.Symbolic(KKT, ordering=1, nd_leaf=32)
    assert np.array_equal(S2.arrays()["perm"], S3.arrays()["perm"])


def test_partition_api_shapes(cb):
    from clarabel_jl_b200 import lib
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)["C3s"])
    S = lib.Symbolic(KKT)
    owner, top, load = S.partition(4)
    assert len(owner) == S.stats["nsuper"] and top.dtype == bool and len(load) == 4
    assert abs(load.sum() - load.sum()) == 0 and (load >= 0).all()


def test_nd_result_independent_of_host_threads(monkeypatch):
    """Disjoint pieces of the dissection are ordered on separate host threads (CB200_ND_THREADS);
    the permutation must not depend on the thread budget.  A 2-D grid is large enough for both
    halves of the first separators to get a thread each."""
    import ctypes as C
    import scipy.sparse as sp
    from clarabel_jl_b200 import lib
    g = 260
    I = sp.identity(g, format="csc")
    T = sp.diags([np.ones(g - 1)], [1], shape=(g, g), format="csc")
    K = sp.triu(sp.kron(I, T) + sp.kron(T, I) + sp.identity(g * g), format="csc")
    n = K.shape[0]
    cp = np.ascontiguousarray(K.indptr, dtype=np.int64); ri = np.ascontiguousarray(K.indices, dtype=np.int64)
    perms = []
    for th in ("1", "4"):
        monkeypatch.setenv("CB200_ND_THREADS", th)
        perm = np.empty(n, dtype=np.int64)
        rc = lib.lib().cb200_order_nd(n, cp.ctypes.data_as(C.c_void_p), ri.ctypes.data_as(C.c_void_p),
                                      C.c_double(0.3), 64, perm.ctypes.data_as(C.c_void_p))
        assert rc == 0 and np.array_equal(np.sort(perm), np.arange(n))
        perms.append(perm)
    assert np.array_equal(perms[0], perms[1])
    # and the dissection really dissected: far less fill than the natural (banded) order
    S_nd = lib.Symbolic(K, ordering=1, nd_leaf=64).stats
    S_nat = lib.Symbolic(K, ordering=2).stats
    assert S_nd["nnzL"] < 0.5 * S_nat["nnzL"]


@pytest.mark.parametrize("seed", range(24))
def test_symbolic_maps_on_random_quasidefinite_patterns(seed):
    """Randomised structures the instance generators do not produce: empty P, empty rows/columns of
    A, disconnected blocks, dense rows/columns, tiny and degenerate sizes; both orderings.  The
    numpy multifrontal runs on exactly the maps the CUDA kernels consume."""
    from clarabel_jl_b200 import lib
    K, Ds, rng = random_quasidefinite(seed)
    N = K.shape[0]
    Kf = sym_full(K)
    b = rng.standard_normal(N)
    xs = np.linalg.solve(Kf.toarray(), b)
    for ordering in (0, 1, 2):
        a = lib.Symbolic(K, ordering=ordering, nd_leaf=8).arrays()
        assert sorted(a["perm"].tolist()) == list(range(N))
        mf = MFNumpy(a)
        D = mf.factor(K.data, Ds)
        assert np.all(np.sign(D) == Ds[a["perm"]]) and mf.nreg == 0
        x = mf.solve(b)
        assert np.abs(x - xs).max() < 1e-8 * max(1.0, np.abs(xs).max())


def _sdp_chain(cb, ncones=12, side=10):
    return cb.problems.c4_sdp(ncones=ncones, side=side, n=40 * ncones, vars_per_cone=70)


def test_cone_block_dissection_order(cb):
    """Ordering 1 with dense cone blocks (PSD): every vertex outside the blocks comes before the
    blocks, the blocks are dissected (shallow tree instead of a chain), and the maps of that
    ordering factor / solve correctly (numpy multifrontal vs SuperLU)."""
    from clarabel_jl_b200 import lib
    from clarabel_jl_b200 import kkt_assembly as ka
    P, q, A, b, K = _sdp_chain(cb)
    data = cb.problemdata.ProblemData(P, q, A, b, K, cb.Settings())
    cones = cb.CompositeCone(data.cones)
    KKT, mp = ka.assemble_kkt_matrix(data.P, data.A, cones)
    N = KKT.shape[0]
    bid = lib.cone_block_ids(cones, data.n, N)
    assert bid is not None and bid.max() == 11
    Sa = lib.Symbolic(KKT, ordering=0)
    Sn = lib.Symbolic(KKT, ordering=1, block_id=bid)
    a = Sn.arrays()
    perm = a["perm"]
    assert sorted(perm.tolist()) == list(range(N))
    # every vertex outside the blocks is eliminated before each block row it is coupled to (the final
    # permutation is the postorder of the elimination tree, so "variables first" holds along every
    # root path, not as one global prefix)
    pos = np.empty(N, dtype=np.int64); pos[perm] = np.arange(N)
    Kc = sym_full(KKT).tocoo()
    sel = (bid[Kc.row] >= 0) & (bid[Kc.col] < 0)
    assert np.all(pos[Kc.col[sel]] < pos[Kc.row[sel]])
    assert Sn.stats["nlevels"] < Sa.stats["nlevels"]           # the chain of cones became a tree
    Ds = ka.fill_Dsigns(data.m, data.n, cones.p, cones)
    rng = np.random.default_rng(0)
    Kv = KKT.copy()
    Kv.data[mp.diag_full] += np.where(Ds > 0, 1.0 + rng.random(N), -1.0 - rng.random(N))
    diag_set = set(mp.diag_full.tolist())
    off = np.array([k for k in mp.Hsblocks if k not in diag_set], dtype=np.int64)
    Kv.data[off] = 0.01 * rng.standard_normal(len(off))
    mf = MFNumpy(a)
    D = mf.factor(Kv.data, Ds)
    assert np.all(np.sign(D) == Ds[perm])
    bb = rng.standard_normal(N)
    x = mf.solve(bb)
    Kf = sym_full(Kv)
    assert np.abs(Kf @ x - bb).max() < 1e-9 * max(1.0, np.abs(x).max())


def test_cone_block_dissection_is_numerically_equivalent_to_amd(cb):
    """The whole IP solve through the QDLDL oracle with the cone-block dissection order: same
    status, same iteration count, no dynamically regularised pivot - like the AMD-class order
    (late iterates of an SDP are where a wrong elimination order of the PSD blocks shows)."""
    from clarabel_jl_b200 import lib
    from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
    P, q, A, b, K = _sdp_chain(cb, ncones=10, side=8)
    sols = {}
    for name in ("amd", "cone_nd"):
        class O(OracleDirectLDLKKTSolver):
            def __init__(self, P_, A_, cones, m, n, settings, _name=name):
                perm = None
                if _name == "cone_nd":
                    from clarabel_jl_b200 import kkt_assembly as ka
                    KKT, _ = ka.assemble_kkt_matrix(P_, A_, cones)
                    S = lib.Symbolic(KKT, ordering=1, block_id=lib.cone_block_ids(cones, n, KKT.shape[0]))
                    assert S.stats["N"] == KKT.shape[0]
                    perm = S.arrays()["perm"]
                super().__init__(P_, A_, cones, m, n, settings, perm=perm)
        cb.register_kktsolver("qd_" + name, O)
        s = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="qd_" + name))
        sol = s.solve()
        sols[name] = (sol, s.kktsystem.kktsolver.ldl.regularize_count)
    (sa, ra), (sn, rn) = sols["amd"], sols["cone_nd"]
    assert sa.status_name == sn.status_name == "SOLVED"
    assert sa.iterations == sn.iterations and ra == rn == 0
    assert abs(sa.obj_val - sn.obj_val) <= 1e-8 * max(1.0, abs(sa.obj_val))
