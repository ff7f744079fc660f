"""Shared helpers for the tests: instance builders and KKT-level fixtures."""
import numpy as np
import scipy.sparse as sp


def small_instances(cb):
    pr = cb.problems
    return {
        "C1": lambda: pr.c1_random_qp(),
        "C1s": lambda: pr.c1_random_qp(n=120, m=260, seed=7),
        "C2s": lambda: pr.c2_portfolio(n=3000),
        "C3s": lambda: pr.c3_socp(n=3000, ncones=60),
        "C4s": lambda: pr.c4_sdp(ncones=6, side=8, n=200, vars_per_cone=50),
        "C4m": lambda: pr.c4_sdp(ncones=4, side=22, n=300, vars_per_cone=120),
        "C5s": lambda: pr.c5_block_angular(nblocks=4, grid=12, nlink=10, link_nnz=8),
    }


def kkt_fixture(cb, gen, seed=0):
    """Assembled KKT (triu) with quasidefinite random values in the cone blocks."""
    from clarabel_jl_b200 import kkt_assembly as ka
    P, q, A, b, K = gen()
    st = cb.Settings()
    data = cb.problemdata.ProblemData(P, q, A, b, K, st)
    cones = cb.CompositeCone(data.cones)
    KKT, mp = ka.assemble_kkt_matrix(data.P, data.A, cones)
    N = KKT.shape[0]
    rng = np.random.default_rng(seed)
    Ds = ka.fill_Dsigns(data.m, data.n, cones.p)
    KKT.data[mp.diag_full] += np.where(Ds > 0, 1.0 + rng.random(N), -1.0 - rng.random(N))
    KKT.data[mp.soc_u] = 0.1 * rng.standard_normal(len(mp.soc_u))
    KKT.data[mp.soc_v] = 0.1 * rng.standard_normal(len(mp.soc_v))
    # dense (non-diagonal) cone blocks: make them negative definite-ish via small off-diagonals
    diag_set = set(mp.diag_full.tolist())
    off = np.array([k for k in mp.Hsblocks if k not in diag_set], dtype=np.int64)
    if len(off):
        KKT.data[off] = 0.02 * rng.standard_normal(len(off))
    return KKT, mp, Ds, data, cones


def cone_table_problem(cb, specs, n=8, seed=0, extra_A=None):
    """(P, A, cones) for a designed cone table: P diagonal positive definite, A (m x n) with one entry
    in every row plus a few random ones, so that K is quasidefinite whatever the cone state.
    extra_A: optional dense m x n array added to A (dense rows / columns)."""
    cones = cb.CompositeCone(specs)
    m = cones.numel
    rng = np.random.default_rng(seed)
    P = sp.diags(1.0 + rng.random(n)).tocsc()
    A = sp.csc_matrix((rng.standard_normal(m), (np.arange(m), rng.integers(0, n, m))), shape=(m, n))
    A = A + sp.random(m, n, density=min(1.0, 2.0 / n), random_state=seed, data_rvs=rng.standard_normal)
    if extra_A is not None:
        A = A + sp.csc_matrix(extra_A)
    A = A.tocsc(); A.sort_indices()
    return P, A, cones


def set_interior_scaling(cones, seed, spread=0.0):
    """cones.update_scaling at a random interior point (s, z); NN / SOC / PSD scales spread over
    10^(+-spread).  Nonsymmetric cones keep the unit initialisation point."""
    m = cones.numel
    rng = np.random.default_rng(seed)
    z, s = np.zeros(m), np.zeros(m)
    cones.unit_initialization(z, s)
    sc = lambda k: 10.0 ** rng.uniform(-spread, spread, k)
    ni = cones.nn_idx
    s[ni] = sc(len(ni)) * (0.5 + rng.random(len(ni))); z[ni] = sc(len(ni)) * (0.5 + rng.random(len(ni)))
    for v in (s, z):
        for ci in cones.soc_cones:
            a, b = int(cones.rng_cones[ci]), int(cones.rng_cones[ci + 1])
            t = rng.standard_normal(b - a - 1)
            v[a] = np.linalg.norm(t) * (1.0 + rng.random()) + 0.1
            v[a + 1:b] = t
            v[a:b] *= sc(1)
        for g in cones.psd_groups:
            k, nn = len(g["cones"]), g["n"]
            M = rng.standard_normal((k, nn, nn))
            S = (M @ np.swapaxes(M, 1, 2)) / nn + 0.2 * np.eye(nn)
            S *= sc(k)[:, None, None]
            v[g["idx"]] = cones._psd_svec(g, S)
    assert cones.update_scaling(s, z, 1.0)
    return s, z


def set_synthetic_state(cones, seed, spread=8.0):
    """A scaling state written field by field: NN w and SOC eta over 10^(+-spread), SOC w unit
    hyperbolic (w0 = sqrt(1 + |w1|^2)) with |w1| over the same range, arbitrary d, u, v, PSD R with
    entries over 10^(+-spread / 4)."""
    rng = np.random.default_rng(seed)
    sc = lambda k: 10.0 ** rng.uniform(-spread, spread, k)
    cones.w[cones.nn_idx] = sc(len(cones.nn_idx))
    for ci in cones.soc_cones:
        a, b = int(cones.rng_cones[ci]), int(cones.rng_cones[ci + 1])
        t = rng.standard_normal(b - a - 1) * sc(1)
        cones.w[a + 1:b] = t
        cones.w[a] = np.sqrt(1.0 + t @ t)
    if cones.nsoc:
        cones.soc_eta[:] = sc(cones.nsoc)
        cones.soc_d[:] = rng.random(cones.nsoc)
        cones.soc_u[:] = rng.standard_normal(len(cones.soc_u)) * sc(len(cones.soc_u))
        cones.soc_v[:] = rng.standard_normal(len(cones.soc_v)) * sc(len(cones.soc_v))
    for g in cones.psd_groups:
        g["R"][:] = rng.standard_normal(g["R"].shape) * 10.0 ** rng.uniform(-spread / 4, spread / 4, g["R"].shape)


def sym_full(K):
    return (K + sp.triu(K, 1).T).tocsc()


def random_quasidefinite(seed):
    """Randomised KKT structures the instance generators do not produce: empty P, empty rows/columns
    of A, disconnected blocks, dense rows/columns, tiny and degenerate sizes.  -> (K triu CSC, Dsigns)"""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(1, 60)); m = int(rng.integers(0, 80))
    dens = float(rng.choice([0.02, 0.1, 0.4]))
    rs = np.random.RandomState(seed)
    Ph = sp.random(n, n, dens, random_state=rs)
    P = (Ph @ Ph.T + sp.identity(n) * (0.5 if seed % 3 else 1.0)).tocsc() if seed % 5 else sp.identity(n, format="csc")
    A = sp.random(m, n, dens, random_state=rs).tolil()
    if m > 3 and n > 3:
        A[0, :] = 1.0 if seed % 2 else 0.0                      # dense or empty row
        A[:, 0] = 0.0                                           # empty column
        if seed % 4 == 0:
            A[m // 2:, : n // 2] = 0.0; A[: m // 2, n // 2:] = 0.0      # two disconnected blocks
    A = A.tocsc()
    K = sp.bmat([[P, A.T], [A, -sp.identity(m) * 0.7]]).tocsc() if m else P
    K = sp.triu(K).tocsc(); K.sort_indices()
    Ds = np.r_[np.ones(n, dtype=np.int64), -np.ones(m, dtype=np.int64)]
    return K, Ds, rng
