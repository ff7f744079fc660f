"""GPU tests of the device NT scaling (cb200_update_scaling, kernels_scaling.cuh) against cones.py on the same s, z.

NN state is bitwise numpy's.  SOC state agrees per cone within 1e-13 relative (the sums run in another order).
PSD R, Rinv and λ come from a Jacobi SVD whose sign and order choices differ from LAPACK's, so the tests compare
what does not depend on them: W = R R', Rinv' Rinv = W^-1, R Rinv = I and the sorted λ."""
import ctypes as C
import numpy as np
import pytest
import scipy.sparse as sp
import reference_cases as rc

pytestmark = pytest.mark.gpu

SOC_DIMS = (2, 3, 4, 5, 64, 3000)
PSD_SIDES = (1, 2, 3, 8, 31, 32, 33, 50, 90)      # 90 > 83, the largest side that fits in shared memory


def _svec(M):
    """mat_to_svec (column-major packed upper triangle, off-diagonals * sqrt(2))."""
    n = M.shape[0]
    out = []
    for j in range(n):
        for i in range(j + 1):
            out.append(M[i, j] if i == j else M[i, j] * np.sqrt(2.0))
    return np.array(out)


def _soc_point(rng, d, scale=1.0):
    x1 = rng.standard_normal(d - 1)
    return scale * np.concatenate([[np.linalg.norm(x1) * (1.0 + rng.uniform(0.01, 1.0))], x1])


def _psd_pair(rng, n, kind):
    if kind == "random":
        B1, B2 = rng.standard_normal((n, n)), rng.standard_normal((n, n))
        return B1 @ B1.T + 0.1 * np.eye(n), B2 @ B2.T + 0.1 * np.eye(n)
    # late-iteration-like: S Z = mu I with eigenvalues spanning 1e8
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    d = 10.0 ** rng.uniform(-4, 4, n)
    mu = 1e-6
    return (Q * (mu / d)) @ Q.T, (Q * d) @ Q.T


def _inputs(specs, seed=0, psd_kind="random"):
    rng = np.random.default_rng(seed)
    s, z = [], []
    for sp_ in specs:
        name, d = sp_[0], sp_[1]
        if name == "NonnegativeConeT":
            s.append(10.0 ** rng.uniform(-8, 8, d)); z.append(10.0 ** rng.uniform(-8, 8, d))
        elif name == "ZeroConeT":
            s.append(np.zeros(d)); z.append(rng.standard_normal(d))
        elif name == "SecondOrderConeT":
            s.append(_soc_point(rng, d, 10.0 ** rng.uniform(-3, 3))); z.append(_soc_point(rng, d, 10.0 ** rng.uniform(-3, 3)))
        else:
            S, Z = _psd_pair(rng, d, psd_kind)
            s.append(_svec(S)); z.append(_svec(Z))
    return np.concatenate(s), np.concatenate(z)


def _solver(cb, specs, n=6, seed=1):
    """A B200KKTSolver over a small random problem with the given cone table (no collapsing of the specs)."""
    from clarabel_jl_b200.kktsolver_b200 import B200KKTSolver
    cones = cb.CompositeCone(specs)
    m = cones.numel
    rng = np.random.default_rng(seed)
    A = sp.random(m, n, density=min(1.0, 2.0 / n), random_state=np.random.RandomState(seed), format="csc")
    P = sp.identity(n, format="csc")
    return B200KKTSolver(P, A, cones, m, n, cb.Settings()), cones


def _pair(cb, specs, **kw):
    """(host cones after cones.update_scaling, device cones after update_scaling, solver, host ok, device ok)"""
    ks, _ = _solver(cb, specs)
    s, z = _inputs(specs, **kw)
    host, dev = cb.CompositeCone(specs), cb.CompositeCone(specs)
    ok_h = host.update_scaling(s, z, 1.0)
    ok_d = ks.update_scaling(s, z, dev)
    return host, dev, ks, ok_h, ok_d, s, z


def test_nn_bitwise(cb):
    specs = [cb.NonnegativeConeT(4000), cb.ZeroConeT(3), cb.NonnegativeConeT(17)]
    host, dev, _, ok_h, ok_d, s, z = _pair(cb, specs)
    assert ok_h and ok_d
    nn = host.nn_idx
    assert np.array_equal(dev.w[nn], host.w[nn]) and np.array_equal(dev.lam[nn], host.lam[nn])
    assert np.ptp(np.log10(s[nn])) > 14                     # the inputs span 1e+-8


def _rel_per_cone(a, b, ptr):
    return max(np.abs(a[p:q] - b[p:q]).max() / max(np.abs(b[p:q]).max(), 1e-300) for p, q in zip(ptr[:-1], ptr[1:]))


@pytest.mark.parametrize("seed", [0, 1])
def test_soc_state(cb, seed):
    specs = [cb.SecondOrderConeT(d) for d in SOC_DIMS] + [cb.NonnegativeConeT(5)] + \
            [cb.SecondOrderConeT(d) for d in reversed(SOC_DIMS)]
    host, dev, ks, ok_h, ok_d, _, _ = _pair(cb, specs, seed=seed)
    assert ok_h and ok_d
    ptr = host.soc_ptr
    si = host.soc_idx
    for a, b in ((dev.w[si], host.w[si]), (dev.lam[si], host.lam[si]), (dev.soc_u, host.soc_u), (dev.soc_v, host.soc_v)):
        assert _rel_per_cone(a, b, ptr) <= 1e-13
    for a, b in ((dev.soc_eta, host.soc_eta), (dev.soc_d, host.soc_d)):
        assert np.all(np.abs(a - b) <= 1e-13 * np.abs(b))


@pytest.mark.parametrize("bad", ["z", "s"])
def test_soc_outside_cone_fails_like_host(cb, bad):
    specs = [cb.SecondOrderConeT(5), cb.SecondOrderConeT(64), cb.SecondOrderConeT(3000)]
    ks, _ = _solver(cb, specs)
    for cone in range(3):
        s, z = _inputs(specs, seed=cone)
        x = z if bad == "z" else s
        host = cb.CompositeCone(specs)
        a = int(host.soc_ptr[cone])
        x[a] = 0.5 * np.linalg.norm(x[a + 1:int(host.soc_ptr[cone + 1])])         # x0 < |x1|
        assert host.update_scaling(s, z, 1.0) is False
        assert ks.update_scaling(s, z, cb.CompositeCone(specs)) is False
    s, z = _inputs(specs, seed=9)
    assert ks.update_scaling(s, z, cb.CompositeCone(specs)) is True


def _psd_checks(host, dev, label):
    """Every metric of every cone is measured first, so that a failure reports all of them."""
    rows, bad = [], []
    eps = np.finfo(float).eps
    for gh, gd in zip(host.psd_groups, dev.psd_groups):
        n = gh["n"]
        for j in range(len(gh["cones"])):
            Rh, Rd, Ih, Id = gh["R"][j], gd["R"][j], gh["Rinv"][j], gd["Rinv"][j]
            Wh, Wd = Rh @ Rh.T, Rd @ Rd.T
            Vh, Vd = Ih.T @ Ih, Id.T @ Id
            E = Rd.astype(np.longdouble) @ Id.astype(np.longdouble) - np.eye(n, dtype=np.longdouble)
            lh, ld = np.sort(gh["lam"][j]), np.sort(gd["lam"][j])
            m = dict(n=n, W=np.linalg.norm(Wd - Wh) / np.linalg.norm(Wh), Winv=np.linalg.norm(Vd - Vh) / np.linalg.norm(Vh),
                     RRinv=float(np.abs(E).max()))
            # R and Rinv are rounded independently, so R Rinv - I grows like n eps cond(R).  Random pairs stay under
            # 1e-12.  Late pairs (cond(R) ~ 1e4) do not: a numpy emulation of the kernel measured 4e-12 (side 33) and
            # 6e-12 (side 50), and the host's LAPACK path itself 2e-12 at side 33.  They are held to n eps cond(R).
            tol_rr = 1e-12 if label == "random" else max(1e-12, n * eps * np.linalg.cond(Rh))
            if label == "random":
                m["lam"] = np.abs(ld - lh).max() / lh.max()
                tol_w, tol_lam = 1e-10, 1e-12
            else:
                # Late pairs have cond(S) = cond(Z) = 1e8, so their scaling is determined only to about
                # eps * 1e8 = 2.2e-8 relative, by the host as much as by the device.  Measured: W and W^-1 differ from
                # the host's by up to 2.4e-10 (side 32); the host's λ is 6.9e-13 (7e-10 relative) away from the exact
                # sqrt(mu) = 1e-3 at side 8, and a numpy emulation of the kernel put both paths 1.2e-9 from it at
                # side 50.  So W, W^-1 are compared with the host's and λ with the exact value, both at eps * 1e8.
                m["lam"] = np.abs(ld - 1e-3).max() / 1e-3
                m["lam_host"] = np.abs(lh - 1e-3).max() / 1e-3
                tol_w = tol_lam = eps * 1e8
            rows.append(m)
            if not (m["W"] <= tol_w and m["Winv"] <= tol_w and m["RRinv"] <= tol_rr and m["lam"] <= tol_lam):
                bad.append(m)
    assert not bad, (label, bad, rows)


@pytest.mark.parametrize("kind", ["random", "late"])
def test_psd_state(cb, kind):
    specs = [cb.PSDTriangleConeT(n) for n in PSD_SIDES] + [cb.NonnegativeConeT(3), cb.PSDTriangleConeT(8)]
    host, dev, ks, ok_h, ok_d, _, _ = _pair(cb, specs, psd_kind=kind)
    assert ok_h and ok_d
    st = ks.ldl.stats()
    assert st["psd_scale_smem"] == len(specs) - 2 and st["psd_scale_global"] == 1      # both paths ran
    assert 1 <= st["jacobi_sweeps"] < 30
    _psd_checks(host, dev, kind)


def test_psd_not_positive_definite_fails_like_host(cb):
    specs = [cb.PSDTriangleConeT(8), cb.PSDTriangleConeT(50)]
    ks, _ = _solver(cb, specs)
    rng = np.random.default_rng(5)
    for which in ("s", "z"):
        s, z = _inputs(specs, seed=3)
        B = rng.standard_normal((50, 50))
        ev = np.linspace(1.0, 2.0, 50); ev[17] = -1e-3
        Q, _ = np.linalg.qr(B)
        bad = _svec((Q * ev) @ Q.T)
        (s if which == "s" else z)[36:] = bad
        assert cb.CompositeCone(specs).update_scaling(s, z, 1.0) is False
        assert ks.update_scaling(s, z, cb.CompositeCone(specs)) is False
    s, z = _inputs(specs, seed=3)
    assert ks.update_scaling(s, z, cb.CompositeCone(specs)) is True


MIXED = lambda cb: [cb.ZeroConeT(2), cb.NonnegativeConeT(30), cb.SecondOrderConeT(3), cb.SecondOrderConeT(4),
                    cb.SecondOrderConeT(9), cb.PSDTriangleConeT(3), cb.PSDTriangleConeT(6), cb.SecondOrderConeT(2000)]


def test_update_cones_from_device_state_is_bitwise_the_upload(cb):
    specs = MIXED(cb)
    ks1, _ = _solver(cb, specs)
    ks2, _ = _solver(cb, specs)
    s, z = _inputs(specs, seed=4)
    c1 = cb.CompositeCone(specs)
    assert ks1.update_scaling(s, z, c1)
    assert ks1.update(c1)                         # NULL pointers: refactor from the device state
    assert ks2.update(c1)                         # the downloaded state, uploaded
    N = ks1.KKT.shape[0]
    assert np.array_equal(ks1.ldl.download(0, ks1.KKT.nnz), ks2.ldl.download(0, ks2.KKT.nnz))
    assert np.array_equal(ks1.ldl.download(1, N), ks2.ldl.download(1, N))
    rng = np.random.default_rng(0)
    rx, rz = rng.standard_normal(ks1.n), rng.standard_normal(ks1.m)
    out = []
    for ks in (ks1, ks2):
        x, zz = np.zeros(ks.n), np.zeros(ks.m)
        ks.setrhs(rx, rz); assert ks.solve(x, zz)
        out.append((x, zz))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


def _state(c):
    return [c.w, c.lam, c.soc_eta, c.soc_d, c.soc_u, c.soc_v] + \
           [g[k] for g in c.psd_groups for k in ("R", "Rinv", "lam")]


def test_repeatable_and_resident(cb):
    import torch
    specs = MIXED(cb) + [cb.PSDTriangleConeT(90)]
    ks, _ = _solver(cb, specs)
    s, z = _inputs(specs, seed=6, psd_kind="late")
    a, b = cb.CompositeCone(specs), cb.CompositeCone(specs)
    assert ks.update_scaling(s, z, a) and ks.update_scaling(s, z, b)
    assert all(np.array_equal(x, y) for x, y in zip(_state(a), _state(b)))
    ts, tz = torch.tensor(s, device="cuda"), torch.tensor(z, device="cuda")
    torch.cuda.synchronize()
    ks.ldl.set_resident(True)
    try:
        assert ks.update_scaling(ts.data_ptr(), tz.data_ptr(), None)
        c = cb.CompositeCone(specs)
        ks.download_scaling(c)
    finally:
        ks.ldl.set_resident(False)
    assert all(np.array_equal(x, y) for x, y in zip(_state(a), _state(c)))
    assert ks.ldl.timers()["scale_ms"] > 0


def test_nonsymmetric_cone_table_is_refused(cb):
    specs = [cb.NonnegativeConeT(3), cb.ExponentialConeT()]
    ks, cones = _solver(cb, specs)
    s, z = np.ones(6), np.ones(6)
    rc_ = ks.ldl._L.cb200_update_scaling(ks.ldl._h, s.ctypes.data_as(C.c_void_p), z.ctypes.data_as(C.c_void_p),
                                        C.byref(C.c_int32()))
    assert rc_ == -2
    with pytest.raises(RuntimeError):
        ks.update_scaling(s, z, cones)


# ---------------------------------------------------------------- whole solves, setting off and on
def _rel(a, b):
    return abs(a - b) / max(1.0, abs(b))


def _both(cb, P, q, A, b, K):
    off = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    on = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200", b200_device_cone_scaling=True))
    return off, off.solve(), on, on.solve()


def _same(so, sn):
    assert sn.status_name == so.status_name and sn.iterations == so.iterations
    if not np.isnan(so.obj_val):
        assert _rel(sn.obj_val, so.obj_val) < 1e-6 and _rel(sn.obj_val_dual, so.obj_val_dual) < 1e-6
        assert abs(sn.r_prim - so.r_prim) < 1e-6 and abs(sn.r_dual - so.r_dual) < 1e-6


@pytest.mark.parametrize("case", rc.cases(), ids=lambda c: c["name"])
def test_golden_cases_device_scaling(cb, case):
    _, so, on, sn = _both(cb, case["P"], case["q"], case["A"], case["b"], case["cones"])
    _same(so, sn)
    assert sn.status_name == case["status"]
    if on.cones.is_symmetric and sn.iterations > 0 and on.data.m > 0:
        assert on.kktsystem.kktsolver.ldl.timers()["scale_ms"] > 0


def test_sdp_chordal_device_scaling_setting(cb):
    """Power cones: the setting leaves the host scaling in place."""
    from test_nonsymmetric_cones import _sdp_chordal_problem
    _, so, on, sn = _both(cb, *_sdp_chordal_problem(cb))
    _same(so, sn)
    assert on.kktsystem.kktsolver.ldl.timers()["scale_ms"] == 0


@pytest.mark.parametrize("name", ["C3", "C4r"])
def test_bench_workloads_device_scaling(cb, name):
    import bench
    _, so, on, sn = _both(cb, *bench.make_problem(name))
    _same(so, sn)
    assert np.abs(sn.x - so.x).max() < 1e-5 * max(1.0, np.abs(so.x).max())
    assert on.kktsystem.kktsolver.ldl.timers()["scale_ms"] > 0
