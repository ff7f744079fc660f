"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C-ABI against
the CPU oracle on the same seeded inputs.

Tolerances: cone->K value update is pure elementwise FP64 => bit-exact for Zero/NN/SOC blocks
(PSD blocks use a different summation order for R*R' => 1e-13 relative); linear solves 1e-9
relative against the QDLDL oracle; whole IP solves must give the identical status and iteration
count and objectives / residual measures within 1e-6 relative (BASELINE.json north_star)."""
import numpy as np
import pytest
import reference_cases as rc
from common import small_instances, kkt_fixture, sym_full

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def b200(cb):
    from clarabel_jl_b200 import kktsolver_b200
    return kktsolver_b200


@pytest.mark.parametrize("name", ["C1s", "C1", "C2s", "C3s", "C4s", "C4m", "C5s"])
@pytest.mark.parametrize("ordering", [0, 1])
def test_inner_boundary_factor_solve_vs_oracle(cb, b200, name, ordering):
    from oracle import qdldl as oq
    KKT, mp, Ds, data, cones = kkt_fixture(cb, small_instances(cb)[name])
    N = KKT.shape[0]
    eng = b200.B200DirectLDLSolver(KKT, Ds, cb.Settings(), ordering=ordering, nd_leaf_size=32)
    assert eng.refactor()
    F = oq.QDLDLFactorisation(KKT, Ds); assert F.refactor()
    rng = np.random.default_rng(3)
    Kf = sym_full(KKT)
    for _ in range(2):
        b = rng.standard_normal(N)
        x = np.zeros(N); eng.solve(x, b)
        xo = b.copy(); F.solve(xo)
        scale = max(1.0, np.abs(xo).max())
        assert np.abs(x - xo).max() < 1e-9 * scale
        assert np.abs(Kf @ x - b).max() < 1e-9 * scale
    # pivots: same signs, same values up to rounding, after mapping through the permutations
    D = eng.download(1, N); perm = eng.download(3, N).astype(np.int64)
    assert np.all(np.sign(D) == Ds[perm])
    # update_values!/scale_values! then refactor
    idx = mp.diag_full[: max(1, N // 3)]
    newv = KKT.data[idx] * 1.5
    eng.update_values(idx, newv); F.update_values(idx, newv)
    eng.scale_values(mp.A[: len(mp.A) // 2], 0.5); F.scale_values(mp.A[: len(mp.A) // 2], 0.5)
    assert eng.refactor() and F.refactor()
    b = rng.standard_normal(N)
    x = np.zeros(N); eng.solve(x, b)
    xo = b.copy(); F.solve(xo)
    assert np.abs(x - xo).max() < 1e-9 * max(1.0, np.abs(xo).max())
    info = eng.info()
    assert info.nnzA == KKT.nnz and info.nnzL > 0


def _iterate_cones(cb, gen, iters=3):
    """Run a few oracle IP iterations so the cone scaling state is realistic."""
    P, q, A, b, K = gen()
    s = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="qdldl"))
    s.solve(max_iter=iters)
    return s


@pytest.mark.parametrize("name", ["C1s", "C2s", "C3s", "C4s", "C5s"])
def test_cone_update_and_regularisation_match_oracle(cb, b200, name):
    s = _iterate_cones(cb, small_instances(cb)[name])
    data, cones, st = s.data, s.cones, s.settings
    oracle = s.kktsystem.kktsolver
    assert oracle.update(cones)
    gpu = b200.B200KKTSolver(data.P, data.A, cones, data.m, data.n, st)
    assert gpu.update(cones)
    nz_gpu, nz_cpu = gpu.device_nzval(), oracle.KKT.data
    mp = oracle.map
    psd_mask = np.zeros(len(nz_cpu), dtype=bool)
    for i, t in enumerate(cones.types):
        if t == cb.cones.PSD:
            psd_mask[mp.Hsblocks[cones.rng_blocks[i]:cones.rng_blocks[i + 1]]] = True
    assert np.array_equal(nz_gpu[~psd_mask], nz_cpu[~psd_mask])          # bit-exact
    if psd_mask.any():
        sc = np.abs(nz_cpu[psd_mask]).max()
        assert np.abs(nz_gpu[psd_mask] - nz_cpu[psd_mask]).max() <= 1e-13 * sc
    eps_gpu = gpu.ldl.download(4, 1)[0]
    assert eps_gpu == oracle.diagonal_regularizer or abs(eps_gpu - oracle.diagonal_regularizer) < 1e-22
    # solves with IR: same answers to 1e-9
    rng = np.random.default_rng(5)
    for _ in range(2):
        rx, rz = rng.standard_normal(data.n), rng.standard_normal(data.m)
        xg, zg = np.zeros(data.n), np.zeros(data.m)
        xo, zo = np.zeros(data.n), np.zeros(data.m)
        gpu.setrhs(rx, rz); assert gpu.solve(xg, zg)
        oracle.setrhs(rx, rz); assert oracle.solve(xo, zo)
        sc = max(1.0, np.abs(xo).max(), np.abs(zo).max())
        assert np.abs(xg - xo).max() < 1e-8 * sc and np.abs(zg - zo).max() < 1e-8 * sc
    # lhs = nothing (None) is accepted, like the reference
    gpu.setrhs(rx, rz); assert gpu.solve(None, zg)


@pytest.mark.parametrize("name", ["C3s", "C4s"])
def test_resident_mode_takes_device_pointers(cb, b200, name):
    """cb200_set_resident: update_cones / setrhs then take DEVICE pointers (inputs staged in HBM, the mode
    bench.py's device-resident `value` is measured in).  Same bits as the host-buffer path."""
    import torch
    s = _iterate_cones(cb, small_instances(cb)[name])
    data, cones, st = s.data, s.cones, s.settings
    gpu = b200.B200KKTSolver(data.P, data.A, cones, data.m, data.n, st)
    N = gpu.KKT.shape[0]
    rng = np.random.default_rng(11)
    rx, rz = rng.standard_normal(data.n), rng.standard_normal(data.m)
    assert gpu.update(cones)
    xg, zg = np.zeros(data.n), np.zeros(data.m)
    gpu.setrhs(rx, rz); assert gpu.solve(xg, zg)
    x_host = gpu.ldl.download(6, N)
    D_host = gpu.ldl.download(1, N)
    state = cones.export_state()
    dev = {k: torch.from_numpy(np.ascontiguousarray(state[k], dtype=np.float64)).cuda() for k in gpu.STATE_KEYS}
    tx, tz = torch.from_numpy(rx).cuda(), torch.from_numpy(rz).cuda()
    torch.cuda.synchronize()
    gpu.ldl.set_resident(True)
    try:
        assert gpu.update_staged([dev[k].data_ptr() if dev[k].numel() else 0 for k in gpu.STATE_KEYS])
        gpu.setrhs_staged(tx.data_ptr(), tz.data_ptr())
        assert gpu.solve(None, None)
        assert np.array_equal(gpu.ldl.download(1, N), D_host)
        assert np.array_equal(gpu.ldl.download(6, N), x_host)
        # NULL pointers keep the state in HBM: same factorisation again
        assert gpu.update_staged([0] * len(gpu.STATE_KEYS))
        assert np.array_equal(gpu.ldl.download(1, N), D_host)
    finally:
        gpu.ldl.set_resident(False)
    # back on the host-buffer path
    x2, z2 = np.zeros(data.n), np.zeros(data.m)
    gpu.setrhs(rx, rz); assert gpu.solve(x2, z2)
    assert np.array_equal(x2, xg) and np.array_equal(z2, zg)


def _rel(a, b):
    return abs(a - b) / max(1.0, abs(b))


@pytest.mark.parametrize("case", rc.cases(), ids=lambda c: c["name"])
def test_reference_goldens_through_gpu_backend(cb, b200, case):
    so = cb.Solver(case["P"], case["q"], case["A"], case["b"], case["cones"],
                   cb.Settings(direct_solve_method="qdldl")).solve()
    sg = cb.Solver(case["P"], case["q"], case["A"], case["b"], case["cones"],
                   cb.Settings(direct_solve_method="b200")).solve()
    assert sg.status_name == case["status"] == so.status_name
    if case.get("x") is not None:
        assert np.linalg.norm(sg.x - np.asarray(case["x"])) < 1e-3
    if case.get("obj") is not None:
        assert abs(sg.obj_val - case["obj"]) < 1e-3
    if not np.isnan(so.obj_val):
        assert _rel(sg.obj_val, so.obj_val) < 1e-6 and _rel(sg.obj_val_dual, so.obj_val_dual) < 1e-6


@pytest.mark.parametrize("name", ["C1", "C2s", "C3s", "C4s", "C4m", "C5s"])
def test_whole_solve_parity_gpu_vs_oracle(cb, b200, name):
    P, q, A, b, K = small_instances(cb)[name]()
    so_s = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="qdldl"))
    so = so_s.solve()
    sg_s = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    sg = sg_s.solve()
    assert sg.status_name == so.status_name == "SOLVED"
    assert sg.iterations == so.iterations
    assert _rel(sg.obj_val, so.obj_val) < 1e-6 and _rel(sg.obj_val_dual, so.obj_val_dual) < 1e-6
    assert abs(sg.r_prim - so.r_prim) < 1e-6 and abs(sg.r_dual - so.r_dual) < 1e-6
    assert np.abs(sg.x - so.x).max() < 1e-5 * max(1.0, np.abs(so.x).max())


def test_data_update_path(cb, b200):
    """update_P!/update_A! (data_updating.jl:56-100): re-solve after an in-place value update equals
    a fresh solve (reference test/OptTests/data_updating.jl, tol 1e-7)."""
    P, q, A, b, K = small_instances(cb)["C1s"]()
    s = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    s.solve()
    P2 = s.data.P.copy(); P2.data *= 1.1
    A2 = s.data.A.copy(); A2.data *= 0.9
    s.data.P.data[:] = P2.data; s.data.A.data[:] = A2.data
    s.kktsystem.update_P(s.data.P); s.kktsystem.update_A(s.data.A)
    sol1 = s.solve()
    x1 = sol1.x.copy()
    # fresh solver on the same (already equilibrated) data
    st = cb.Settings(direct_solve_method="b200", equilibrate_enable=False)
    s2 = cb.Solver(s.data.P, s.data.q, s.data.A, s.data.b, s.data.cones, st)
    s2.data.d[:] = s.data.d; s2.data.dinv[:] = s.data.dinv
    s2.data.e[:] = s.data.e; s2.data.einv[:] = s.data.einv; s2.data.c = s.data.c
    s2.data.normq, s2.data.normb = s.data.normq, s.data.normb
    sol2 = s2.solve()
    assert sol1.status_name == sol2.status_name == "SOLVED"
    assert np.abs(x1 - sol2.x).max() < 1e-7 * max(1.0, np.abs(x1).max())
