"""GPU kernel tests (run with -m gpu on an H100): every factorisation and solve kernel path against
the extended-precision multifrontal reference (mf_numpy with np.longdouble) on the front zoo
(front_zoo.py), compared in the device storage format: D (download selector 1) and the whole panel
storage (selector 2) entry by entry, before iterative refinement can hide anything.

Bounds.  Well-conditioned parts: |gpu - ref| <= 1e-12 * max(1, |ref|) for every D and L entry
(the zoo keeps |L| < 1 and |D| in [0.5, 10.5], so a correct FP64 factor is within ~1e-14).  The
poorly scaled part is S K0 S with S = diag(2^k), |k| <= 7: scaling by powers of two commutes with
rounding, so the computed factor is the scaled factor of K0 and entry (i, j) of L may carry the
error of K0's factor times s_i / s_j; the bound there is 1e-12 * max(s_i / s_j, |ref|) (s_i^2 for
D).  Solves: max |x - x_ref| <= 1e-12 * max |x_ref| (weighted by S for the scaled part)."""
import os
import subprocess
import sys
import numpy as np
import pytest
import front_zoo as fz
from common import sym_full
from mf_numpy import MFNumpy, gpu_storage

pytestmark = pytest.mark.gpu

VARIANTS = {
    "default": {},
    "tma_tile128": {"CB200_TMA_TILE": "128"},
    "tma_tile_by_size": {"CB200_TMA_TILE": "0"},     # the size rule picks the 64 tile below 1024 rows, i.e. on every zoo front
    "ldg_gemm": {"CB200_NO_TMA": "1"},
    "tma_natural_order": {"CB200_TMA_NATURAL": "1"},
    "no_panel_kernel": {"CB200_NO_PANEL": "1"},
    "panel_max_nf96": {"CB200_PANEL_MAX_NF": "96"},
    "single_stream": {"CB200_MULTISTREAM": "0"},
    "no_graph": {"CB200_GRAPH": "0"},
    "solve_subtrees": {"CB200_SUBTREE": "1"},
    "split_row_loads": {"CB200_MERGED_ROWS": "0"},
}
PARTS = {d.name: d for d in fz.parts()}
_LAYOUT_KEYS = ("CB200_NO_PANEL", "CB200_PANEL_MAX_NF")      # variants that change the symbolic layout
_REF = {}


def _opts(env):
    return fz.Options(no_panel=env.get("CB200_NO_PANEL") == "1",
                      panel_max_nf=int(env.get("CB200_PANEL_MAX_NF", 152)))


def _set_env(monkeypatch, env):
    for k, v in {**fz.ZOO_ENV, **env}.items():
        monkeypatch.setenv(k, v)


def reference(design, env):
    """(K, signs, symbolic arrays, MFNumpy, storage, tolerance and region masks), cached per layout"""
    key = (design.name, tuple(env.get(k) for k in _LAYOUT_KEYS))
    if key not in _REF:
        from clarabel_jl_b200 import lib
        K, sg, _ = design.build()
        a = lib.Symbolic(K, ordering=2).arrays()
        fz.check_design(design, a)
        mf = MFNumpy(a, np.longdouble)
        mf.factor(K.data, sg)
        st = gpu_storage(mf)
        sp_ = design.scale[a["perm"]]                        # scale of each permuted index
        tol = np.zeros(len(st)); lower = np.zeros(len(st), bool); upper = np.zeros(len(st), bool)
        pad = np.zeros(len(st), bool)
        fronts, _, _ = fz.route(a, K, _opts(env))
        for sn in range(mf.nsuper):
            f, l = int(a["sn_first"][sn]), int(a["sn_first"][sn + 1]); ns = l - f
            rows = a["rows"][a["rows_ptr"][sn]:a["rows_ptr"][sn + 1]]
            nf = ns + len(rows); ld = int(a["panel_ld"][sn]); off = int(a["panel_off"][sn])
            g = np.r_[np.arange(f, l), rows]                 # permuted index of every front row
            idx = np.arange(off, off + ld * ns).reshape(ns, ld)    # [column, row]
            ratio = sp_[g][None, :] / sp_[f:l][:, None]
            ratio[np.arange(ns), np.arange(ns)] = sp_[f:l] ** 2
            r, c = np.meshgrid(np.arange(nf), np.arange(ns))
            tol[idx[:, :nf]] = 1e-12 * np.maximum(ratio, np.abs(st[idx[:, :nf]]).astype(float))
            lower[idx[:, :nf][r >= c]] = True
            upper[idx[:, :nf][r < c]] = True
            pad[idx[:, nf:]] = True
        # D: 1e-12 * max(s^2, |D|)
        tolD = 1e-12 * np.maximum(sp_ ** 2, np.abs(mf.D).astype(float))
        panel_fronts = np.zeros(len(st), bool)
        for sn, fr in enumerate(fronts):
            if fr["kernel"].startswith("panel"):
                off = int(a["panel_off"][sn]); panel_fronts[off:off + int(a["panel_ld"][sn]) * fr["ns"]] = True
        _REF[key] = dict(design=design, K=K, sg=sg, a=a, mf=mf, st=st, tol=tol, tolD=tolD, lower=lower, upper=upper,
                         pad=pad, panel_fronts=panel_fronts, fronts=fronts)
    return _REF[key]


def _handle(K, sg, **over):
    from clarabel_jl_b200.kktsolver_b200 import B200DirectLDLSolver
    return B200DirectLDLSolver(K, sg, None, ordering=2, **over)


def check_factor(h, R):
    N = len(R["sg"])
    D = h.download(1, N)
    assert np.all(np.abs(D - R["mf"].D.astype(float)) <= R["tolD"])
    Lg = h.download(2, len(R["st"]))
    err = np.abs(Lg - R["st"].astype(float))
    bad = np.flatnonzero(R["lower"] & ~(err <= R["tol"]))
    assert bad.size == 0, f"{bad.size} panel entries off, first at storage offset {bad[:5]}"
    # above the diagonal of L11: never read by the solves; zero except inside the 64-blocks of the
    # panel kernel, which keeps the mirror of the inverted block there
    assert np.all(np.isfinite(Lg[R["upper"]]))
    assert np.all(Lg[R["upper"] & ~R["panel_fronts"]] == 0)
    assert np.all(Lg[R["pad"]] == 0)                         # padding rows nf..ld-1 stay zero
    return D, Lg


def _rhs_set(R, design):
    a, N = R["a"], len(R["sg"])
    rng = np.random.default_rng(7)
    ns = np.diff(a["sn_first"])
    sn = int(np.argmax(ns))
    q = int(a["sn_first"][sn]) + min(int(ns[sn]), 64) - 1     # last column of the first 64-block
    ek = np.zeros(N); ek[a["perm"][q]] = 1.0
    return {"random": rng.standard_normal(N), "zero": np.zeros(N), "e_k": ek,
            "wide": rng.standard_normal(N) * 10.0 ** rng.uniform(-8, 8, N)}


def check_solves(h, R, design):
    w = design.scale                                          # 1 except for the scaled part
    xs = {}
    for name, b in _rhs_set(R, design).items():
        x = np.zeros(len(b)); h.solve(x, b)
        xr = R["mf"].solve(b).astype(float)
        if name == "zero":
            assert np.all(x == 0)
        else:
            assert np.abs(w * (x - xr)).max() <= 1e-12 * np.abs(w * xr).max(), name
        xs[name] = x
    return xs


@pytest.mark.parametrize("part", list(PARTS))
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_factor_and_solve_parity(monkeypatch, variant, part):
    env = VARIANTS[variant]
    _set_env(monkeypatch, env)
    d = PARTS[part]
    R = reference(d, env)
    h = _handle(R["K"], R["sg"])
    assert h.refactor()
    check_factor(h, R)
    assert h.download(5, 1)[0] == 0
    check_solves(h, R, d)
    st = h.stats()
    assert st["nsuper"] == len(R["fronts"])
    assert st["nlarge"] == sum(f["kernel"] == "large" for f in R["fronts"])
    assert st["use_tma"] == (0 if env.get("CB200_NO_TMA") == "1" else 1)
    if st["use_tma"]:
        assert st["tma_kmajor"] == (0 if env.get("CB200_TMA_NATURAL") == "1" else 1)
    nsub = sum(f["subtree_root"] for f in R["fronts"])
    assert st["subtrees"] == (nsub if env.get("CB200_SUBTREE") == "1" else 0)
    if part == "subtree":
        assert nsub == 1


@pytest.mark.parametrize("flag", ["CB200_POISON=1", "CB200_WARP16=0"])
def test_process_wide_switches(flag):
    """CB200_POISON (0xFF-filled device buffers: the read-before-write check) and CB200_WARP16 are
    read once per process: run the default parity tests in a fresh interpreter with each set"""
    k, v = flag.split("=")
    env = dict(os.environ, **{k: v})
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(here, "test_gpu_kernels.py"), "-k", "test_factor_and_solve_parity and default"],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


EXPECTED_FINE = {"factor_small_nf16", "factor_small_nf32", "factor_small_nf64", "factor_small_nf152",
                 "factor_panel_c0", "factor_panel_c1", "factor_panel_c2", "factor_panel_c3",
                 "zero_update_blocks", "assemble_large", "piv_diag", "piv_rows", "schur_gemm", "finish_large",
                 "panel_update", "fwd_leaf", "fwd_warp", "fwd_cta", "fwd_big_assemble", "fwd_big_tri",
                 "fwd_big_gemv", "bwd_leaf", "bwd_warp", "bwd_cta", "bwd_big_gemvT", "bwd_big_tri"}


@pytest.mark.parametrize("variant,parts,expected", [
    ("default", list(PARTS), EXPECTED_FINE),
    ("solve_subtrees", ["subtree"], {"fwd_sub", "bwd_sub"}),
    ("no_panel_kernel", ["panel"], {"factor_small_nf96", "factor_small_nf128", "factor_small_nf152"})])
def test_zoo_reaches_every_kernel_class(monkeypatch, variant, parts, expected):
    env = VARIANTS[variant]
    _set_env(monkeypatch, env)
    seen = set()
    for name in parts:
        R = reference(PARTS[name], env)
        h = _handle(R["K"], R["sg"])
        h.set_detail(2)
        assert h.refactor()
        b = np.ones(len(R["sg"]))
        x = np.zeros_like(b); h.solve(x, b)
        xr = R["mf"].solve(b).astype(float)
        assert np.abs(x - xr).max() <= 1e-12 * np.abs(xr).max()
        seen |= {k for k, v in h.fine_timers().items() if v > 0}
    assert expected <= seen, sorted(expected - seen)


def _pos(a):
    p = np.empty(len(a["perm"]), dtype=np.int64); p[a["perm"]] = np.arange(len(a["perm"]))
    return p


@pytest.mark.parametrize("extra", [0, 66])
@pytest.mark.parametrize("variant", ["default", "ldg_gemm", "no_panel_kernel"])
def test_dynamic_regularisation(monkeypatch, variant, extra):
    """zero / wrong-sign Schur pivots in small, panel and large fronts (first / last columns, the
    16-column step boundary 15/16/17, the 64-block boundary 0/63/64 and the last partial block)"""
    env = VARIANTS[variant]
    _set_env(monkeypatch, env)
    R = reference(fz.part_reg(extra), env)
    want = R["design"].reg_columns()
    assert R["mf"].nreg == len(want)
    h = _handle(R["K"], R["sg"])
    assert h.refactor()
    D, _ = check_factor(h, R)
    delta = 2e-7
    q = _pos(R["a"])[want]
    assert np.all(D[q] == delta * R["sg"][want])               # exactly +-delta
    assert h.download(5, 1)[0] == len(want)
    log = h.download(7, 64)
    if len(want) <= 64:
        assert sorted(log[:len(want)].astype(int).tolist()) == want and np.all(log[len(want):] == -1)
    else:                                                     # slots filled in atomicAdd order
        assert len(set(log.astype(int).tolist())) == 64 and set(log.astype(int).tolist()) <= set(want)
    b = np.random.default_rng(3).standard_normal(R["K"].shape[0])
    x = np.zeros_like(b); h.solve(x, b)
    xr = R["mf"].solve(b).astype(float)
    assert np.abs(x - xr).max() <= 1e-12 * np.abs(xr).max()


def test_zero_pivot_without_regularisation_fails_softly(monkeypatch):
    _set_env(monkeypatch, {})
    R = reference(fz.part_reg(), {})
    h = _handle(R["K"], R["sg"], dynamic_regularization_enable=0)
    assert h.refactor() is False
    assert h.download(5, 1)[0] == 0


@pytest.mark.parametrize("part", ["large", "children2049", "panel"])
def test_refactor_graph_replay_matches_fresh_handle(monkeypatch, part):
    """refactor, update_values + scale_values, refactor again (a replay of the captured factor
    graph) == the first refactor of a fresh handle on the new values: bit for bit, except where
    k_assemble_atomic (more than 2048 children) sums in a run-dependent order"""
    _set_env(monkeypatch, {})
    d = PARTS[part]
    R = reference(d, {})
    K, sg = R["K"], R["sg"]
    diag = np.array([K.indptr[j + 1] - 1 for j in range(K.shape[0])])      # sorted: diagonal last
    assert np.all(K.indices[diag] == np.arange(K.shape[0]))
    idx = diag[::3]; newv = K.data[idx] * 1.5
    sidx = np.setdiff1d(np.arange(K.nnz), diag)[::2]
    K2 = K.copy(); K2.data[idx] = newv; K2.data[sidx] *= 0.5
    h1 = _handle(K, sg, use_cuda_graph=3)
    assert h1.refactor()
    assert h1.stats()["factor_graphs"] == 1                 # captured by the first refactor
    h1.update_values(idx, newv); h1.scale_values(sidx, 0.5)
    assert h1.refactor()                                     # ... and replayed here
    assert h1.stats()["factor_graphs"] == 1
    h2 = _handle(K2, sg, use_cuda_graph=3)
    assert h2.refactor()
    b = np.random.default_rng(5).standard_normal(K.shape[0])
    x1, x2 = np.zeros_like(b), np.zeros_like(b)
    h1.solve(x1, b); h2.solve(x2, b)
    N, nL = K.shape[0], int(R["a"]["panel_off"][-1])
    got = [h1.download(1, N), h1.download(2, nL), x1]
    ref = [h2.download(1, N), h2.download(2, nL), x2]
    exact = not any(f["atomic"] for f in R["fronts"])
    for g, r in zip(got, ref):
        if exact:
            assert np.array_equal(g, r)
        else:
            assert np.abs(g - r).max() <= 1e-13 * max(1.0, np.abs(r).max())
    # and the new factor is the right one
    mf = MFNumpy(R["a"], np.longdouble); mf.factor(K2.data, sg)
    assert np.abs(got[0] - mf.D.astype(float)).max() <= 1e-12 * np.abs(mf.D).max()


def test_refinement_with_a_long_row(cb):
    """B200KKTSolver (cb200_solve_ir: k_residual_long for the K row of more than 2048 entries)
    against the extended-precision solve of the same K"""
    import scipy.sparse as sp
    from clarabel_jl_b200 import lib
    from clarabel_jl_b200.kktsolver_b200 import B200KKTSolver
    rng = np.random.default_rng(17)
    n, m = 2100, 40
    P = sp.diags(1.0 + rng.random(n), format="csc")
    A = sp.random(m - 1, n, 0.01, random_state=np.random.RandomState(3), format="csr")
    A = sp.vstack([sp.csr_matrix(np.ones((1, n))), A]).tocsc()
    q = rng.standard_normal(n); b = np.ones(m)
    s = cb.Solver(P, q, A, b, [cb.cones.NonnegativeConeT(m)], cb.Settings(direct_solve_method="qdldl"))
    s.solve(max_iter=2)
    data, cones, st = s.data, s.cones, s.settings
    gpu = B200KKTSolver(data.P, data.A, cones, data.m, data.n, st)
    assert gpu.update(cones)
    K = gpu.KKT.copy(); K.data = gpu.device_nzval()
    assert np.diff(sym_full(K).indptr).max() > fz.LONG_ROW
    a = lib.Symbolic(K).arrays()
    mf = MFNumpy(a, np.longdouble); mf.factor(K.data, gpu.Dsigns)
    assert mf.nreg == 0
    rx, rz = rng.standard_normal(data.n), rng.standard_normal(data.m)
    ref = mf.solve(np.r_[rx, rz]).astype(float)
    xg, zg = np.zeros(data.n), np.zeros(data.m)
    gpu.setrhs(rx, rz); assert gpu.solve(xg, zg)
    sc = np.abs(ref).max()
    assert np.abs(xg - ref[:n]).max() <= 1e-10 * sc and np.abs(zg - ref[n:n + m]).max() <= 1e-10 * sc
