"""CPU: the extended-precision multifrontal reference (mf_numpy with np.longdouble) against the QDLDL
oracle and a dense solve, its storage-format conversion, and the front zoo's designed shapes and
kernel-path coverage (routing rules restated in front_zoo.route)."""
import numpy as np
import pytest
import front_zoo as fz
from common import sym_full, random_quasidefinite
from mf_numpy import MFNumpy, gpu_storage, panel_view, SB


@pytest.fixture
def zoo_env(monkeypatch):
    for k, v in fz.ZOO_ENV.items():
        monkeypatch.setenv(k, v)


def test_longdouble_is_extended_precision():
    assert np.finfo(np.longdouble).eps < 1e-18


@pytest.mark.parametrize("part", [d.name for d in fz.parts()])
def test_reference_solves_each_zoo_matrix(zoo_env, part):
    """the extended-precision reference runs on the product's symbolic maps (a_map, rel, children);
    a dense residual check of each zoo matrix makes the GPU comparisons independent of them"""
    from clarabel_jl_b200 import lib
    d = {d.name: d for d in fz.parts()}[part]
    K, sg, _ = d.build()
    mf = MFNumpy(lib.Symbolic(K, ordering=2).arrays(), np.longdouble)
    mf.factor(K.data, sg)
    assert mf.nreg == 0
    Kf = sym_full(K)
    b = np.random.default_rng(2).standard_normal(K.shape[0])
    x = mf.solve(b).astype(float)
    r = Kf @ x - b
    assert np.abs(r).max() <= 1e-14 * (abs(Kf) @ np.abs(x) + np.abs(b)).max()


@pytest.mark.parametrize("seed", range(0, 24, 3))
def test_longdouble_reference_matches_qdldl_and_dense_solve(seed):
    from clarabel_jl_b200 import lib
    from oracle import qdldl as oq
    K, Ds, rng = random_quasidefinite(seed)
    N = K.shape[0]
    b = rng.standard_normal(N)
    Kd = sym_full(K).toarray()
    xs = np.linalg.solve(Kd, b)
    F = oq.QDLDLFactorisation(K, Ds); assert F.refactor()
    xo = b.copy(); F.solve(xo)
    for ordering in (0, 2):
        a = lib.Symbolic(K, ordering=ordering, nd_leaf=8).arrays()
        mf = MFNumpy(a, np.longdouble)
        D = mf.factor(K.data, Ds)
        assert D.dtype == np.longdouble and mf.nreg == 0 and mf.reglog == []
        assert np.all(np.sign(D) == Ds[a["perm"]])
        x = mf.solve(b)
        sc = max(1.0, np.abs(xs).max())
        assert np.abs(x - xs).max() < 1e-9 * sc and np.abs(x - xo).max() < 1e-9 * sc
        # the extended-precision residual is far below what a double solve reaches
        r = Kd.astype(np.longdouble) @ x - b
        assert np.abs(r).max() < 1e-15 * sc * max(1.0, np.abs(Kd).max())


def test_sign_rule_count_log_and_settings(zoo_env):
    """the reference's regularisation: exact replacement, count, original indices, eps/delta and
    the enable switch taken from the caller"""
    from clarabel_jl_b200 import lib
    d = fz.part_reg()
    K, sg, _ = d.build()
    a = lib.Symbolic(K, ordering=2).arrays()
    want = d.reg_columns()
    mf = MFNumpy(a, np.longdouble)
    D = mf.factor(K.data, sg)
    pos = np.empty(d.N, dtype=np.int64); pos[a["perm"]] = np.arange(d.N)
    assert mf.nreg == len(want) and sorted(mf.reglog) == want
    assert np.all(D[pos[want]] == np.longdouble(2e-7) * sg[want])
    mf.factor(K.data, sg, delta=1e-3)
    assert np.all(mf.D[pos[want]] == np.longdouble(1e-3) * sg[want])
    with np.errstate(all="ignore"):
        mf.factor(K.data, sg, eps=11.0)       # every unreplaced pivot of the zoo has |D| < 11
    assert mf.nreg > len(want) and mf.D[0] == np.longdouble(2e-7) * sg[a["perm"][0]]
    with np.errstate(all="ignore"):
        mf.factor(K.data, sg, enable=False)
    assert mf.nreg == 0 and np.any(mf.D == 0)


def test_gpu_storage_format(zoo_env):
    """D on the diagonal, inverted unit-lower diagonal blocks of SB columns from column 0 of each
    supernode, plain L elsewhere, zero above the diagonal and in the padding rows"""
    from clarabel_jl_b200 import lib
    d = fz.part_large()
    K, sg, _ = d.build()
    a = lib.Symbolic(K, ordering=2).arrays()
    mf = MFNumpy(a, np.longdouble); mf.factor(K.data, sg)
    st = gpu_storage(mf)
    seen_pad = 0
    for sn in range(mf.nsuper):
        f, l = int(a["sn_first"][sn]), int(a["sn_first"][sn + 1]); ns = l - f
        nf = ns + int(a["rows_ptr"][sn + 1] - a["rows_ptr"][sn]); ld = int(a["panel_ld"][sn])
        P, Q = panel_view(st, a, sn, nf, ns).T, panel_view(mf.L, a, sn, nf, ns).T
        assert np.all(np.diag(P[:ns]) == mf.D[f:l])
        assert np.all(np.triu(P[:ns], 1) == 0)
        for b0 in range(0, ns, SB):
            b1 = min(ns, b0 + SB)
            Lb = np.tril(Q[b0:b1, b0:b1], -1) + np.eye(b1 - b0, dtype=np.longdouble)
            Xb = np.tril(P[b0:b1, b0:b1], -1) + np.eye(b1 - b0, dtype=np.longdouble)
            assert np.abs(Xb @ Lb - np.eye(b1 - b0)).max() < 1e-16
            assert np.array_equal(P[b1:, b0:b1], Q[b1:, b0:b1])
        off = int(a["panel_off"][sn])
        pad = st[off:off + ld * ns].reshape(ns, ld)[:, nf:]
        assert np.all(pad == 0); seen_pad += pad.size
    assert seen_pad > 0


# cells of the kernel-path table: (description, predicate over one routed front)
def _cells():
    c = []
    for nf in (1, 2, 16, 17, 32, 33, 63, 64):
        c.append(("small nf=%d ns=1" % nf, lambda f, nf=nf: f["kernel"].startswith("small") and f["nf"] == nf and f["ns"] == 1))
        c.append(("small nf=%d ns=nf" % nf, lambda f, nf=nf: f["kernel"].startswith("small") and f["nf"] == nf == f["ns"]))
    c.append(("small nr=0 root", lambda f: f["kernel"].startswith("small") and f["nr"] == 0))
    for nf in (65, 96, 97, 128, 129, 151, 152):
        c.append(("panel nf=%d" % nf, lambda f, nf=nf: f["kernel"].startswith("panel") and f["nf"] == nf))
    for ns in (1, 15, 16, 17, 63, 64, 65, 150):
        c.append(("panel ns=%d" % ns, lambda f, ns=ns: f["kernel"].startswith("panel") and f["ns"] == ns))
    for k in range(4):
        c.append(("panel class %d" % k, lambda f, k=k: f["kernel"] == "panel%d" % k))
    for nf in (151, 152):
        c.append(("small<256> nf=%d ns>=151" % nf, lambda f, nf=nf: f["kernel"] == "small5" and f["nf"] == nf and f["ns"] >= 151))
    for nf in (153, 160, 161, 257):
        c.append(("large nf=%d" % nf, lambda f, nf=nf: f["kernel"] == "large" and f["nf"] == nf))
    c.append(("large nf~600", lambda f: f["kernel"] == "large" and 560 <= f["nf"] <= 600))
    for ns in (1, 2, 63, 64, 65, 127, 128, 129, 200, 512):
        c.append(("large ns=%d" % ns, lambda f, ns=ns: f["kernel"] == "large" and f["ns"] == ns))
    for nr in (0, 1, 7, 63, 64, 65, 128, 129):
        c.append(("large nr=%d" % nr, lambda f, nr=nr: f["kernel"] == "large" and f["nr"] == nr))
    c.append(("large nf%8!=0", lambda f: f["kernel"] == "large" and f["nf"] % 8 != 0))
    c.append(("large ns%64!=0", lambda f: f["kernel"] == "large" and f["ns"] % 64 != 0 and f["ns"] > 64))
    c.append(("large parent with exactly 2048 children", lambda f: f["kernel"] == "large" and f["nchild"] == 2048 and not f["atomic"]))
    c.append(("large parent with 2049 children (atomic)", lambda f: f["kernel"] == "large" and f["nchild"] == 2049 and f["atomic"]))
    c.append(("parent with > 64 children", lambda f: f["nchild"] > 64))
    for sol in ("leaf", "warp16", "warp32", "cta", "big"):
        c.append(("solve " + sol, lambda f, sol=sol: f["solve"] == sol))
    return c


def _context_cells(fronts_by_part, arrays_by_part):
    """cells that relate fronts to each other (levels, parents)"""
    hit = set()
    for name, fr in fronts_by_part.items():
        a = arrays_by_part[name]
        par = a["sn_parent"]; lvl = a["sn_level"]
        by_level = {}
        for s, f in enumerate(fr):
            if f["kernel"] == "large":
                by_level.setdefault(int(lvl[s]), set()).add(f["ns"])
            p = par[s]
            if p >= 0:
                if f["kernel"] == "large" and fr[p]["kernel"].startswith("small"):
                    hit.add("large child of a small parent")
                if fr[p]["kernel"] == "large" and f["kernel"].startswith("small"):
                    hit.add("small child of a large parent")
                if fr[p]["kernel"] == "large" and f["kernel"].startswith("panel"):
                    hit.add("panel child of a large parent")
        if any(len(v) >= 3 for v in by_level.values()):
            hit.add("large fronts of different ns in one level")
    return hit


def test_zoo_shapes_and_kernel_path_coverage(zoo_env):
    from clarabel_jl_b200 import lib
    fronts, arrays, asm_fwd, long_row = {}, {}, set(), False
    for d in fz.parts():
        K, sg, _ = d.build()
        a = lib.Symbolic(K, ordering=2).arrays()
        fz.check_design(d, a)
        fr, asm, lr = fz.route(a, K)
        fronts[d.name], arrays[d.name] = fr, a
        asm_fwd |= asm; long_row |= lr
    allf = [f for fr in fronts.values() for f in fr]
    missed = [name for name, pred in _cells() if not any(pred(f) for f in allf)]
    assert missed == []
    ctx = _context_cells(fronts, arrays)
    assert ctx == {"large child of a small parent", "small child of a large parent",
                   "panel child of a large parent", "large fronts of different ns in one level"}
    assert asm_fwd == {1, 32, 256} and long_row
    # CB200_SUBTREE=1: the subtree part holds exactly one bottom subtree (21 supernodes), no other part any
    assert {name: sum(f["subtree_root"] for f in fr) for name, fr in fronts.items()} == \
        {name: int(name == "subtree") for name in fronts}
    # CB200_NO_PANEL=1: every panel front of the zoo goes to k_factor_small, classes 3..5
    panel_nf = {f["nf"] for f in allf if f["kernel"].startswith("panel")}
    assert {65, 96, 97, 128, 129, 151, 152} <= panel_nf
    d = fz.part_panel(); K, sg, _ = d.build()
    fr, _, _ = fz.route(lib.Symbolic(K, ordering=2).arrays(), K, fz.Options(no_panel=True))
    assert {f["kernel"] for f in fr if 64 < f["nf"] <= 152} == {"small3", "small4", "small5"}
