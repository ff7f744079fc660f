"""Per-front child lists of the shared-memory front kernel (symbolic.h, Symbolic::kids).

k_factor_small adds the children's update blocks one child after the other, reading each child's
update-block offset, rel offset and nr from this list.  Expanded in numpy, the list must name each
front's children in child_list order and give exactly the (destination, source) pairs of the
destination-owner assembly maps (asm_colptr / asm_src / asm_child, expanded independently), each
destination summed in the same order.  Checked on every front of the zoo and on the fronts of C5
(all entries compared field by field, a sample expanded)."""
import numpy as np
import pytest
import front_zoo as fz


def _expand(a, kids, s):
    """(row, col, child, i, j, position) of every source of front s, from its child list, sorted by
    (row, col, position)"""
    rel = a["rel"]
    q0, q1 = a["child_ptr"][s], a["child_ptr"][s + 1]
    out = []
    for pos, q in enumerate(range(q0, q1)):
        uoff, roff, nrc = kids[q]
        r = rel[roff:roff + nrc]
        i, j = np.tril_indices(nrc)
        out.append(np.stack([r[i], r[j], np.full(len(i), a["child_list"][q]), i, j, np.full(len(i), pos)], 1))
    p = np.concatenate(out) if out else np.zeros((0, 6), np.int64)
    return p[np.lexsort((p[:, 5], p[:, 1], p[:, 0]))]


def _owner_pairs(a, m, s):
    """(row, col, child, i, j) of every source of front s from the destination-owner maps: destination
    column d takes the sources asm_src[asm_base[s] + asm_colptr[front_ptr[s] + d] ...) in list order,
    source q = child column j = q - rows_ptr[c] adding rows i >= j; sorted by (row, col), keeping that
    order within a destination"""
    rp, rel = a["rows_ptr"], a["rel"]
    nf = int(a["sn_first"][s + 1] - a["sn_first"][s] + rp[s + 1] - rp[s])
    cp = m["asm_colptr"][m["front_ptr"][s]:m["front_ptr"][s] + nf + 1]
    base = m["asm_base"][s]
    out = []
    for d in range(nf):
        for e in range(cp[d], cp[d + 1]):
            q, c = m["asm_src"][base + e], m["asm_child"][base + e]
            j = q - rp[c]
            assert rel[q] == d
            i = np.arange(j, rp[c + 1] - rp[c])
            out.append(np.stack([rel[rp[c] + i], np.full(len(i), d), np.full(len(i), c), i,
                                 np.full(len(i), j), np.full(len(i), len(out))], 1))
    p = np.concatenate(out) if out else np.zeros((0, 6), np.int64)
    return p[np.lexsort((p[:, 5], p[:, 1], p[:, 0]))][:, :5]


def check_lists(a, kids, maps, expand):
    cl = a["child_list"]
    assert kids.shape == (len(cl), 3)
    np.testing.assert_array_equal(kids[:, 0], a["upd_off"][cl])
    np.testing.assert_array_equal(kids[:, 1], a["rows_ptr"][cl])
    np.testing.assert_array_equal(kids[:, 2], np.diff(a["rows_ptr"])[cl])
    nf = np.diff(a["sn_first"]) + np.diff(a["rows_ptr"])
    for s in expand:
        e = _expand(a, kids, s)
        ref = _owner_pairs(a, maps, s)
        np.testing.assert_array_equal(e[:, :5], ref)   # same pairs, same per-destination order
        assert e.size == 0 or (e[:, 0].max() < nf[s] and np.all(e[:, 0] >= e[:, 1]))


@pytest.fixture
def zoo_env(monkeypatch):
    for k, v in fz.ZOO_ENV.items():
        monkeypatch.setenv(k, v)


def test_zoo(zoo_env):
    from clarabel_jl_b200 import lib
    for d in fz.parts():
        K, _, _ = d.build()
        S = lib.Symbolic(K, ordering=2)
        a = S.arrays()
        check_lists(a, S.kid_lists(), S.asm_maps(), range(S.stats["nsuper"]))


def test_c5():
    """C5 (the bench workload, AMD ordering): every entry, and the fronts of the shared-memory kernel
    with the most children expanded"""
    import clarabel_jl_b200 as cb
    from clarabel_jl_b200 import lib, problems as pr, kkt_assembly as ka
    P, q, A, b, K = pr.c5_block_angular()
    data = cb.problemdata.ProblemData(P, q, A, b, K, cb.Settings())
    KKT, _ = ka.assemble_kkt_matrix(data.P, data.A, cb.CompositeCone(data.cones))
    S = lib.Symbolic(KKT, ordering=0)
    a = S.arrays()
    nch = np.diff(a["child_ptr"])
    nf = np.diff(a["sn_first"]) + np.diff(a["rows_ptr"])
    small = np.flatnonzero((nf <= 64) & (nch > 0))
    assert len(small) > 50_000
    wide = small[np.argsort(-nch[small], kind="stable")[:200]]
    rng = np.random.default_rng(3)
    check_lists(a, S.kid_lists(), S.asm_maps(), np.r_[wide, rng.choice(small, 2000, replace=False)])
