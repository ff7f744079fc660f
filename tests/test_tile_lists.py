"""Per-tile source lists of the large-front extend-add (symbolic.h, build_tile_lists).

The Schur GEMM epilogue and k_assemble_tiles add the children's update blocks to a tile one
rectangle after the other.  Expanded in numpy, the rectangles must give exactly the (destination,
source) pairs of the destination-owner assembly, each destination summed in child_list order, and
the Schur list must be exactly the tiles the GEMM updates.  Checked for both tile sizes on the
designed fronts of test_gpu_schur_assembly.py and test_gpu_tile_assembly.py, on the zoo, and on the
large fronts of C5 (whole lists counted, the widest fronts expanded)."""
import numpy as np
import pytest
import front_zoo as fz
import test_gpu_schur_assembly as tsa
import test_gpu_tile_assembly as tta


def _large_batches(a, fronts):
    """the large fronts of each level, as build_plans batches them (widest first)"""
    lv = a["sn_level"]
    out = {}
    for s, fr in enumerate(fronts):
        if fr["kernel"] == "large":
            out.setdefault(int(lv[s]), []).append(s)
    return [sorted(v, key=lambda s: -fronts[s]["ns"]) for _, v in sorted(out.items())]


def _children(a, s):
    """children of s in child_list order (cb200_symbolic_get selector 11)"""
    return a["child_list"][a["child_ptr"][s]:a["child_ptr"][s + 1]]


def _pairs(a, s, lo, hi, active=None):
    """destination-owner pairs of front s with destination column in [lo, hi) from its active
    children: (row, col, child, i, j, position of the child in child_list order), sorted by
    (row, col, position)"""
    rp, rel = a["rows_ptr"], a["rel"]
    out = []
    for pos, c in enumerate(_children(a, s)):
        if active is not None and not active[c]:
            continue
        r = rel[rp[c]:rp[c + 1]]
        i, j = np.tril_indices(len(r))
        keep = (r[j] >= lo) & (r[j] < hi)
        i, j = i[keep], j[keep]
        out.append(np.stack([r[i], r[j], np.full(len(i), c), i, j, np.full(len(i), pos)], 1))
    p = np.concatenate(out) if out else np.zeros((0, 6), np.int64)
    return p[np.lexsort((p[:, 5], p[:, 1], p[:, 0]))]


def _expand(a, tiles, rects, t, T):
    """(row, col, child, i, j, rectangle) of tile t; asserts every destination lies in the tile"""
    rp, rel = a["rows_ptr"], a["rel"]
    ti, tj = tiles[t, 1], tiles[t, 2]
    out = []
    for q in range(tiles[t, 3], tiles[t + 1, 3]):
        c, ja, jb, ia, ib = rects[q]
        assert 0 <= ja < jb <= ib and ia < ib <= rp[c + 1] - rp[c]
        j, i = np.meshgrid(np.arange(ja, jb), np.arange(ia, ib), indexing="ij")
        keep = i >= j
        i, j = i[keep], j[keep]
        r = rel[rp[c]:rp[c + 1]]
        e = np.stack([r[i], r[j], np.full(len(i), c), i, j, np.full(len(i), q)], 1)
        assert np.all(e[:, 0] // T == ti) and np.all(e[:, 1] // T == tj)
        out.append(e)
    return out


def check_batch(S, a, batch, T, schur, gather=True, expand=None, active=None):
    """checks the lists of one batch; expand: the slots whose rectangles are expanded (all if None);
    active: per-supernode mask of the children assembled (multi-GPU).  Returns (tiles, rectangles)."""
    tiles, rects = S.tile_lists(batch, T, schur, gather, active)
    rp = a["rows_ptr"]
    ns_ = np.diff(a["sn_first"]); nr_ = np.diff(rp)
    nch = np.diff(a["child_ptr"])
    assert np.all(np.diff(tiles[:, 3]) >= 0) and tiles[-1, 3] == len(rects)
    by_slot = {}
    for t in range(len(tiles) - 1):
        by_slot.setdefault(int(tiles[t, 0]), []).append(t)
    assert list(by_slot) == sorted(by_slot)                                  # front by front
    for k, s in enumerate(batch):
        ns, nf = int(ns_[s]), int(ns_[s] + nr_[s])
        gathers = gather and nch[s] <= fz.MANY_CHILDREN
        ts = by_slot.get(k, [])
        got = [(int(tiles[t, 1]), int(tiles[t, 2])) for t in ts]
        if schur:
            want = [(ti, tj) for tj in range(ns // T, (nf - 1) // T + 1) for ti in range(tj, (nf - 1) // T + 1)] \
                if nf > ns else []
            assert got == want, (s, got[:5], want[:5])
            lo, hi = ns, nf
            if not gathers:
                assert all(tiles[t, 3] == tiles[t + 1, 3] for t in ts)           # updated in place
                continue
        else:
            if nch[s] > fz.MANY_CHILDREN:                                        # k_assemble_atomic
                assert not ts
                continue
            lo, hi = 0, ns if gathers else nf
            assert got == sorted(got, key=lambda x: (x[1], x[0]))                # column strip by column strip
        if expand is not None and k not in expand:
            continue
        ref = _pairs(a, s, lo, hi, active)
        if not schur:                                 # exactly the tiles some child reaches
            assert sorted(got) == sorted(set(zip((ref[:, 0] // T).tolist(), (ref[:, 1] // T).tolist())))
        e = [x for t in ts for x in _expand(a, tiles, rects, t, T)]
        e = np.concatenate(e) if e else np.zeros((0, 6), np.int64)
        e = e[np.lexsort((e[:, 5], e[:, 1], e[:, 0]))]                  # by rectangle within a destination
        np.testing.assert_array_equal(e[:, :5], ref[:, :5])    # same pairs, same per-destination order
    return len(tiles) - 1, len(rects)


def _check_design(design, T):
    from clarabel_jl_b200 import lib
    K, _, _ = design.build()
    S = lib.Symbolic(K, ordering=2)
    a = S.arrays()
    fronts, _, _ = fz.route(a, K)
    for batch in _large_batches(a, fronts):
        for schur in (True, False):
            for gather in (True, False):
                check_batch(S, a, batch, T, schur, gather)
    return S, a, fronts


@pytest.fixture
def zoo_env(monkeypatch):
    for k, v in fz.ZOO_ENV.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("T", [64, 128])
@pytest.mark.parametrize("part", list(tsa.PARTS) + list(tta.PARTS))
def test_designed_fronts(zoo_env, part, T):
    _check_design({**tsa.PARTS, **tta.PARTS}[part], T)


@pytest.mark.parametrize("T", [64, 128])
def test_multi_gpu_masks_drop_inactive_children(zoo_env, T):
    """multi-GPU: a rank assembles only the contributions of its active children.  Their rectangles
    are left out of the lists (the kernels process every listed rectangle, one barrier each), and
    what remains still gives each destination its active sources in child_list order.  Masks: the
    ranks of a two-way partition (top children on rank 0 only, as cb200_dist_init sets them) and
    random ones, for both the gather and the pre-assembled (replicated top front) lists."""
    from clarabel_jl_b200 import lib
    rng = np.random.default_rng(5)
    for d in (tta.PARTS["tiles"], tsa.PARTS["gather"]):
        K, _, _ = d.build()
        S = lib.Symbolic(K, ordering=2)
        a = S.arrays()
        fronts, _, _ = fz.route(a, K)
        owner, top, _ = S.partition(2)
        masks = [np.where(top, rank == 0, owner == rank) for rank in (0, 1)]
        masks += [rng.random(len(owner)) < 0.5 for _ in range(2)]
        dropped = 0
        for active in masks:
            for batch in _large_batches(a, fronts):
                for schur in (True, False):
                    for gather in (True, False):
                        check_batch(S, a, batch, T, schur, gather, active=active)
                _, r_all = S.tile_lists(batch, T, False, False)
                _, r_act = S.tile_lists(batch, T, False, False, active)
                assert np.all(active[r_act[:, 0]])
                dropped += len(r_all) - len(r_act)
        assert dropped > 0


@pytest.mark.parametrize("T", [64, 128])
def test_zoo(zoo_env, T):
    for d in fz.parts():
        _check_design(d, T)


@pytest.mark.parametrize("T", [64, 128])
def test_designed_tile_cases_are_reached(zoo_env, T):
    """the shapes test_gpu_tile_assembly.py is for are in its lists"""
    d = tta.PARTS["tiles"]
    S, a, fronts = _check_design(d, T)
    rp, rel = a["rows_ptr"], a["rel"]
    interleaved3 = col_only = unreached = many = 0
    for batch in _large_batches(a, fronts):
        tiles, rects = S.tile_lists(batch, T, True)
        for t in range(len(tiles) - 1):
            rs = rects[tiles[t, 3]:tiles[t + 1, 3]]
            unreached += len(rs) == 0 and fronts[batch[tiles[t, 0]]]["nchild"] <= fz.MANY_CHILDREN
            if len(rs) >= 3:
                owner = {}
                for c, ja, jb, ia, ib in rs:
                    for r in rel[rp[c] + ia:rp[c] + ib]:
                        owner[int(r)] = int(c)
                seq = [owner[r] for r in sorted(owner)]
                interleaved3 += len(set(seq)) >= 3 and sum(x != y for x, y in zip(seq, seq[1:])) >= 4
        # a child whose columns reach a Schur tile's column window but none of its rows
        for k, s in enumerate(batch):
            ns, nf = fronts[s]["ns"], fronts[s]["nf"]
            for c in a["children"][s]:
                r = rel[rp[c]:rp[c + 1]]
                for tj in range(ns // T, (nf - 1) // T + 1):
                    cols = r[(r >= max(ns, tj * T)) & (r < (tj + 1) * T)]
                    if len(cols):
                        col_only += any(not np.any((r >= ti * T) & (r < (ti + 1) * T))
                                        for ti in range(tj + 1, (nf - 1) // T + 1))
        fr = [fronts[s] for s in batch]
        many += any(f["nchild"] > fz.MANY_CHILDREN and f["nr"] > 0 for f in fr) and \
            any(f["nchild"] <= fz.MANY_CHILDREN and f["nr"] > 0 for f in fr)
    assert interleaved3 and col_only and unreached and many, (interleaved3, col_only, unreached, many)
    root = [s for s, f in enumerate(fronts) if a["sn_parent"][s] < 0 and f["kernel"] == "large"]
    assert len(root) == 1
    at, ar = S.tile_lists(root, 64, False)
    widest = max(len({int(c) for c in ar[at[t, 3]:at[t + 1, 3], 0]}) for t in range(len(at) - 1))
    assert widest >= 64                                         # a panel tile with 64 children


def test_c5_large_fronts():
    """C5 (the bench workload, AMD ordering): every batch's lists are consistent, the rectangles of
    every front cover its destination-owner pairs (counted), and the widest fronts are expanded"""
    import clarabel_jl_b200 as cb
    from clarabel_jl_b200 import lib, problems as pr, kkt_assembly as ka
    P, q, A, b, K = pr.c5_block_angular()
    data = cb.problemdata.ProblemData(P, q, A, b, K, cb.Settings())
    KKT, _ = ka.assemble_kkt_matrix(data.P, data.A, cb.CompositeCone(data.cones))
    S = lib.Symbolic(KKT, ordering=0)
    a = S.arrays()
    fronts, _, _ = fz.route(a, KKT)
    rp = a["rows_ptr"]; ns_ = np.diff(a["sn_first"])
    nr_ = np.diff(rp)
    totals = {}
    for T in (64, 128):
        tot = np.zeros(4, np.int64)
        for batch in _large_batches(a, fronts):
            wide = {k for k in range(len(batch)) if k < 2}                 # widest two of each level
            tot[:2] += check_batch(S, a, batch, T, True, expand=wide)
            if T == 64:
                tot[2:] += check_batch(S, a, batch, T, False, expand=wide)
            for schur in (True, False):
                tiles, rects = S.tile_lists(batch, T if schur else 64, schur)
                cnt = np.zeros(len(batch), np.int64)        # pairs covered, per front
                for t in range(len(tiles) - 1):
                    rs = rects[tiles[t, 3]:tiles[t + 1, 3]]
                    for c, ja, jb, ia, ib in rs:
                        j = np.arange(ja, jb)
                        cnt[tiles[t, 0]] += int(np.sum(ib - np.maximum(ia, j)))
                for k, s in enumerate(batch):
                    if fronts[s]["nchild"] > fz.MANY_CHILDREN:
                        continue
                    ns = int(ns_[s])
                    want = 0
                    for c in a["children"][s]:
                        r = a["rel"][rp[c]:rp[c + 1]]
                        cols = np.flatnonzero(r >= ns) if schur else np.flatnonzero(r < ns)
                        want += int(np.sum(len(r) - cols))
                    assert cnt[k] == want, (s, schur, cnt[k], want)
        totals[T] = tot
    print("C5 tile lists (Schur tiles, rectangles; assembly tiles, rectangles):", totals)
    assert 100_000 < totals[64][0] < 150_000
