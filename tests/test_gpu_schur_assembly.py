"""Assembly of the update blocks U of large fronts.

A gather front (at most MANY_CHILDREN children) builds every Schur tile of its U from the children's
update blocks in the epilogue of the Schur GEMM; a front with more children is zeroed, assembled
with FP64 atomics and updated in place.  The designs here reach what the zoo of test_gpu_kernels.py
does not: gather tiles that straddle the ns boundary, U rows no child contributes to (they must come
out as exactly -L21 D L21'), rows of two children interleaved inside one tile, and a non-root front
with more than MANY_CHILDREN children and nr > 0 (the in-place epilogue on one GPU), next to a gather
front of the same level.  The shape properties are asserted on the CPU; D and the panel storage are
compared with the extended-precision reference at 1e-12 on the GPU."""
import numpy as np
import pytest
import scipy.sparse as sp
import front_zoo as fz
import test_gpu_kernels as tgk


class RowDesign(fz.Design):
    """A Design whose nodes may take any subset of the parent's front as their rows (`sel`: sorted
    positions in the parent's front, starting with 0, the parent's first column, so that the
    parent stays one supernode) instead of a prefix."""

    def node(self, ns, parent=None, nr=0, sel=None):
        if sel is not None:
            sel = np.asarray(sel, dtype=np.int64)
            assert sel[0] == 0 and np.all(np.diff(sel) > 0)
            nr = len(sel)
        v = super().node(ns, parent, nr)
        self.__dict__.setdefault("sel", {})[v] = sel
        return v

    def build(self):
        n = len(self.nodes)
        kids = [[] for _ in range(n)]
        for v, node in enumerate(self.nodes):
            if node[1] is not None:
                kids[node[1]].append(v)
        order = []                                   # children before parents
        for r in [v for v in range(n) if self.nodes[v][1] is None]:
            stack = [(r, 0)]
            while stack:
                v, i = stack.pop()
                if i < len(kids[v]):
                    stack.append((v, i + 1)); stack.append((kids[v][i], 0))
                else:
                    order.append(v)
        cols, nxt = [None] * n, 0
        for v in order:
            cols[v] = np.arange(nxt, nxt + self.nodes[v][0]); nxt += self.nodes[v][0]
        N = nxt
        front = [None] * n
        for v in reversed(order):                    # parents before children
            ns, p, nr = self.nodes[v]
            sel = self.sel.get(v)
            rows = np.empty(0, np.int64) if p is None else (front[p][:nr] if sel is None else front[p][sel])
            front[v] = np.concatenate([cols[v], rows])
        I, J = [], []
        for v in range(n):
            c, rows = cols[v], front[v][len(cols[v]):]
            a, b = np.triu_indices(len(c), 1)
            I.append(c[a]); J.append(c[b])
            if len(rows):
                I.append(np.repeat(c, len(rows))); J.append(np.tile(rows, len(c)))
        I, J = np.concatenate(I), np.concatenate(J)
        deg = np.bincount(np.r_[I, J], minlength=N) + 1
        rng = np.random.default_rng(self.seed)
        off = rng.uniform(-0.5, 0.5, len(I)) / np.maximum(deg[I], deg[J])
        sign = np.where(rng.random(N) < 0.5, -1, 1).astype(np.int64)
        diag = sign * rng.uniform(1.0, 10.0, N)
        K = sp.csc_matrix((np.r_[off, diag], (np.r_[I, np.arange(N)], np.r_[J, np.arange(N)])), shape=(N, N))
        K.sort_indices()
        self.cols, self.N, self.scale = cols, N, np.ones(N)
        return K, sign, cols


def part_gather():
    """P (ns 100, nr 300) under a root: its children take the even and the odd U rows of P's front
    below 400 and 300, and a prefix of 250 rows; U rows 300..399 of odd position are nobody's"""
    d = RowDesign("gather", 21)
    R = d.node(310)
    P = d.node(100, R, 300)
    d.node(8, P, sel=np.r_[0, np.arange(100, 400, 2)])
    d.node(12, P, sel=np.r_[0, np.arange(101, 300, 2)])
    d.node(4, P, 250)
    d.node(30, d.node(6, P, 170), 90)                          # a large child with a child of its own
    return d


def part_many_children_nonroot():
    """Q (ns 64, nr 100, 2049 single-column children that reach into its U) and a gather front G of
    the same level, both under one root"""
    d = RowDesign("many_children_nonroot", 22)
    R = d.node(200)
    Q = d.node(64, R, 100)
    d.children(Q, fz.MANY_CHILDREN + 1, 1, [60 + k % 50 for k in range(fz.MANY_CHILDREN + 1)])
    G = d.node(40, R, 150)
    d.node(3, G, sel=np.r_[0, np.arange(40, 190, 3)]); d.node(2, G, 120)
    return d


PARTS = {d.name: d for d in (part_gather(), part_many_children_nonroot())}


def _fronts(design):
    from clarabel_jl_b200 import lib
    K, _, _ = design.build()
    a = lib.Symbolic(K, ordering=2).arrays()
    fz.check_design(design, a)
    fronts, _, _ = fz.route(a, K)
    return a, fronts


@pytest.mark.parametrize("T", [64, 128])
def test_gather_fronts_have_the_designed_tiles(monkeypatch, T):
    for k, v in fz.ZOO_ENV.items():
        monkeypatch.setenv(k, v)
    a, fronts = _fronts(PARTS["gather"])
    rp, rel = a["rows_ptr"], a["rel"]
    straddle = uncovered = interleaved = 0
    for s, fr in enumerate(fronts):
        if fr["kernel"] != "large" or fr["nr"] == 0 or fr["atomic"]:
            continue
        ns, nf = fr["ns"], fr["nf"]
        owner = np.full(nf, -1)                                # child whose rows land on each front row (-2: several)
        covered = np.zeros(nf, bool)
        for c in a["children"][s]:
            r = rel[rp[c]:rp[c + 1]]
            covered[r] = True
            owner[r] = np.where(owner[r] == -1, c, -2)
        for tj in range(ns // T, (nf - 1) // T + 1):
            straddle += tj * T < ns < (tj + 1) * T
            for ti in range(tj, (nf - 1) // T + 1):
                rows = np.arange(max(ti * T, ns), min((ti + 1) * T, nf))
                uncovered += int(np.any(~covered[rows]))
                o = owner[rows]; o = o[o >= 0]
                interleaved += int(np.count_nonzero(np.diff(o)) >= 2)     # c1 c2 c1 at least
    assert straddle and uncovered and interleaved, (straddle, uncovered, interleaved)


def test_many_children_front_is_not_the_root_and_has_an_update_block(monkeypatch):
    for k, v in fz.ZOO_ENV.items():
        monkeypatch.setenv(k, v)
    a, fronts = _fronts(PARTS["many_children_nonroot"])
    atomic = [s for s, fr in enumerate(fronts) if fr["atomic"]]
    assert len(atomic) == 1
    s = atomic[0]
    assert fronts[s]["nr"] > 0 and a["sn_parent"][s] >= 0
    lv = a["sn_level"][s]
    assert any(fr["kernel"] == "large" and not fr["atomic"] and fr["nr"] > 0 and a["sn_level"][g] == lv
               for g, fr in enumerate(fronts))                # a gather front in the same batch
    rp = a["rows_ptr"]
    rows = np.concatenate([a["rel"][rp[c]:rp[c + 1]] for c in a["children"][s]])
    assert rows.max() >= fronts[s]["ns"]                       # the children reach into U


VARIANTS = {"default": {}, "tma_tile128": {"CB200_TMA_TILE": "128"}, "ldg_gemm": {"CB200_NO_TMA": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("part", list(PARTS))
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_factor_parity(monkeypatch, variant, part):
    env = VARIANTS[variant]
    tgk._set_env(monkeypatch, env)
    R = tgk.reference(PARTS[part], env)
    h = tgk._handle(R["K"], R["sg"])
    assert h.refactor()
    tgk.check_factor(h, R)
    assert h.download(5, 1)[0] == 0
    tgk.check_solves(h, R, PARTS[part])
    assert h.stats()["use_tma"] == (0 if env.get("CB200_NO_TMA") == "1" else 1)
