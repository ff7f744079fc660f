"""Test helper: the "front zoo", KKT matrices whose supernodal fronts have designed shapes.

A design is a forest of nodes.  Node v owns ns_v consecutive columns that are dense among
themselves and densely coupled to nr_v rows R_v; R_v is a strict prefix of the parent's front
(the parent's columns, then the parent's rows), so the parent's first column is v's first row and
the parent's front has room for every update of v.  Under the natural ordering, with subtree
collapse and relaxed amalgamation turned off (ZOO_ENV), each node becomes exactly one supernode
with front nf = ns + nr: a child is never merged into its parent because its row count is smaller
than the parent's front.  `check_design` asserts this on the product's symbolic analysis.

Values: off-diagonal entry (i, j) is uniform in +-0.5 / max(deg_i, deg_j) (deg = entries of the
full row), the diagonal is sign * U[1, 10].  Every row is then strictly diagonally dominant, which
elimination preserves, so every pivot keeps its sign, |D| lies in about [0.5, 10.5] and |L| < 1.
Columns listed in `reg_zero` / `reg_wrong` are numerically decoupled (every off-diagonal value in
their row and column is exactly 0) with diagonal 0 / -sign * 3: their Schur pivot is that value
in every summation order, so the sign rule must replace it by delta * sign and nothing else changes.

The routing rules of the numeric factorisation and of the solves are restated in `route`
(symbolic.h front_to_panel / front_is_large, api_cuda.cu build_plans and launch_fwd_level) so that
a CPU test can assert which kernel classes a part reaches."""
import numpy as np
import scipy.sparse as sp

ZOO_ENV = {"CB200_COLLAPSE_NF": "0", "CB200_RELAX": "0,0,0,0,512"}
SMALL_NF = (16, 32, 64, 96, 128, 152)            # api_cuda.cu kSmallNf
PANEL_DOUBLES = (4096, 9000, 16000, 1 << 30)     # api_cuda.cu kPanelDoubles
MANY_CHILDREN = 2048                             # kernels.cuh
LONG_ROW = 2048                                  # kernels.cuh
SUB_MAXNF, SUB_MINSN = 192, 16                   # kernels.cuh SUB_MAXNF, api_cuda.cu build_plans MINSN


class Design:
    def __init__(self, name, seed):
        self.name, self.seed = name, seed
        self.nodes = []                          # [ns, parent, nr]
        self.reg_zero, self.reg_wrong = [], []   # (node, local column)
        self.scale_pow2 = 0                      # > 0: symmetric scaling by 2^U{-p..p}

    def node(self, ns, parent=None, nr=0):
        assert ns >= 1 and (parent is None) == (nr == 0)
        if parent is not None:
            pns, _, pnr = self.nodes[parent]
            assert 1 <= nr < pns + pnr, "rows must be a strict prefix of the parent's front"
        self.nodes.append([ns, parent, nr])
        return len(self.nodes) - 1

    def children(self, parent, count, ns, nr):
        for _ in range(count):
            self.node(ns, parent, nr if np.isscalar(nr) else nr[_])

    # ------------------------------------------------------------------ assembly of the matrix
    def build(self):
        """-> (K upper-triangular CSC, Dsigns, cols) ; cols[v] = the original indices of node v."""
        n = len(self.nodes)
        kids = [[] for _ in range(n)]
        for v, (_, p, _) in enumerate(self.nodes):
            if p is not None:
                kids[p].append(v)
        cols, nxt = [None] * n, 0
        order = []                                   # children before parents
        for r in [v for v in range(n) if self.nodes[v][1] is None]:
            stack = [(r, 0)]
            while stack:
                v, i = stack.pop()
                if i < len(kids[v]):
                    stack.append((v, i + 1)); stack.append((kids[v][i], 0))
                else:
                    order.append(v)
        for v in order:
            cols[v] = np.arange(nxt, nxt + self.nodes[v][0]); nxt += self.nodes[v][0]
        N = nxt
        front = [None] * n
        for v in reversed(order):                    # parents before children
            ns, p, nr = self.nodes[v]
            rows = np.empty(0, dtype=np.int64) if p is None else front[p][:nr]
            front[v] = np.concatenate([cols[v], rows])
        I, J = [], []
        for v in range(n):
            c, rows = cols[v], front[v][len(cols[v]):]
            a, b = np.triu_indices(len(c), 1)
            I.append(c[a]); J.append(c[b])
            if len(rows):
                I.append(np.repeat(c, len(rows))); J.append(np.tile(rows, len(c)))
        I = np.concatenate(I) if I else np.empty(0, dtype=np.int64)
        J = np.concatenate(J) if J else np.empty(0, dtype=np.int64)
        deg = np.bincount(np.r_[I, J], minlength=N) + 1
        rng = np.random.default_rng(self.seed)
        off = rng.uniform(-0.5, 0.5, len(I)) / np.maximum(deg[I], deg[J])
        sign = np.where(rng.random(N) < 0.5, -1, 1).astype(np.int64)
        diag = sign * rng.uniform(1.0, 10.0, N)
        for v, k in self.reg_zero + self.reg_wrong:
            g = cols[v][k]
            off[(I == g) | (J == g)] = 0.0
            diag[g] = 0.0 if (v, k) in self.reg_zero else -3.0 * sign[g]
        if self.scale_pow2:
            s = np.ldexp(1.0, rng.integers(-self.scale_pow2, self.scale_pow2 + 1, N))
            off = off * s[I] * s[J]; diag = diag * s * s
            self.scale = s
        else:
            self.scale = np.ones(N)
        K = sp.csc_matrix((np.r_[off, diag], (np.r_[I, np.arange(N)], np.r_[J, np.arange(N)])), shape=(N, N))
        K.sort_indices()
        self.cols, self.N = cols, N
        return K, sign, cols

    def reg_columns(self):
        """original indices of the pivots the sign rule must replace"""
        return sorted(int(self.cols[v][k]) for v, k in self.reg_zero + self.reg_wrong)


def check_design(d, arrays):
    """every node is one supernode with the designed front (columns in order, ns, nr)"""
    a = arrays
    pos = np.empty(d.N, dtype=np.int64); pos[a["perm"]] = np.arange(d.N)
    sn_of = np.repeat(np.arange(len(a["sn_first"]) - 1), np.diff(a["sn_first"]))
    for v, (ns, p, nr) in enumerate(d.nodes):
        q = pos[d.cols[v]]
        s = sn_of[q[0]]
        assert np.array_equal(q, np.arange(a["sn_first"][s], a["sn_first"][s + 1])), (d.name, v)
        assert a["rows_ptr"][s + 1] - a["rows_ptr"][s] == nr, (d.name, v)


# ---------------------------------------------------------------------- routing restated
class Options:
    def __init__(self, no_panel=False, panel_min_nf=64, panel_max_nf=152, small_max_nf=152):
        self.use_panel, self.pmin, self.pmax, self.smax = not no_panel, panel_min_nf, panel_max_nf, small_max_nf

    def to_panel(self, nf, ns):
        return self.use_panel and self.pmin < nf <= self.pmax and ns <= 150 and nf * ns + nf * 25 <= 27000

    def to_large(self, nf, ns):
        return nf > self.smax and not self.to_panel(nf, ns)


def route(arrays, K, opt=None):
    """Per supernode: (ns, nr, nf, factor kernel, solve class) and the per-part assembly / residual
    paths, by the rules of api_cuda.cu build_plans, factor_body and launch_fwd_level."""
    opt = opt or Options()
    a = arrays
    ns_ = np.diff(a["sn_first"]); nr_ = np.diff(a["rows_ptr"]); nch = np.diff(a["child_ptr"])
    fronts, big_levels = [], {}
    for s in range(len(ns_)):
        ns, nr = int(ns_[s]), int(nr_[s]); nf = ns + nr
        if opt.to_panel(nf, ns):
            kern = "panel%d" % next(c for c in range(4) if nf * ns + 25 * nf <= PANEL_DOUBLES[c])
        elif opt.to_large(nf, ns) or nf > SMALL_NF[-1]:
            kern = "large"
        else:
            kern = "small%d" % next(c for c in range(6) if nf <= SMALL_NF[c])
        leaf = ns == 1 and nch[s] == 0
        big = nf * ns >= 65536 and ns > 32
        sol = "leaf" if leaf else ("warp16" if ns <= 16 else "warp32") if (ns <= 32 and nf <= 192) else \
              ("big" if big else "cta")
        fronts.append(dict(ns=ns, nr=nr, nf=nf, kernel=kern, solve=sol, nchild=int(nch[s]),
                           atomic=kern == "large" and nch[s] > MANY_CHILDREN))
        if big:
            lv = int(a["sn_level"][s])
            src = (int(a["asm_base"][s + 1] - a["asm_base"][s]) if "asm_base" in a else
                   int(nr_[a["children"][s]].sum())) // nf
            b = big_levels.setdefault(lv, dict(src=0, many=False))
            b["src"] = max(b["src"], src); b["many"] |= bool(nch[s] > 64)
    asm_fwd = {256 if b["src"] >= 512 else 32 if b["many"] else 1 for b in big_levels.values()}
    # bottom subtrees of the CB200_SUBTREE=1 solves (build_plans): complete subtrees of narrow supernodes
    # (ns <= 32, nf <= SUB_MAXNF) within the shared-memory window, with at least SUB_MINSN supernodes
    n = len(ns_); par = a["sn_parent"]
    ok = np.ones(n, bool); wc = ns_.astype(np.int64).copy(); wr = nr_.astype(np.int64).copy()
    wp = ((ns_ + nr_) * ns_).astype(np.int64); cnt = np.ones(n, np.int64)
    for s in range(n):                                     # children precede parents
        if ns_[s] > 32 or ns_[s] + nr_[s] > SUB_MAXNF or wc[s] > 2048 or wr[s] > 6144 or wp[s] > 131072:
            ok[s] = False
        p = par[s]
        if p >= 0:
            wc[p] += wc[s]; wr[p] += wr[s]; wp[p] += wp[s]; cnt[p] += cnt[s]; ok[p] &= ok[s]
    for s in range(n):
        fronts[s]["subtree_root"] = bool(ok[s] and (par[s] < 0 or not ok[par[s]]) and cnt[s] >= SUB_MINSN)
    Kf = K + sp.triu(K, 1).T
    long_row = int(np.diff(Kf.tocsc().indptr).max(initial=0)) > LONG_ROW
    return fronts, asm_fwd, long_row


# ---------------------------------------------------------------------- the zoo
def part_small():
    d = Design("small", 11)
    top = d.node(64)                                          # nf = 64 = ns, nr = 0 root
    for nr in (1, 15, 16, 31, 32, 62, 63):                    # ns = 1, nf in {2, 16, 17, 32, 33, 63, 64}
        d.node(1, top, nr)
    for ns in (1, 2, 16, 17, 32, 33, 63):                     # ns = nf roots (nr = 0)
        d.node(ns)
    mid = d.node(20, d.node(40), 30)                          # warp32 front (ns 20, nf 50) with children
    d.node(5, mid, 12); d.node(3, mid, 49)                    # warp16
    return d


def part_panel():
    d = Design("panel", 12)
    top = d.node(152)                                          # k_factor_small<256>: nf 152, ns 152
    for ns, nr in ((1, 64), (15, 81), (16, 81), (17, 111), (63, 66), (64, 87), (65, 87),
                   (150, 1), (150, 2), (151, 1), (120, 9), (30, 98), (16, 50)):
        d.node(ns, top, nr)
    d.node(151)                                                # nf 151, ns 151
    return d


def part_large():
    d = Design("large", 13)
    P = d.node(200)                                            # large root, nr = 0
    for ns, nr in ((512, 88), (1, 152), (2, 158), (63, 98), (64, 129), (65, 128), (127, 130),
                   (128, 129), (129, 64), (250, 7), (150, 63), (100, 65), (160, 1)):
        d.node(ns, P, nr)                                      # large fronts of different ns, one level
    d.node(5, P, 10); d.node(20, P, 80)                        # small and panel children of a large parent
    d.node(153)                                                # nf 153, nr 0
    d.node(200, d.node(30), 20)                                # large child of a small parent
    return d


def part_many_children(nchild):
    """a big-solve root (ns 256) with `nchild` single-column children"""
    d = Design("children%d" % nchild, 14)
    P = d.node(256)
    if nchild > MANY_CHILDREN:                                 # >= 512 assembly sources per row
        d.children(P, nchild, 1, 64)
    else:
        d.children(P, nchild, 1, [1 + k % 4 for k in range(nchild)])
    return d


def part_subtree():
    """a complete subtree of 21 narrow supernodes (ns <= 32, nf <= 192) below a wide panel front:
    the bottom-subtree solve kernels (CB200_SUBTREE=1) take it whole"""
    d = Design("subtree", 17)
    top = d.node(100)
    root = d.node(24, top, 40)                                 # front 64
    for _ in range(4):
        c = d.node(8, root, 30)                                # front 38
        for nr in (10, 20, 30, 37):
            d.node(4, c, nr)
    return d


def part_scaled():
    """the large and panel shapes of a smaller tree, symmetrically scaled by powers of two so that
    D spans about 1e8.  Scaling by powers of two commutes with rounding: the computed factor is
    exactly the scaled factor of the unscaled matrix, so this part checks the scale-aware bounds
    and the dynamic range of the stored values, not the kernels' behaviour on ill-conditioned
    fronts (it adds no rounding stress of its own)."""
    d = Design("scaled", 15)
    P = d.node(180)
    d.node(130, P, 70); d.node(20, P, 100); d.node(3, P, 9)
    d.scale_pow2 = 7
    return d


def part_reg(extra=0):
    """pivots that are exactly 0 or of the wrong sign: first / last column of a small front,
    columns 15, 16, 17 of a panel front, columns 0, 63, 64 and one in the last partial block of a
    large front; `extra` more decoupled columns of the large front (more than 64 in total)"""
    d = Design("reg%d" % extra, 16)
    sm = d.node(40)
    d.reg_zero += [(sm, 0)]; d.reg_wrong += [(sm, 39)]
    pp = d.node(70)
    pn = d.node(40, pp, 60)
    d.reg_zero += [(pn, 15), (pn, 17)]; d.reg_wrong += [(pn, 16)]
    lg = d.node(200)
    d.reg_zero += [(lg, 0), (lg, 64)]; d.reg_wrong += [(lg, 63), (lg, 197)]
    taken = {0, 63, 64, 197}
    extra_cols = [k for k in range(1, 200) if k not in taken][:extra]
    d.reg_zero += [(lg, k) for k in extra_cols]
    d.node(10, lg, 150)                                        # a child assembling around the decoupled columns
    return d


def parts():
    return [part_small(), part_panel(), part_large(), part_many_children(2048),
            part_many_children(2049), part_subtree(), part_scaled()]
