"""Extended-precision references for the cone-block update, the static regularisation and the
refinement residual of the KKT backend.

Every helper starts from the state the device gets (the CompositeCone scaling fields, the assembled
K, the device's elimination order) and computes in np.longdouble (x87 extended, 64-bit mantissa),
so a kernel result can be compared entry by entry at a bound derived from FP64 rounding:

  * cone_entries / psd_columns: -Hs of every cone as K stores it (coneops_nncone.jl,
    coneops_socone.jl:161-187, directldl_datamaps.jl:61-79, skron! coneops_psdtrianglecone.jl:502-540);
  * static_eps: eps = c + p * max|diag K| (kktsolver_directldl.jl:297-310), in FP64 as the kernels do;
  * residual: e = b - K x on the unshifted K, with a per-row bound;
  * LDSolver: LDL' of K + eps * diag(Dsigns) in a given elimination order (mf_numpy, longdouble).
"""
import numpy as np

LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)


def _pk():
    from clarabel_jl_b200 import cones
    return cones


# ------------------------------------------------------------------ cone blocks
def cone_entries(cones, mp):
    """(positions in K.data, longdouble values) of every entry the Zero, NN and SOC cones own:
    their Hs blocks, and for SOCs of dimension > 4 the u / v expansion columns and D."""
    C = _pk()
    rc, rb = cones.rng_cones, cones.rng_blocks
    w = np.asarray(cones.w, dtype=LD)
    soc_k = {int(ci): k for k, ci in enumerate(cones.soc_cones)}
    pos, val = [], []
    for i, t in enumerate(cones.types):
        a, b = int(rc[i]), int(rc[i + 1])
        blk = mp.Hsblocks[rb[i]:rb[i + 1]]
        if t == C.ZERO:
            v = np.zeros(b - a, dtype=LD)
        elif t == C.NONNEG:
            v = -(w[a:b] ** 2)
        elif t == C.SOC:
            k = soc_k[i]
            e2 = LD(cones.soc_eta[k]) ** 2
            if cones.is_sparse[i]:
                v = np.full(b - a, -e2, dtype=LD)
                v[0] = -e2 * LD(cones.soc_d[k])
            else:
                # eta^2 (2 w w' - J), packed column-major upper, J = diag(1, -1, ..., -1)
                wc = w[a:b]
                v = []
                for col in range(b - a):
                    for row in range(col + 1):
                        h = 2 * wc[row] * wc[col]
                        if row == col:
                            h += -1 if col == 0 else 1
                        v.append(-h * e2)
                v = np.array(v, dtype=LD)
        else:
            continue
        pos.append(blk); val.append(v)
    off = 0
    for k in np.nonzero(cones.soc_sparse)[0]:
        a, b = int(cones.soc_ptr[k]), int(cones.soc_ptr[k + 1])
        me2 = -(LD(cones.soc_eta[k]) ** 2)
        pos += [mp.soc_u[off:off + b - a], mp.soc_v[off:off + b - a]]
        val += [np.asarray(cones.soc_u[a:b], dtype=LD) * me2, np.asarray(cones.soc_v[a:b], dtype=LD) * me2]
        off += b - a
    if cones.soc_sparse.any():
        e2 = np.asarray(cones.soc_eta[cones.soc_sparse], dtype=LD) ** 2
        D = np.empty(2 * len(e2), dtype=LD); D[0::2] = -e2; D[1::2] = e2
        pos.append(mp.soc_D); val.append(D)
    if not pos:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=LD)
    return np.concatenate(pos).astype(np.int64), np.concatenate(val)


def psd_cones(cones, mp):
    """[(cone index, side n, K.data positions of the packed triu Hs block, R)] for every PSD cone."""
    C = _pk()
    R = {}
    for g in cones.psd_groups:
        for j, ci in enumerate(g["cones"]):
            R[int(ci)] = g["R"][j]
    rb = cones.rng_blocks
    return [(i, int(cones.dims[i]), mp.Hsblocks[rb[i]:rb[i + 1]], R[i])
            for i in range(len(cones.types)) if cones.types[i] == C.PSD]


def _svec_pairs(n):
    ti, tj = np.tril_indices(n)
    return tj, ti                       # svec index p -> (i <= j), column-major packed upper


def skron_columns(A, cols):
    """Columns `cols` (ascending svec indices q) of triu(A (x)_s A): (offsets q(q+1)/2 + p into the packed
    block, values) with rows p = 0..q, in A's dtype.  Entry ((i,j),(k,l)) is
    c_ij c_kl (A_ik A_jl + A_il A_jk) / 2 with c = 1 on the diagonal and sqrt(2) off it."""
    T = A.dtype.type
    I, J = _svec_pairs(A.shape[0])
    c = np.where(I == J, T(1), np.sqrt(T(2)))
    offs, vals = [], []
    cols = np.asarray(cols, dtype=np.int64)
    for lo in range(0, len(cols), 64):
        Q = cols[lo:lo + 64]
        P = np.arange(int(Q.max()) + 1)
        k, l, i, j = I[Q][None, :], J[Q][None, :], I[P][:, None], J[P][:, None]
        V = (A[i, k] * A[j, l] + A[i, l] * A[j, k]) * c[P][:, None] * c[Q][None, :] / T(2)
        keep = P[:, None] <= Q[None, :]
        pq = (Q * (Q + 1) // 2)[None, :] + P[:, None]
        offs.append(pq.T[keep.T]); vals.append(V.T[keep.T])     # column by column, rows ascending
    return np.concatenate(offs), np.concatenate(vals)


def psd_columns(R, cols):
    """For the PSD cone with scaling R: (offsets into its packed Hs block, longdouble K values
    -skron(RR'), entrywise bound 4 (n + 2) eps (|R||R|' (x)_s |R||R|')) of the columns `cols`.  An FP64
    evaluation of RR' and of the skron products in any order is within the bound; an index error is
    O(1) relative and is not."""
    n = R.shape[0]
    Rl = np.asarray(R, dtype=LD)
    off, v = skron_columns(Rl @ Rl.T, cols)
    Ra = np.abs(R)
    _, bnd = skron_columns(Ra @ Ra.T, cols)
    return off, -v, 4 * (n + 2) * EPS * bnd


def psd_check_columns(ne, rng, full_upto=1275, nsample=96):
    """Columns to compare: all of them up to `full_upto`, otherwise the first and last 32 and a sample."""
    if ne <= full_upto:
        return np.arange(ne)
    mid = rng.choice(np.arange(32, ne - 32), size=nsample, replace=False)
    return np.unique(np.r_[np.arange(32), mid, np.arange(ne - 32, ne)])


def within_ulps(x, ref, k):
    """|x - ref| <= k * eps * |ref| entrywise (ref in longdouble)."""
    return np.abs(np.asarray(x, dtype=LD) - ref) <= k * EPS * np.abs(ref)


# ------------------------------------------------------------------ static regularisation
def static_eps(nz, diag_full, c, p):
    """c + p * max|nz[diag_full]| with the product and the sum rounded separately (FP64)."""
    m = np.float64(np.abs(nz[diag_full]).max()) if len(diag_full) else np.float64(0.0)
    return np.float64(c) + np.float64(p) * m


def shifted_values(nz, diag_full, Dsigns, eps):
    """nz with eps added to the diagonal entries of +1 sign and subtracted from the others (FP64)."""
    out = np.array(nz, dtype=np.float64)
    out[diag_full] = out[diag_full] + np.where(np.asarray(Dsigns) > 0, np.float64(eps), -np.float64(eps))
    return out


# ------------------------------------------------------------------ residual
def _sym_entries(K):
    """Entries (row, col, value) of the symmetric matrix whose upper triangle K (CSC) stores."""
    col = np.repeat(np.arange(K.shape[1]), np.diff(K.indptr))
    row = K.indices.astype(np.int64)
    off = row != col
    return np.r_[row, col[off]], np.r_[col, row[off]], np.r_[K.data, K.data[off]]


def row_lengths(K):
    """Stored entries per row of the symmetric matrix (explicit zeros included)."""
    r, _, _ = _sym_entries(K)
    return np.bincount(r, minlength=K.shape[0])


def sym_matvec(K, x):
    """K x in longdouble for the symmetric K stored as its upper triangle."""
    r, c, v = _sym_entries(K)
    xl = np.asarray(x, dtype=LD)
    out = np.zeros(K.shape[0], dtype=LD)
    np.add.at(out, r, np.asarray(v, dtype=LD) * xl[c])
    return out


def residual(K, x, b):
    """(e = b - K x in longdouble, per-row bound (len_i + 2) eps (|b_i| + sum_j |K_ij| |x_j|)) for the
    symmetric K stored as its upper triangle.  Any FP64 summation order of row i is within the bound."""
    r, c, v = _sym_entries(K)
    xl = np.asarray(x, dtype=LD)
    absKx = np.zeros(K.shape[0], dtype=LD)
    np.add.at(absKx, r, np.abs(np.asarray(v, dtype=LD) * xl[c]))
    e = np.asarray(b, dtype=LD) - sym_matvec(K, x)
    bound = (row_lengths(K) + 2) * EPS * (np.abs(np.asarray(b, dtype=LD)) + absKx)
    return e, bound


# ------------------------------------------------------------------ factor and solve
class LDSolver:
    """LDL' of K + eps * diag(Dsigns) (K: upper CSC with the diagonal last in every column) in the
    elimination order `perm` (download selector 3), factored and solved in longdouble by mf_numpy with
    the dynamic regularisation rule of the kernels.  D is in elimination order, as selector 1."""

    def __init__(self, K, Dsigns, perm, eps=0.0, dyn_eps=1e-13, dyn_delta=2e-7):
        from clarabel_jl_b200 import lib
        from mf_numpy import MFNumpy
        perm = np.asarray(perm, dtype=np.int64)
        sym = lib.Symbolic(K, perm=perm).arrays()
        assert np.array_equal(sym["perm"], perm)
        diag = K.indptr[1:] - 1
        self.nz = shifted_values(K.data, diag, Dsigns, eps) if eps else np.array(K.data, dtype=np.float64)
        self.mf = MFNumpy(sym, dtype=LD)
        self.D = self.mf.factor(self.nz, Dsigns, eps=dyn_eps, delta=dyn_delta)
        self.nreg = self.mf.nreg

    def solve(self, b):
        return self.mf.solve(b)
