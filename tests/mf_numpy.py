"""Test helper: numpy emulation of the multifrontal numeric phase on the product's symbolic
structures (panels, update blocks, a_map, rel).  It exercises exactly the index maps the CUDA
kernels use, so symbolic-analysis bugs are caught on the CPU.  Not part of the product.

With dtype=np.longdouble (x87 extended precision, 64-bit mantissa) it is the high-precision
reference the GPU kernel tests compare with: `gpu_storage` converts its factor into the exact
layout the kernels leave in device memory."""
import numpy as np

SB = 64          # width of the inverted diagonal blocks of L11 (kernels.cuh: SB == PB)


def panel_view(L, s, sn, nf, ns):
    """(ns, nf) view (transposed panel) of supernode sn; the panel is column-major with leading
    dimension panel_ld[sn] (>= nf: large fronts are padded)."""
    ld = int(s["panel_ld"][sn]) if "panel_ld" in s else nf
    off = int(s["panel_off"][sn])
    return L[off:off + ld * ns].reshape(ns, ld)[:, :nf]


class MFNumpy:
    def __init__(self, sym, dtype=np.float64):
        """sym: dict of arrays from cb200_symbolic_get (see lib.Symbolic.arrays())."""
        self.s = sym
        self.N = len(sym["perm"])
        self.nsuper = len(sym["sn_first"]) - 1
        self.dtype = dtype

    def factor(self, nzval, dsigns_orig, eps=1e-13, delta=2e-7, enable=True):
        """LDL' with QDLDL's sign rule: if D[k]*sign < eps then D[k] = delta*sign (when enabled).
        Counts the replaced pivots (nreg) and records their ORIGINAL indices (reglog, in order)."""
        s, T = self.s, self.dtype
        L = np.zeros(int(s["panel_off"][-1]), dtype=T)
        U = np.zeros(int(s["upd_off"][-1]), dtype=T)
        np.add.at(L, s["a_map"], np.asarray(nzval, dtype=np.float64).astype(T))
        D = np.zeros(self.N, dtype=T)
        dsp = np.asarray(dsigns_orig)[s["perm"]]
        eps, delta = T(eps), T(delta)
        self.nreg, self.reglog = 0, []
        for sn in range(self.nsuper):
            f, l = int(s["sn_first"][sn]), int(s["sn_first"][sn + 1])
            ns = l - f
            nr = int(s["rows_ptr"][sn + 1] - s["rows_ptr"][sn])
            nf = ns + nr
            F = np.zeros((nf, nf), dtype=T)
            F[:, :ns] = panel_view(L, s, sn, nf, ns).T
            for c in s["children"][sn]:
                nrc = int(s["rows_ptr"][c + 1] - s["rows_ptr"][c])
                rel = s["rel"][s["rows_ptr"][c]:s["rows_ptr"][c + 1]]
                Uc = U[s["upd_off"][c]:s["upd_off"][c] + nrc * nrc].reshape(nrc, nrc).T
                F[np.ix_(rel, rel)] += np.tril(Uc)
            for k in range(ns):
                d = F[k, k]
                if enable and d * dsp[f + k] < eps:
                    d = delta * dsp[f + k]; self.nreg += 1
                    self.reglog.append(int(s["perm"][f + k]))
                D[f + k] = d
                col = F[k + 1:, k].copy()
                F[k + 1:, k] = col / d
                F[k + 1:, k + 1:] -= np.tril(np.outer(col, col / d))
                F[k, k] = 1.0
            panel_view(L, s, sn, nf, ns)[:, :] = F[:, :ns].T
            if nr:
                U[s["upd_off"][sn]:s["upd_off"][sn] + nr * nr] = np.tril(F[ns:, ns:]).T.reshape(-1)
        self.L, self.D = L, D
        return D

    def solve(self, b):
        s = self.s
        y = np.asarray(b, dtype=np.float64).astype(self.dtype)[s["perm"]].copy()
        # forward (right-looking form; equivalent to the multifrontal form the kernels use)
        for sn in range(self.nsuper):
            f, l = int(s["sn_first"][sn]), int(s["sn_first"][sn + 1])
            ns = l - f
            rows = s["rows"][s["rows_ptr"][sn]:s["rows_ptr"][sn + 1]]
            nf = ns + len(rows)
            P = panel_view(self.L, s, sn, nf, ns).T
            for k in range(ns):
                y[f + k + 1:l] -= P[k + 1:ns, k] * y[f + k]
            y[rows] -= P[ns:, :] @ y[f:l]
        y /= self.D
        for sn in range(self.nsuper - 1, -1, -1):
            f, l = int(s["sn_first"][sn]), int(s["sn_first"][sn + 1])
            ns = l - f
            rows = s["rows"][s["rows_ptr"][sn]:s["rows_ptr"][sn + 1]]
            nf = ns + len(rows)
            P = panel_view(self.L, s, sn, nf, ns).T
            y[f:l] -= P[ns:, :].T @ y[rows]
            for k in range(ns - 1, -1, -1):
                y[f + k] -= P[k + 1:ns, k] @ y[f + k + 1:l]
        x = np.empty(self.N, dtype=self.dtype)
        x[s["perm"]] = y
        return x


def invert_unit_lower(T):
    """Inverse of a unit-lower-triangular block by row-wise forward substitution, in T's dtype
    (numpy's LAPACK path would round a longdouble block to double)."""
    n = T.shape[0]
    X = np.zeros_like(T)
    for i in range(n):
        X[i, i] = 1
        if i:
            X[i, :i] = -(T[i, :i] @ X[:i, :i])
    return X


def gpu_storage(mf):
    """The factor of `mf` in the device storage format of the panels (DESIGN.md section 3): every
    supernode's nf x ns panel column-major at panel_off with leading dimension panel_ld, D on the
    diagonal, and each diagonal block of L11 of up to SB columns (blocks start at column 0 of the
    supernode) replaced by the inverse of its unit-lower factor, computed in mf's dtype.  Entries
    above the diagonal of L11 and rows nf..ld-1 are set to 0; the kernels make no promise about
    the former (see the GPU tests) and leave the padding rows zero."""
    s = mf.s
    out = np.zeros_like(mf.L)
    for sn in range(mf.nsuper):
        f, l = int(s["sn_first"][sn]), int(s["sn_first"][sn + 1])
        ns = l - f
        nf = ns + int(s["rows_ptr"][sn + 1] - s["rows_ptr"][sn])
        P = np.tril(panel_view(mf.L, s, sn, nf, ns).T)          # nf x ns, unit diagonal
        for b0 in range(0, ns, SB):
            b1 = min(ns, b0 + SB)
            P[b0:b1, b0:b1] = invert_unit_lower(P[b0:b1, b0:b1])
        P[np.arange(ns), np.arange(ns)] = mf.D[f:l]
        panel_view(out, s, sn, nf, ns)[:, :] = P.T
    return out
