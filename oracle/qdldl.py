"""ctypes face of oracle/qdldl_oracle.c (QDLDL restatement) — TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, "qdldl_oracle.c"),
            os.path.join(_HERE, "..", "clarabel.jl_b200", "csrc", "ordering.cpp")]
    stale = (not os.path.exists(so)) or any(
        os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        # rebuilt when stale; a tree that cannot be written to (a read-only checkout the benchmark runs
        # from) uses the library build() left there
        L = C.CDLL(build() if os.access(_HERE, os.W_OK) or not os.path.exists(so) else so)
        I, D, P = C.c_int64, C.c_double, C.c_void_p
        L.qdldl_oracle_new.restype = P
        L.qdldl_oracle_new.argtypes = [I, P, P, P, P, P, D, D, C.c_int]
        L.qdldl_oracle_free.argtypes = [P]
        L.qdldl_oracle_update_values.argtypes = [P, P, P, I]
        L.qdldl_oracle_scale_values.argtypes = [P, P, I, D]
        L.qdldl_oracle_refactor.argtypes = [P]; L.qdldl_oracle_refactor.restype = C.c_int
        L.qdldl_oracle_solve.argtypes = [P, P]
        for f in ("nnzL", "nnzA", "regularize_count"):
            getattr(L, "qdldl_oracle_" + f).argtypes = [P]
            getattr(L, "qdldl_oracle_" + f).restype = I
        L.qdldl_oracle_sum_lnz_sq.argtypes = [P]; L.qdldl_oracle_sum_lnz_sq.restype = D
        for f in ("D", "Dinv", "Lp", "Li", "Lx", "perm"):
            getattr(L, "qdldl_oracle_" + f).argtypes = [P]
            getattr(L, "qdldl_oracle_" + f).restype = P
        L.cb200_order_amd.argtypes = [I, P, P, D, P]; L.cb200_order_amd.restype = C.c_int32
        L.cb200_order_nd.argtypes = [I, P, P, D, I, P]; L.cb200_order_nd.restype = C.c_int32
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def amd_order(K, dense_scale=1.5):
    """AMD-class ordering of the symmetric pattern of scipy CSC K (either triangle)."""
    n = K.shape[0]
    cp = np.ascontiguousarray(K.indptr, dtype=np.int64)
    ri = np.ascontiguousarray(K.indices, dtype=np.int64)
    perm = np.empty(n, dtype=np.int64)
    rc = lib().cb200_order_amd(n, _p(cp), _p(ri), float(dense_scale), _p(perm))
    assert rc == 0
    return perm


def nd_order(K, dense_scale=1.5, leaf_size=64):
    n = K.shape[0]
    cp = np.ascontiguousarray(K.indptr, dtype=np.int64)
    ri = np.ascontiguousarray(K.indices, dtype=np.int64)
    perm = np.empty(n, dtype=np.int64)
    rc = lib().cb200_order_nd(n, _p(cp), _p(ri), float(dense_scale), int(leaf_size), _p(perm))
    assert rc == 0
    return perm


class QDLDLFactorisation:
    """QDLDL.qdldl(K; perm, Dsigns, regularize_eps, regularize_delta, logical=true) as called at
    directldl_qdldl.jl:18-25.  K: scipy CSC upper triangular."""

    def __init__(self, K, Dsigns, eps=1e-13, delta=2e-7, perm=None, regularize=True):
        self.n = K.shape[0]
        self._cp = np.ascontiguousarray(K.indptr, dtype=np.int64)
        self._ri = np.ascontiguousarray(K.indices, dtype=np.int64)
        self._nz = np.ascontiguousarray(K.data, dtype=np.float64)
        if perm is None:
            perm = amd_order(K, 1.5)
        self.perm = np.ascontiguousarray(perm, dtype=np.int64)
        ds = np.ascontiguousarray(Dsigns, dtype=np.int64)
        self._h = lib().qdldl_oracle_new(self.n, _p(self._cp), _p(self._ri), _p(self._nz),
                                         _p(self.perm), _p(ds), eps, delta, int(regularize))
        self.nnzL = lib().qdldl_oracle_nnzL(self._h)
        self.nnzA = lib().qdldl_oracle_nnzA(self._h)
        self.sum_lnz_sq = lib().qdldl_oracle_sum_lnz_sq(self._h)

    def __del__(self):
        try:
            if self._h:
                lib().qdldl_oracle_free(self._h); self._h = None
        except Exception:
            pass

    def update_values(self, index, values):
        index = np.ascontiguousarray(index, dtype=np.int64)
        values = np.ascontiguousarray(values, dtype=np.float64)
        lib().qdldl_oracle_update_values(self._h, _p(index), _p(values), len(index))

    def scale_values(self, index, scale):
        index = np.ascontiguousarray(index, dtype=np.int64)
        lib().qdldl_oracle_scale_values(self._h, _p(index), len(index), float(scale))

    def refactor(self):
        return bool(lib().qdldl_oracle_refactor(self._h))

    def solve(self, x):
        assert x.dtype == np.float64 and x.flags.c_contiguous
        lib().qdldl_oracle_solve(self._h, _p(x))

    @property
    def regularize_count(self):
        return lib().qdldl_oracle_regularize_count(self._h)

    def _arr(self, name, n, dtype):
        ptr = getattr(lib(), "qdldl_oracle_" + name)(self._h)
        ct = C.c_double if dtype == np.float64 else C.c_int64
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(n,)).copy()

    def factors(self):
        """(Lp, Li, Lx, D, Dinv) copies — strictly-lower L in CSC, permuted coordinates."""
        n = self.n
        return (self._arr("Lp", n + 1, np.int64), self._arr("Li", self.nnzL, np.int64),
                self._arr("Lx", self.nnzL, np.float64), self._arr("D", n, np.float64),
                self._arr("Dinv", n, np.float64))
