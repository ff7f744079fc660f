"""`B200KKTSolver`: the AbstractKKTSolver implementation over the C-ABI.

Mirrors the 6-method interface of src/kktsolvers/kktsolver_defaults.jl:1-47 and the constructor
signature `DirectLDLKKTSolver{T}(P, A, cones, m, n, settings)` (kktsolver_directldl.jl:46-52).
Assembly of the KKT pattern and of the index maps stays on the host (setup-time, as in the
reference); everything per-iteration runs on the device:

    update(cones)  -> cb200_update_cones   (H2D of the NT scaling state, G1/G2 value update,
                                            G3 static regularisation, G4-G6 factorisation)
    setrhs + solve -> cb200_solve_ir       (G7 triangular solves, G8 residuals, IR loop)

`B200DirectLDLSolver` below is the INNER boundary (AbstractDirectLDLSolver, the reference's own
plugin registry: directldl_defaults.jl:1-72), kept so that the stock DirectLDLKKTSolver logic
(oracle/kktsolver_oracle.py in this repo's tests) can drive the device factorisation through
update_values!/scale_values!/refactor!/solve! exactly as it drives QDLDL.
"""
import ctypes as C
import os
import sys
import numpy as np

from . import lib as _lib
from .kkt_assembly import assemble_kkt_matrix, fill_Dsigns
from .kktsystem import register_kktsolver


class LinearSolverInfo:
    """LinearSolverInfo(name, threads, direct, nnzA, nnzL)  (src/types.jl:198-206)."""
    def __init__(self, name, threads, direct, nnzA, nnzL):
        self.name, self.threads, self.direct, self.nnzA, self.nnzL = name, threads, direct, nnzA, nnzL


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


class B200DirectLDLSolver:
    """INNER boundary: ldlsolver_constructor(::Val{:b200}), ldlsolver_matrix_shape = :triu."""
    matrix_shape = "triu"

    def __init__(self, KKT, Dsigns, settings, **cs_over):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        cs = _lib.make_settings(settings, **cs_over)
        self._keep = (_i64(KKT.indptr), _i64(KKT.indices), _c64(KKT.data), _i64(Dsigns))
        cp, ri, nz, ds = self._keep
        _lib.check(self._L.cb200_create(KKT.shape[0], _p(cp), _p(ri), _p(nz), _p(ds), C.byref(cs),
                                        C.byref(self._h)), "cb200_create")
        self.N = KKT.shape[0]

    def __del__(self):
        try:
            if self._h:
                self._L.cb200_destroy(self._h); self._h = None
        except Exception:
            pass

    def update_values(self, index, values):
        index, values = _i64(index), _c64(values)
        _lib.check(self._L.cb200_update_values(self._h, _p(index), _p(values), len(index)),
                   "cb200_update_values")

    def scale_values(self, index, scale):
        index = _i64(index)
        _lib.check(self._L.cb200_scale_values(self._h, _p(index), len(index), float(scale)),
                   "cb200_scale_values")

    def refactor(self):
        return _lib.check(self._L.cb200_refactor(self._h), "cb200_refactor")

    def solve(self, x, b=None):
        """solve!(s, KKT, x, b); with b=None solves in place (QDLDL.jl convention)."""
        bb = _c64(x.copy() if b is None else b)
        assert x.dtype == np.float64 and x.flags.c_contiguous
        _lib.check(self._L.cb200_solve(self._h, _p(x), _p(bb)), "cb200_solve")

    def solve_multi(self, X, B):
        """cb200_solve_multi: X[:, j] = K^-1 B[:, j] for every column of the N x k arrays, one pass over L per
        sweep of up to 4 columns.  Both arrays in Fortran (column-major) order; X is written in place."""
        B = np.asfortranarray(B, dtype=np.float64)
        assert X.dtype == np.float64 and X.flags.f_contiguous and X.shape == B.shape and B.shape[0] == self.N
        _lib.check(self._L.cb200_solve_multi(self._h, B.shape[1], _p(X), self.N, _p(B), self.N), "cb200_solve_multi")

    def info(self):
        a, l, g = C.c_int64(), C.c_int64(), C.c_int32()
        self._L.cb200_info(self._h, C.byref(a), C.byref(l), C.byref(g))
        return LinearSolverInfo("b200", g.value, True, a.value, l.value)

    linear_solver_info = info

    def download(self, what, n):
        out = np.empty(n)
        _lib.check(self._L.cb200_download(self._h, what, _p(out), n), "cb200_download")
        return out

    def timers(self):
        out = np.zeros(12)
        self._L.cb200_get_timers(self._h, _p(out), 12)
        return dict(cone_ms=out[0], factor_ms=out[1], solve_ms=out[2], spmv_ms=out[3],
                    nfactor=int(out[4]), nsolve=int(out[5]), nlaunch=int(out[6]),
                    schur_ms=out[7], panel_ms=out[8], small_ms=out[9], asm_ms=out[10], scale_ms=out[11])

    def set_detail(self, level):
        """0 off, 1 (or True) factorisation groups, 2 every kernel class (see fine_timers)."""
        self._L.cb200_set_detail(self._h, int(level))

    def fine_timers(self):
        """{kernel class: accumulated ms} recorded while set_detail(2) was on."""
        n = self._L.cb200_get_fine_timers(self._h, None, 0)
        out = np.zeros(n)
        self._L.cb200_get_fine_timers(self._h, _p(out), n)
        return {self._L.cb200_fine_timer_name(i).decode(): float(out[i]) for i in range(n)}

    def stats(self):
        out = np.zeros(26)
        self._L.cb200_get_stats(self._h, _p(out), 26)
        keys = ["flops", "schur_flops", "panel_flops", "nnzL", "nlevels", "nsuper", "nlarge",
                "big_solve_bytes", "upd_bytes", "panel_bytes", "ordering_used", "rank_flops", "use_tma", "tma_kmajor",
                "factor_graphs", "solve_graph", "subtrees", "schur_tiles", "schur_rects", "asm_tiles", "asm_rects",
                "multi_sweeps", "multi_percol", "psd_scale_smem", "psd_scale_global", "jacobi_sweeps"]
        return dict(zip(keys, out.tolist()))

    def reset_timers(self):
        self._L.cb200_reset_timers(self._h)

    def dist_init(self, rank, nranks, uid):
        """Multi-GPU: join the NCCL communicator (uid: 128 bytes from nccl_unique_id() on rank 0)."""
        buf = C.create_string_buffer(bytes(uid), 128)
        _lib.check(self._L.cb200_dist_init(self._h, int(rank), int(nranks), buf), "cb200_dist_init")

    def stream_ptr(self):
        return self._L.cb200_get_stream(self._h)

    resident = False

    def set_resident(self, flag):
        """Device-resident mode (include/clarabel_b200.h): pointer arguments of update_cones / setrhs are
        then device pointers (B200KKTSolver.update_staged / setrhs_staged) or NULL (keep the state)."""
        self.resident = bool(flag)
        self._L.cb200_set_resident(self._h, int(bool(flag)))


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    _lib.check(_lib.lib().cb200_nccl_unique_id(buf), "cb200_nccl_unique_id")
    return bytes(buf.raw)


def dist_init_from_torch(ldl):
    """Join all ranks of the default torch.distributed group (one process per GPU)."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    obj = [nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    ldl.dist_init(rank, world, obj[0])


def nonsym_update_index(mp, cones):
    """0-based K.data positions of every value the nonsymmetric cones own, in the order
    nonsym_update_values() lists them: Hs blocks in cone order, then genpow q, r, p, D."""
    hs = [mp.Hsblocks[cones.rng_blocks[i]:cones.rng_blocks[i + 1]] for i, _ in cones.nonsym]
    return _i64(np.concatenate(hs + [mp.gp_q, mp.gp_r, mp.gp_p, mp.gp_D]))


def nonsym_update_values(mp, cones):
    """The matching K values: -Hs (get_Hs! then `values *= -1`, kktsolver_directldl.jl:219-226),
    the expansion columns scaled by -sqrt(mu) and D = (-1,-1,+1) (directldl_datamaps.jl:146-166)."""
    blk = cones.export_nonsymmetric_blocks()
    ngp = len(mp.gp_D) // 3
    return _c64(np.concatenate([-blk["hs"], blk["q"], blk["r"], blk["p"],
                                np.tile([-1.0, -1.0, 1.0], ngp)]))


class B200KKTSolver:
    """OUTER boundary: AbstractKKTSolver over the fused C-ABI entry points."""

    def __init__(self, P, A, cones, m, n, settings, **cs_over):
        self.m, self.n = m, n
        self.settings = settings
        self.KKT, self.map = assemble_kkt_matrix(P, A, cones)
        self.p = cones.p
        self.Dsigns = fill_Dsigns(m, n, self.p, cones)
        # Ordering: left to the library (cb200_settings.ordering = 1, auto).  It detects dense PSD cone
        # blocks from the pattern + Dsigns and then eliminates the variables coupled to them first and
        # dissects the block graph (or falls back to the AMD-class order for a handful of blocks); see
        # cb200_create in csrc/api_cuda.cu and DESIGN.md section 5.  The Julia shim gets the same rule.
        if "device" not in cs_over:
            cs_over = dict(cs_over, device=int(os.environ.get("LOCAL_RANK", "0")))
        self.ldl = B200DirectLDLSolver(self.KKT, self.Dsigns, settings, **cs_over)
        # one process per GPU: if the caller runs under torch.distributed, shard the elimination
        # tree over the ranks (every rank must then make the same calls with the same inputs)
        # (a process group can only be initialised if torch is already imported: do not pay the
        # torch import in single-GPU callers)
        if "torch" in sys.modules:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                dist_init_from_torch(self.ldl)
        L, h = self.ldl._L, self.ldl._h
        mp = self.map
        ctype = np.ascontiguousarray(cones.types, dtype=np.int32)
        cdim = _i64(cones.dims)
        self._maps = [_i64(mp.P), _i64(mp.A), _i64(mp.Hsblocks), _i64(mp.diag_full),
                      _i64(mp.soc_u), _i64(mp.soc_v), _i64(mp.soc_D)]
        mP, mA, mH, mD, mu, mv, mDD = self._maps
        _lib.check(L.cb200_set_maps(h, n, m, self.p, _p(mP), len(mP), _p(mA), len(mA), _p(mH), len(mH),
                                    _p(mD), len(ctype), _p(ctype), _p(cdim), _p(mu), _p(mv), _p(mDD)),
                   "cb200_set_maps")
        self.ir_rounds = 0; self.n_solves = 0

    def linear_solver_info(self):
        return self.ldl.info()

    def update(self, cones):
        if getattr(cones, "nonsym", None):
            # exp / pow / genpow blocks are host-computed (their scaling is not an NT scaling):
            # -Hs, the scaled expansion columns and D go in with one update_values! call
            if not hasattr(self, "_ns_idx"):
                self._ns_idx = nonsym_update_index(self.map, cones)
            self.ldl.update_values(self._ns_idx, nonsym_update_values(self.map, cones))
        if self.ldl.resident or self._state_on_device:
            # resident mode reads no host array, and after update_scaling the device already holds the state:
            # refactor from the state in HBM
            self._state_on_device = False
            return _lib.check(self.ldl._L.cb200_update_cones(self.ldl._h, *([None] * 6)), "cb200_update_cones")
        st = cones.export_state()
        arrs = [_c64(st[k]) for k in ("w", "soc_eta", "soc_d", "soc_u", "soc_v", "psd_R")]
        return _lib.check(self.ldl._L.cb200_update_cones(self.ldl._h, *[_p(a) for a in arrs]),
                          "cb200_update_cones")

    STATE_KEYS = ("w", "soc_eta", "soc_d", "soc_u", "soc_v", "psd_R")
    _state_on_device = False

    def update_scaling(self, s, z, cones):
        """update_scaling! of the symmetric cones on the device (cb200_update_scaling).  The state goes back into
        the CompositeCone fields the host cone operations read (w, lam, soc_eta/d/u/v, psd_groups R / Rinv / lam),
        and the next update(cones) refactors from the device copy instead of uploading it.  Returns ok_scale:
        False exactly where cones.update_scaling returns False.  In resident mode s and z are device addresses
        (int) and nothing is downloaded."""
        L, h = self.ldl._L, self.ldl._h
        ok = C.c_int32(0)
        if self.ldl.resident:
            _lib.check(L.cb200_update_scaling(h, C.c_void_p(s), C.c_void_p(z), C.byref(ok)), "cb200_update_scaling")
            return bool(ok.value)
        sv, zv = _c64(s), _c64(z)
        _lib.check(L.cb200_update_scaling(h, _p(sv), _p(zv), C.byref(ok)), "cb200_update_scaling")
        if not ok.value:
            return False
        self.download_scaling(cones)
        self._state_on_device = True
        return True

    def download_scaling(self, cones):
        """Copy the device scaling state into the CompositeCone fields (cb200_get_scaling)."""
        if not hasattr(self, "_psd_slots"):
            # (group, position in group, side) of every PSD cone in cone order: the device keeps them in cone order
            slot = {}
            for gi, g in enumerate(cones.psd_groups):
                for j, ci in enumerate(g["cones"]):
                    slot[int(ci)] = (gi, j, g["n"])
            self._psd_slots = [slot[i] for i in sorted(slot)]
            self._psd_rtotal = sum(n * n for _, _, n in self._psd_slots)
            self._psd_ltotal = sum(n for _, _, n in self._psd_slots)
            # rows of w / λ that update_scaling writes (NN and SOC); the others keep their host values
            self._wl_rows = np.zeros(cones.numel, dtype=bool)
            self._wl_rows[cones.nn_idx] = True; self._wl_rows[cones.soc_idx] = True
        m = cones.numel
        direct = bool(self._wl_rows.all()) and cones.w.flags.c_contiguous and cones.lam.flags.c_contiguous
        w, lam = (cones.w, cones.lam) if direct else (np.empty(m), np.empty(m))
        R, Ri, pl = np.empty(self._psd_rtotal), np.empty(self._psd_rtotal), np.empty(self._psd_ltotal)
        _lib.check(self.ldl._L.cb200_get_scaling(self.ldl._h, *[_p(a) for a in (w, lam, cones.soc_eta, cones.soc_d,
                                                                              cones.soc_u, cones.soc_v, R, Ri, pl)]),
                   "cb200_get_scaling")
        if not direct:
            np.copyto(cones.w, w, where=self._wl_rows); np.copyto(cones.lam, lam, where=self._wl_rows)
        ro = lo = 0
        for gi, j, n in self._psd_slots:
            g = cones.psd_groups[gi]
            g["R"][j] = R[ro:ro + n * n].reshape((n, n), order="F")
            g["Rinv"][j] = Ri[ro:ro + n * n].reshape((n, n), order="F")
            g["lam"][j] = pl[lo:lo + n]
            ro += n * n; lo += n

    def update_staged(self, dev_ptrs):
        """Resident mode: kktsolver_update! from a cone state the caller has staged in HBM.
        dev_ptrs: device addresses (int, 0 = keep) in STATE_KEYS order."""
        assert self.ldl.resident
        args = [C.c_void_p(p) if p else None for p in dev_ptrs]
        return _lib.check(self.ldl._L.cb200_update_cones(self.ldl._h, *args), "cb200_update_cones")

    def setrhs_staged(self, px, pz):
        """Resident mode: kktsolver_setrhs! from device addresses (stream-ordered device-to-device copy)."""
        assert self.ldl.resident
        _lib.check(self.ldl._L.cb200_setrhs(self.ldl._h, C.c_void_p(px) if px else None,
                                            C.c_void_p(pz) if pz else None), "cb200_setrhs")

    def setrhs(self, rhsx, rhsz):
        # kktsolver_setrhs!: the right-hand side goes straight to the device (no host staging copy)
        if self.ldl.resident:
            return
        rx, rz = _c64(rhsx), _c64(rhsz)
        _lib.check(self.ldl._L.cb200_setrhs(self.ldl._h, _p(rx), _p(rz)), "cb200_setrhs")

    def solve(self, lhsx, lhsz):
        if lhsx is not None:
            assert lhsx.dtype == np.float64 and lhsx.flags.c_contiguous
        if lhsz is not None:
            assert lhsz.dtype == np.float64 and lhsz.flags.c_contiguous
        rounds = C.c_int32(0)
        ok = _lib.check(self.ldl._L.cb200_solve_ir(self.ldl._h, None, None,
                                                   _p(lhsx), _p(lhsz), C.byref(rounds)),
                        "cb200_solve_ir")
        self.ir_rounds += rounds.value; self.n_solves += 1
        return ok

    def solve_multi(self, rhsx, rhsz, lhsx=None, lhsz=None):
        """setrhs + solve for k systems at once (cb200_solve_ir_multi): rhsx n x k, rhsz m x k, lhsx / lhsz the
        same shapes or None.  The arrays are column-major: Fortran order, or the transpose of a C-order
        k x n array.  Column j equals setrhs(rhsx[:, j], rhsz[:, j]) + solve bit for bit, with the same
        refinement rounds.  Returns (ok[k], ir_rounds[k]); a failed column's lhs is NaN.  Leaves what
        setrhs stored untouched."""
        rx = np.asfortranarray(rhsx, dtype=np.float64); rz = np.asfortranarray(rhsz, dtype=np.float64)
        k = rx.shape[1]
        assert rx.shape == (self.n, k) and rz.shape == (self.m, k)
        for a, n in ((lhsx, self.n), (lhsz, self.m)):
            if a is not None:
                assert a.dtype == np.float64 and a.flags.f_contiguous and a.shape == (n, k)
        rounds = np.zeros(k, dtype=np.int32); status = np.zeros(k, dtype=np.int32)
        _lib.check(self.ldl._L.cb200_solve_ir_multi(self.ldl._h, k, _p(rx), _p(rz), _p(lhsx), _p(lhsz),
                                                     _p(rounds), _p(status)), "cb200_solve_ir_multi")
        self.ir_rounds += int(rounds.sum()); self.n_solves += k
        return status == 0, rounds

    def solve_multi_staged(self, px, pz, k):
        """Resident mode: solve_multi from device addresses of the column-major n x k / m x k right-hand sides;
        the solutions stay on the device (download selector 8, N x k).  Returns (ok[k], ir_rounds[k])."""
        assert self.ldl.resident
        rounds = np.zeros(k, dtype=np.int32); status = np.zeros(k, dtype=np.int32)
        _lib.check(self.ldl._L.cb200_solve_ir_multi(self.ldl._h, int(k), C.c_void_p(px) if px else None,
                                                     C.c_void_p(pz) if pz else None, None, None,
                                                     _p(rounds), _p(status)), "cb200_solve_ir_multi")
        self.ir_rounds += int(rounds.sum()); self.n_solves += int(k)
        return status == 0, rounds

    def update_P(self, P):
        v = _c64(P.data)
        _lib.check(self.ldl._L.cb200_update_P(self.ldl._h, _p(v), len(v)), "cb200_update_P")

    def update_A(self, A):
        v = _c64(A.data)
        _lib.check(self.ldl._L.cb200_update_A(self.ldl._h, _p(v), len(v)), "cb200_update_A")

    def device_nzval(self):
        return self.ldl.download(0, self.KKT.nnz)


register_kktsolver("b200", B200KKTSolver)
