"""ctypes binding of libclarabel_b200.so (C-ABI: include/clarabel_b200.h).

Loading fails loudly if the library has not been built; compute entry points fail loudly
(negative status -> RuntimeError) if no CUDA device is present.  There is no CPU fallback.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CB200_LIB_PATH") or os.path.join(_HERE, "libclarabel_b200.so")    # (override: dev builds)
_LIB = None

# every symbol include/clarabel_b200.h declares
EXPORTED = [
    "cb200_default_settings", "cb200_symbolic_create", "cb200_symbolic_destroy",
    "cb200_symbolic_stat", "cb200_symbolic_flops", "cb200_symbolic_get", "cb200_symbolic_tile_lists",
    "cb200_order_amd", "cb200_order_nd",
    "cb200_create", "cb200_destroy", "cb200_update_values", "cb200_scale_values",
    "cb200_refactor", "cb200_solve", "cb200_solve_multi", "cb200_info",
    "cb200_set_maps", "cb200_update_cones", "cb200_update_scaling", "cb200_get_scaling", "cb200_setrhs", "cb200_solve_ir", "cb200_solve_ir_multi", "cb200_update_P", "cb200_update_A",
    "cb200_download", "cb200_get_timers", "cb200_reset_timers", "cb200_last_error",
    "cb200_get_stream", "cb200_set_resident",
    "cb200_symbolic_partition", "cb200_nccl_unique_id", "cb200_dist_init",
    "cb200_set_detail", "cb200_get_fine_timers", "cb200_fine_timer_name", "cb200_get_stats", "cb200_hint_blocks",
]


class CSettings(C.Structure):
    _fields_ = [("index_base", C.c_int32), ("device", C.c_int32),
                ("static_regularization_enable", C.c_int32),
                ("static_regularization_constant", C.c_double),
                ("static_regularization_proportional", C.c_double),
                ("dynamic_regularization_enable", C.c_int32),
                ("dynamic_regularization_eps", C.c_double),
                ("dynamic_regularization_delta", C.c_double),
                ("iterative_refinement_enable", C.c_int32),
                ("iterative_refinement_reltol", C.c_double),
                ("iterative_refinement_abstol", C.c_double),
                ("iterative_refinement_max_iter", C.c_int32),
                ("iterative_refinement_stop_ratio", C.c_double),
                ("ordering", C.c_int32), ("amd_dense_scale", C.c_double),
                ("nd_leaf_size", C.c_int32), ("use_cuda_graph", C.c_int32),
                ("reserved", C.c_int32 * 8)]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with __graft_entry__.build() "
                "(nvcc, sm_90a).  The CUDA backend has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        I64, I32, D, P = C.c_int64, C.c_int32, C.c_double, C.c_void_p
        L.cb200_default_settings.argtypes = [P]
        L.cb200_symbolic_create.argtypes = [I64, P, P, P, P, P]; L.cb200_symbolic_create.restype = I32
        L.cb200_symbolic_destroy.argtypes = [P]
        L.cb200_symbolic_stat.argtypes = [P, I32]; L.cb200_symbolic_stat.restype = I64
        L.cb200_symbolic_flops.argtypes = [P]; L.cb200_symbolic_flops.restype = D
        L.cb200_symbolic_get.argtypes = [P, I32, P, I64]; L.cb200_symbolic_get.restype = I32
        L.cb200_symbolic_tile_lists.argtypes = [P, P, I32, I32, I32, I32, P, P, P, P]
        L.cb200_symbolic_tile_lists.restype = I32
        L.cb200_order_amd.argtypes = [I64, P, P, D, P]; L.cb200_order_amd.restype = I32
        L.cb200_order_nd.argtypes = [I64, P, P, D, I64, P]; L.cb200_order_nd.restype = I32
        L.cb200_create.argtypes = [I64, P, P, P, P, P, P]; L.cb200_create.restype = I32
        L.cb200_destroy.argtypes = [P]
        L.cb200_update_values.argtypes = [P, P, P, I64]; L.cb200_update_values.restype = I32
        L.cb200_scale_values.argtypes = [P, P, I64, D]; L.cb200_scale_values.restype = I32
        L.cb200_refactor.argtypes = [P]; L.cb200_refactor.restype = I32
        L.cb200_solve.argtypes = [P, P, P]; L.cb200_solve.restype = I32
        L.cb200_solve_multi.argtypes = [P, I32, P, I64, P, I64]; L.cb200_solve_multi.restype = I32
        L.cb200_info.argtypes = [P, P, P, P]; L.cb200_info.restype = I32
        L.cb200_set_maps.argtypes = [P, I64, I64, I64, P, I64, P, I64, P, I64, P, I64, P, P, P, P, P]
        L.cb200_set_maps.restype = I32
        L.cb200_update_cones.argtypes = [P] * 7; L.cb200_update_cones.restype = I32
        L.cb200_update_scaling.argtypes = [P] * 4; L.cb200_update_scaling.restype = I32
        L.cb200_get_scaling.argtypes = [P] * 10; L.cb200_get_scaling.restype = I32
        L.cb200_solve_ir.argtypes = [P] * 6; L.cb200_solve_ir.restype = I32
        L.cb200_solve_ir_multi.argtypes = [P, I32] + [P] * 6; L.cb200_solve_ir_multi.restype = I32
        L.cb200_setrhs.argtypes = [P, P, P]; L.cb200_setrhs.restype = I32
        L.cb200_update_P.argtypes = [P, P, I64]; L.cb200_update_P.restype = I32
        L.cb200_update_A.argtypes = [P, P, I64]; L.cb200_update_A.restype = I32
        L.cb200_download.argtypes = [P, I32, P, I64]; L.cb200_download.restype = I32
        L.cb200_get_timers.argtypes = [P, P, I32]; L.cb200_get_timers.restype = I32
        L.cb200_reset_timers.argtypes = [P]; L.cb200_reset_timers.restype = I32
        L.cb200_last_error.restype = C.c_char_p
        L.cb200_get_stream.argtypes = [P]; L.cb200_get_stream.restype = C.c_void_p
        L.cb200_set_resident.argtypes = [P, I32]; L.cb200_set_resident.restype = I32
        L.cb200_symbolic_partition.argtypes = [P, I32, P, P, P]; L.cb200_symbolic_partition.restype = I32
        L.cb200_nccl_unique_id.argtypes = [P]; L.cb200_nccl_unique_id.restype = I32
        L.cb200_dist_init.argtypes = [P, I32, I32, P]; L.cb200_dist_init.restype = I32
        L.cb200_set_detail.argtypes = [P, I32]; L.cb200_set_detail.restype = I32
        L.cb200_get_fine_timers.argtypes = [P, P, I32]; L.cb200_get_fine_timers.restype = I32
        L.cb200_fine_timer_name.argtypes = [I32]; L.cb200_fine_timer_name.restype = C.c_char_p
        L.cb200_get_stats.argtypes = [P, P, I32]; L.cb200_get_stats.restype = I32
        L.cb200_hint_blocks.argtypes = [P, I64]; L.cb200_hint_blocks.restype = I32
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def last_error():
    return lib().cb200_last_error().decode()


def check(rc, what):
    """<0: usage / CUDA error -> raise (Julia shim: error()); >0: numerical failure -> False."""
    if rc < 0:
        raise RuntimeError(f"{what} failed ({rc}): {last_error()}")
    return rc == 0


def make_settings(settings=None, **over):
    cs = CSettings()
    lib().cb200_default_settings(C.byref(cs))
    if settings is not None:
        for f in ("static_regularization_enable", "static_regularization_constant",
                  "static_regularization_proportional", "dynamic_regularization_enable",
                  "dynamic_regularization_eps", "dynamic_regularization_delta",
                  "iterative_refinement_enable", "iterative_refinement_reltol",
                  "iterative_refinement_abstol", "iterative_refinement_max_iter",
                  "iterative_refinement_stop_ratio"):
            setattr(cs, f, type(getattr(cs, f))(getattr(settings, f)))
    if os.environ.get("CB200_GRAPH") is not None:     # bit mask: 1 solve sweeps, 2 factorisation
        cs.use_cuda_graph = int(os.environ["CB200_GRAPH"])
    for k, v in over.items():
        setattr(cs, k, v)
    return cs


def hint_blocks(block_id):
    """cb200_hint_blocks: dense cone blocks nested dissection must keep whole (None clears)."""
    if block_id is None:
        lib().cb200_hint_blocks(None, 0)
    else:
        b = np.ascontiguousarray(block_id, dtype=np.int64)
        lib().cb200_hint_blocks(_p(b), len(b))


def cone_block_ids(cones, n, N):
    """block id per KKT row/column for the dense (non-diagonal) cone blocks, -1 elsewhere."""
    bid = np.full(N, -1, dtype=np.int64)
    k = 0
    for i in range(len(cones.specs)):
        if not cones.Hs_is_diagonal[i] and cones.numels[i] > 1:
            bid[n + cones.rng_cones[i]:n + cones.rng_cones[i + 1]] = k
            k += 1
    return bid if k else None


_SYM_ARRAYS = ["perm", "sn_first", "rows_ptr", "rows", "rel", "sn_parent", "panel_off", "upd_off",
               "a_map", "sn_level", "child_ptr", "child_list", "panel_ld"]


class Symbolic:
    """Host-only symbolic analysis (no CUDA call)."""

    def __init__(self, K, ordering=1, nd_leaf=96, dense_scale=0.3, perm=None, block_id=None):
        L = lib()
        hint_blocks(block_id)
        cs = make_settings(ordering=ordering, nd_leaf_size=nd_leaf, amd_dense_scale=dense_scale)
        cp = np.ascontiguousarray(K.indptr, dtype=np.int64)
        ri = np.ascontiguousarray(K.indices, dtype=np.int64)
        pp = None if perm is None else np.ascontiguousarray(perm, dtype=np.int64)
        self._h = C.c_void_p()
        check(L.cb200_symbolic_create(K.shape[0], _p(cp), _p(ri), C.byref(cs), _p(pp),
                                      C.byref(self._h)), "cb200_symbolic_create")
        names = ["N", "nsuper", "nnzL", "nlevels", "max_front", "max_width", "upd_total",
                 "panel_total", "rows_total", "nnzK"]
        self.stats = {nm: int(L.cb200_symbolic_stat(self._h, i)) for i, nm in enumerate(names)}
        self.stats["flops"] = float(L.cb200_symbolic_flops(self._h))

    def arrays(self):
        L = lib(); s = self.stats
        nroots_len = None
        lens = dict(perm=s["N"], sn_first=s["nsuper"] + 1, rows_ptr=s["nsuper"] + 1,
                    rows=s["rows_total"], rel=s["rows_total"], sn_parent=s["nsuper"],
                    panel_off=s["nsuper"] + 1, upd_off=s["nsuper"] + 1, a_map=s["nnzK"],
                    sn_level=s["nsuper"], child_ptr=s["nsuper"] + 1)
        out = {}
        lens["panel_ld"] = s["nsuper"]
        for i, nm in enumerate(_SYM_ARRAYS):
            a = np.empty(lens[nm] if nm != "child_list" else out["child_ptr"][-1], dtype=np.int64)
            check(L.cb200_symbolic_get(self._h, i, _p(a), len(a)), "cb200_symbolic_get")
            out[nm] = a
        ch = [[] for _ in range(s["nsuper"])]
        for sn, par in enumerate(out["sn_parent"]):
            if par >= 0:
                ch[par].append(sn)
        out["children"] = ch
        return out

    def kid_lists(self):
        """Per-front child lists of the shared-memory front kernel (cb200_symbolic_get selector 13):
        [len(child_list), 3] of (update-block offset, rel offset, nr), row q for child_list[q]."""
        L = lib()
        cp = np.empty(self.stats["nsuper"] + 1, dtype=np.int64)
        check(L.cb200_symbolic_get(self._h, 10, _p(cp), len(cp)), "cb200_symbolic_get")
        out = np.empty(3 * int(cp[-1]), dtype=np.int64)
        check(L.cb200_symbolic_get(self._h, 13, _p(out), len(out)), "cb200_symbolic_get")
        return out.reshape(-1, 3)

    def asm_maps(self):
        """The destination-owner assembly maps (symbolic.h; selectors 14-18): front_ptr, asm_base,
        asm_colptr, asm_src, asm_child"""
        L = lib(); n = self.stats["nsuper"] + 1
        out = {}
        for sel, nm in ((14, "front_ptr"), (15, "asm_base")):
            out[nm] = np.empty(n, dtype=np.int64)
            check(L.cb200_symbolic_get(self._h, sel, _p(out[nm]), n), "cb200_symbolic_get")
        for sel, nm, ln in ((16, "asm_colptr", out["front_ptr"][-1]), (17, "asm_src", out["asm_base"][-1]),
                            (18, "asm_child", out["asm_base"][-1])):
            out[nm] = np.empty(int(ln), dtype=np.int64)
            check(L.cb200_symbolic_get(self._h, sel, _p(out[nm]), len(out[nm])), "cb200_symbolic_get")
        return out

    def partition(self, nranks):
        n = self.stats["nsuper"]
        owner = np.empty(n, dtype=np.int64); top = np.empty(n, dtype=np.int64)
        load = np.zeros(max(1, nranks))
        check(lib().cb200_symbolic_partition(self._h, int(nranks), _p(owner), _p(top), _p(load)),
              "cb200_symbolic_partition")
        return owner, top.astype(bool), load

    def tile_lists(self, fronts, T, schur, gather=True, active=None):
        """Per-tile source lists of the large-front extend-add for one batch of fronts:
        tiles [n, 4] (slot, ti, tj, first rectangle; a final sentinel row holds the end) and
        rects [m, 5] (child, ja, jb, ia, ib).  active: optional per-supernode mask (multi-GPU) of
        the children whose contributions are assembled."""
        L = lib()
        fr = np.ascontiguousarray(fronts, dtype=np.int64)
        act = None if active is None else np.ascontiguousarray(active, dtype=np.int64)
        cnt = np.zeros(2, dtype=np.int64)
        args = (self._h, _p(fr), len(fr), int(T), int(bool(schur)), int(bool(gather)), _p(act), _p(cnt))
        check(L.cb200_symbolic_tile_lists(*args, None, None), "cb200_symbolic_tile_lists")
        tiles = np.zeros((cnt[0] + 1, 4), dtype=np.int64)
        rects = np.zeros((cnt[1], 5), dtype=np.int64)
        check(L.cb200_symbolic_tile_lists(*args, _p(tiles), _p(rects)), "cb200_symbolic_tile_lists")
        tiles[-1, 3] = cnt[1]
        return tiles, rects

    def __del__(self):
        try:
            if self._h:
                lib().cb200_symbolic_destroy(self._h); self._h = None
        except Exception:
            pass
