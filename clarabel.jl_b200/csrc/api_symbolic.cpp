// C-ABI: host-only symbolic analysis entry points (include/clarabel_b200.h).
#include "../../include/clarabel_b200.h"
#include "symbolic.h"
#include "api_common.h"

#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>

struct cb200_symbolic { cb200::Symbolic S; };

namespace cb200 {
thread_local std::string g_last_error;
void set_error(const std::string& s) { g_last_error = s; }
thread_local std::vector<int32_t> g_block_hint;     // consumed by the next symbolic analysis
SymbolicOptions options_from_settings(const cb200_settings* st) {
    SymbolicOptions o;
    o.block_id = g_block_hint.empty() ? nullptr : g_block_hint.data();
    if (const char* e = getenv("CB200_RELAX")) {       // tuning aid: "small,z1,z2,z3,maxwidth"
        double a, b, c, d, w;
        if (sscanf(e, "%lf,%lf,%lf,%lf,%lf", &a, &b, &c, &d, &w) == 5) {
            o.relax_small = (int32_t)a; o.relax_z1 = b; o.relax_z2 = c; o.relax_z3 = d; o.max_width = (int32_t)w;
        }
    }
    auto env_int = [](const char* name, int dflt, int lo, int hi) {
        const char* e = getenv(name);
        return e ? std::max(lo, std::min(hi, atoi(e))) : dflt;
    };
    o.collapse_nf = env_int("CB200_COLLAPSE_NF", 32, 0, 64);
    o.use_panel_kernel = !(getenv("CB200_NO_PANEL") && getenv("CB200_NO_PANEL")[0] == '1');
    o.panel_min_nf = env_int("CB200_PANEL_MIN_NF", 64, 16, 152);
    o.panel_max_nf = env_int("CB200_PANEL_MAX_NF", 152, 16, 152);
    o.small_max_nf = env_int("CB200_SMALL_MAX_NF", 152, 16, 152);
    if (st) {
        o.ordering = st->ordering;
        if (st->amd_dense_scale > 0) o.dense_scale = st->amd_dense_scale;
        if (st->nd_leaf_size > 0) o.nd_leaf = st->nd_leaf_size;
    }
    return o;
}
}  // namespace cb200

template <class V> static int32_t copy_out(const V& v, int64_t* out, int64_t len) {
    if ((int64_t)v.size() != len) { cb200::set_error("cb200_symbolic_get: length mismatch"); return -2; }
    for (int64_t i = 0; i < len; ++i) out[i] = (int64_t)v[i];
    return 0;
}

extern "C" {

const char* cb200_last_error(void) { return cb200::g_last_error.c_str(); }

void cb200_default_settings(cb200_settings* s) {
    std::memset(s, 0, sizeof(*s));
    s->index_base = 0; s->device = 0;
    s->static_regularization_enable = 1;
    s->static_regularization_constant = 1e-8;
    s->static_regularization_proportional = 2.220446049250313e-16 * 2.220446049250313e-16;
    s->dynamic_regularization_enable = 1;
    s->dynamic_regularization_eps = 1e-13;
    s->dynamic_regularization_delta = 2e-7;
    s->iterative_refinement_enable = 1;
    s->iterative_refinement_reltol = 1e-13;
    s->iterative_refinement_abstol = 1e-12;
    s->iterative_refinement_max_iter = 10;
    s->iterative_refinement_stop_ratio = 5.0;
    s->ordering = 1; s->amd_dense_scale = 0.3; s->nd_leaf_size = 96;
    s->use_cuda_graph = 1;
}

int32_t cb200_hint_blocks(const int64_t* block_id, int64_t N) {
    cb200::g_block_hint.clear();
    if (block_id) { cb200::g_block_hint.resize(N); for (int64_t i = 0; i < N; ++i) cb200::g_block_hint[i] = (int32_t)block_id[i]; }
    return 0;
}

int32_t cb200_symbolic_create(int64_t N, const int64_t* colptr, const int64_t* rowval,
                              const cb200_settings* st, const int64_t* user_perm,
                              cb200_symbolic** out) {
    try {
        std::vector<int64_t> cp, ri;
        const int64_t base = st ? st->index_base : 0;
        if (base) {
            cp.resize(N + 1); for (int64_t i = 0; i <= N; ++i) cp[i] = colptr[i] - base;
            ri.resize(cp[N]); for (int64_t i = 0; i < cp[N]; ++i) ri[i] = rowval[i] - base;
            colptr = cp.data(); rowval = ri.data();
        }
        std::vector<int64_t> up;
        if (user_perm && base) { up.resize(N); for (int64_t i = 0; i < N; ++i) up[i] = user_perm[i] - base; user_perm = up.data(); }
        auto* s = new cb200_symbolic();
        if (!cb200::g_block_hint.empty() && (int64_t)cb200::g_block_hint.size() != N) cb200::g_block_hint.clear();
        cb200::symbolic_analyze(N, colptr, rowval, cb200::options_from_settings(st), user_perm, s->S);
        cb200::g_block_hint.clear();
        *out = s;
        return 0;
    } catch (const std::exception& e) { cb200::set_error(e.what()); return -1; }
}

void cb200_symbolic_destroy(cb200_symbolic* s) { delete s; }

int64_t cb200_symbolic_stat(const cb200_symbolic* s, int32_t what) {
    const auto& S = s->S;
    switch (what) {
        case 0: return S.N; case 1: return S.nsuper; case 2: return S.nnzL; case 3: return S.nlevels;
        case 4: return S.max_front; case 5: return S.max_width; case 6: return S.upd_total;
        case 7: return S.panel_off.empty() ? 0 : S.panel_off.back();
        case 8: return (int64_t)S.rows.size(); case 9: return S.nnzK;
        case 10: return S.ordering_used;
    }
    return -1;
}
double cb200_symbolic_flops(const cb200_symbolic* s) { return s->S.flops; }

int32_t cb200_symbolic_partition(const cb200_symbolic* s, int32_t nranks, int64_t* owner,
                                 int64_t* is_top, double* rank_load) {
    std::vector<int32_t> ow; std::vector<int8_t> tp; std::vector<double> ld;
    cb200::partition_subtrees(s->S, nranks, ow, tp, &ld);
    for (size_t i = 0; i < ow.size(); ++i) { owner[i] = ow[i]; is_top[i] = tp[i]; }
    if (rank_load) for (size_t i = 0; i < ld.size(); ++i) rank_load[i] = ld[i];
    return 0;
}

int32_t cb200_symbolic_get(const cb200_symbolic* s, int32_t which, int64_t* out, int64_t len) {
    const auto& S = s->S;
    switch (which) {
        case 0: return copy_out(S.perm, out, len);      case 1: return copy_out(S.sn_first, out, len);
        case 2: return copy_out(S.rows_ptr, out, len);  case 3: return copy_out(S.rows, out, len);
        case 4: return copy_out(S.rel, out, len);       case 5: return copy_out(S.sn_parent, out, len);
        case 6: return copy_out(S.panel_off, out, len); case 7: return copy_out(S.upd_off, out, len);
        case 8: return copy_out(S.a_map, out, len);     case 9: return copy_out(S.sn_level, out, len);
        case 10: return copy_out(S.child_ptr, out, len); case 11: return copy_out(S.child_list, out, len);
        case 12: return copy_out(S.panel_ld, out, len);
        case 14: return copy_out(S.front_ptr, out, len); case 15: return copy_out(S.asm_base, out, len);
        case 16: return copy_out(S.asm_colptr, out, len); case 17: return copy_out(S.asm_src, out, len);
        case 18: return copy_out(S.asm_child, out, len);
        case 13:
            if ((int64_t)S.kids.size() * 3 != len) { cb200::set_error("cb200_symbolic_get: length mismatch"); return -2; }
            for (size_t q = 0; q < S.kids.size(); ++q) {
                out[3 * q] = S.kids[q].uoff; out[3 * q + 1] = S.kids[q].roff; out[3 * q + 2] = S.kids[q].nrc;
            }
            return 0;
    }
    cb200::set_error("cb200_symbolic_get: bad selector"); return -2;
}

int32_t cb200_symbolic_tile_lists(const cb200_symbolic* s, const int64_t* fronts, int32_t nfronts, int32_t T,
                                  int32_t schur, int32_t gather, const int64_t* active, int64_t* counts,
                                  int64_t* tiles, int64_t* rects) {
    const auto& S = s->S;
    if (T != 64 && T != 128) { cb200::set_error("cb200_symbolic_tile_lists: T must be 64 or 128"); return -2; }
    std::vector<int32_t> fr(nfronts);
    for (int32_t k = 0; k < nfronts; ++k) {
        if (fronts[k] < 0 || fronts[k] >= S.nsuper) { cb200::set_error("cb200_symbolic_tile_lists: bad front"); return -2; }
        fr[k] = (int32_t)fronts[k];
    }
    std::vector<int8_t> act;
    if (active) { act.resize(S.nsuper); for (int32_t q = 0; q < S.nsuper; ++q) act[q] = active[q] != 0; }
    std::vector<cb200::TileEntry> te; std::vector<cb200::TileRect> tr;
    cb200::build_tile_lists(S, fr.data(), nfronts, T, schur != 0, gather != 0, active ? act.data() : nullptr, te, tr);
    counts[0] = (int64_t)te.size(); counts[1] = (int64_t)tr.size();
    if (tiles)
        for (size_t i = 0; i < te.size(); ++i) {
            tiles[4 * i] = te[i].slot; tiles[4 * i + 1] = te[i].ti; tiles[4 * i + 2] = te[i].tj; tiles[4 * i + 3] = te[i].rect;
        }
    if (rects)
        for (size_t i = 0; i < tr.size(); ++i) {
            const cb200::TileRect& r = tr[i];
            rects[5 * i] = r.child; rects[5 * i + 1] = r.ja; rects[5 * i + 2] = r.jb; rects[5 * i + 3] = r.ia; rects[5 * i + 4] = r.ib;
        }
    return 0;
}

}  // extern "C"
