// Fill-reducing orderings for the symmetric KKT pattern (host, setup-time).
//
// The reference obtains its ordering from AMD.jl -> SuiteSparse AMD inside QDLDL.jl
// (reference call site: src/kktsolvers/direct-ldl/directldl_qdldl.jl:18-25, with
// amd_dense_scale = 1.5).  Neither library is part of the Clarabel.jl repository, so this
// file restates the published algorithm (Amestoy, Davis, Duff, "An approximate minimum degree
// ordering algorithm", SIMAX 1996): quotient graph, element absorption, approximate external
// degree, mass elimination, supervariable detection by hashing, aggressive absorption and
// dense-row deferral.  It is written from the paper's description with std::vector storage
// (no in-place workspace / garbage collection), not from SuiteSparse source.
//
// cb200_order_amd      : AMD-class ordering (used for the CPU baseline and GPU leaf blocks)
// cb200_order_nd       : nested dissection by BFS level-structure separators over AMD leaves,
//                        gives the wide, shallow elimination trees the GPU factorization and
//                        the multi-GPU subtree split need (SURVEY.md section 8e).
#include <cstdint>
#include <cstring>
#include <cmath>
#include <vector>
#include <algorithm>
#include <numeric>
#include <atomic>
#include <thread>
#include <deque>
#include <exception>
#include <cstdlib>

#include "ordering.h"

namespace cb200 {

// Build full symmetric adjacency (no diagonal, no duplicates) from an upper- or
// lower-triangular (or full) CSC pattern.
void build_sym_graph(int64_t n, const int64_t* Ap, const int64_t* Ai,
                     std::vector<int64_t>& xadj, std::vector<int32_t>& adj) {
    std::vector<int64_t> cnt(n + 1, 0);
    for (int64_t j = 0; j < n; ++j)
        for (int64_t p = Ap[j]; p < Ap[j + 1]; ++p) {
            int64_t i = Ai[p];
            if (i == j) continue;
            cnt[i + 1]++; cnt[j + 1]++;
        }
    xadj.assign(n + 1, 0);
    for (int64_t i = 0; i < n; ++i) xadj[i + 1] = xadj[i] + cnt[i + 1];
    adj.resize(xadj[n]);
    std::vector<int64_t> pos(xadj.begin(), xadj.end() - 1);
    for (int64_t j = 0; j < n; ++j)
        for (int64_t p = Ap[j]; p < Ap[j + 1]; ++p) {
            int64_t i = Ai[p];
            if (i == j) continue;
            adj[pos[i]++] = (int32_t)j; adj[pos[j]++] = (int32_t)i;
        }
    // sort + unique each list (input may hold both triangles)
    std::vector<int64_t> nx(n + 1, 0);
    int64_t w = 0;
    for (int64_t i = 0; i < n; ++i) {
        int64_t a = xadj[i], b = xadj[i + 1];
        std::sort(adj.begin() + a, adj.begin() + b);
        int64_t s = w;
        for (int64_t p = a; p < b; ++p)
            if (p == a || adj[p] != adj[p - 1]) adj[w++] = adj[p];
        nx[i] = s;
    }
    nx[n] = w;
    xadj = nx; adj.resize(w);
}

namespace {

struct AMD {
    int32_t n;
    std::vector<std::vector<int32_t>> adjV, adjE, evars;
    std::vector<int32_t> nv, degree, mark, head, next, last, elen_deg, merged_next, merged_tail;
    std::vector<int64_t> w;
    std::vector<uint8_t> state;   // 0 = live variable, 1 = live element, 2 = dead
    int64_t wflg = 2;
    int32_t tag = 0, mindeg = 0;

    void list_remove(int32_t i) {
        int32_t d = degree[i];
        int32_t nx = next[i], lt = last[i];
        if (nx != -1) last[nx] = lt;
        if (lt != -1) next[lt] = nx; else head[d] = nx;
    }
    void list_insert(int32_t i) {
        int32_t d = degree[i];
        int32_t h = head[d];
        next[i] = h; last[i] = -1;
        if (h != -1) last[h] = i;
        head[d] = i;
        if (d < mindeg) mindeg = d;
    }
};

}  // namespace

// graph: full symmetric adjacency xadj/adj over n nodes.  perm_out[k] = k-th pivot.
void amd_order_graph(int32_t n, const int64_t* xadj, const int32_t* adj, double dense_scale,
                     int32_t* perm_out) {
    if (n == 0) return;
    AMD S; S.n = n;
    S.adjV.resize(n); S.adjE.resize(n); S.evars.resize(n);
    S.nv.assign(n, 1); S.degree.assign(n, 0); S.w.assign(n, 1); S.mark.assign(n, 0);
    S.head.assign(n + 1, -1); S.next.assign(n, -1); S.last.assign(n, -1);
    S.elen_deg.assign(n, 0); S.merged_next.assign(n, -1); S.merged_tail.resize(n);
    S.state.assign(n, 0);
    for (int32_t i = 0; i < n; ++i) S.merged_tail[i] = i;

    // dense rows are deferred to the end (AMD's "dense" control; default 10*sqrt(n),
    // scaled by amd_dense_scale like QDLDL.jl does)
    double dthr = dense_scale * 10.0 * std::sqrt((double)n);
    int32_t dense = (int32_t)std::max(16.0, std::min(dthr, (double)n));
    std::vector<int32_t> dense_nodes;
    std::vector<uint8_t> is_dense(n, 0);
    for (int32_t i = 0; i < n; ++i) {
        int64_t d = xadj[i + 1] - xadj[i];
        if (d > dense) { is_dense[i] = 1; dense_nodes.push_back(i); }
    }
    int32_t nlive = 0;
    for (int32_t i = 0; i < n; ++i) {
        if (is_dense[i]) { S.state[i] = 2; S.nv[i] = 0; continue; }
        auto& v = S.adjV[i];
        v.reserve(xadj[i + 1] - xadj[i]);
        for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p)
            if (!is_dense[adj[p]]) v.push_back(adj[p]);
        S.degree[i] = (int32_t)v.size();
        nlive++;
    }
    S.mindeg = n;
    for (int32_t i = 0; i < n; ++i) if (S.state[i] == 0) S.list_insert(i);

    std::vector<int32_t> order; order.reserve(n);
    std::vector<int32_t> Lp, hashv(n, 0), bucket_head, cand;
    std::vector<int64_t> hkey(n, 0);
    int32_t eliminated = 0;
    auto emit = [&](int32_t p) {           // p and everything merged into it
        for (int32_t q = p; q != -1; q = S.merged_next[q]) order.push_back(q);
    };

    while (eliminated < nlive) {
        // ---- pick pivot of minimum approximate degree
        while (S.mindeg < n && S.head[S.mindeg] == -1) S.mindeg++;
        int32_t p = S.head[S.mindeg];
        S.list_remove(p);
        eliminated += S.nv[p];
        // ---- build Lp (pattern of the new element)
        S.tag++;
        int32_t tag = S.tag;
        Lp.clear();
        S.mark[p] = tag;
        int32_t degme = 0;
        for (int32_t j : S.adjV[p])
            if (S.state[j] == 0 && S.nv[j] > 0 && S.mark[j] != tag) {
                S.mark[j] = tag; Lp.push_back(j); degme += S.nv[j];
            }
        for (int32_t e : S.adjE[p]) {
            if (S.state[e] != 1) continue;
            for (int32_t j : S.evars[e])
                if (S.state[j] == 0 && S.nv[j] > 0 && S.mark[j] != tag) {
                    S.mark[j] = tag; Lp.push_back(j); degme += S.nv[j];
                }
            S.state[e] = 2;                       // absorbed into p
            std::vector<int32_t>().swap(S.evars[e]);
        }
        std::vector<int32_t>().swap(S.adjV[p]);
        std::vector<int32_t>().swap(S.adjE[p]);
        S.state[p] = 1;                           // p becomes an element
        for (int32_t i : Lp) S.list_remove(i);

        // ---- first pass: w[e] - wflg = |Le \ Lp| for every element adjacent to Lp
        const int64_t wflg = S.wflg;
        for (int32_t i : Lp) {
            auto& E = S.adjE[i];
            size_t k = 0;
            for (int32_t e : E) {
                if (S.state[e] != 1) continue;     // drop absorbed elements
                E[k++] = e;
                if (S.w[e] < wflg) S.w[e] = S.elen_deg[e] + wflg;
                S.w[e] -= S.nv[i];
            }
            E.resize(k);
        }
        // ---- second pass: degrees, pruning, aggressive absorption, hashing
        int32_t nleft = nlive - eliminated;
        size_t keep = 0;
        for (size_t t = 0; t < Lp.size(); ++t) {
            int32_t i = Lp[t];
            auto& E = S.adjE[i];
            int64_t deg = 0; int64_t h = 0;
            size_t k = 0;
            for (int32_t e : E) {
                int64_t dext = S.w[e] - wflg;
                if (dext > 0) { deg += dext; E[k++] = e; h += e; }
                else { /* aggressive absorption: Le subset of Lp */
                    S.state[e] = 2; std::vector<int32_t>().swap(S.evars[e]);
                }
            }
            E.resize(k);
            auto& V = S.adjV[i];
            k = 0;
            for (int32_t j : V) {
                if (S.state[j] != 0 || S.nv[j] <= 0) continue;   // dead / absorbed variable
                if (S.mark[j] == tag) continue;                  // edge now covered by element p
                V[k++] = j; deg += S.nv[j]; h += j;
            }
            V.resize(k);
            if (deg == 0 && E.empty()) {
                // mass elimination: i is indistinguishable from p once p is eliminated
                eliminated += S.nv[i];
                degme -= S.nv[i];
                S.merged_next[S.merged_tail[p]] = i;
                S.merged_tail[p] = S.merged_tail[i];
                S.nv[i] = 0; S.state[i] = 2;
                std::vector<int32_t>().swap(V); std::vector<int32_t>().swap(E);
                continue;
            }
            E.push_back(p); h += p;
            int64_t d1 = (int64_t)S.degree[i] + degme - S.nv[i];     // old bound + new element
            int64_t d2 = deg + degme - S.nv[i];
            int64_t d = std::min(d1, d2);
            d = std::min<int64_t>(d, nleft - S.nv[i]);
            if (d < 0) d = 0;
            S.degree[i] = (int32_t)d;       // provisional (external degree incl. Lp \ i)
            hkey[i] = h;
            Lp[keep++] = i;
        }
        Lp.resize(keep);
        // ---- supervariable detection among Lp (hash on adjacency)
        if (Lp.size() > 1) {
            cand.assign(Lp.begin(), Lp.end());
            std::sort(cand.begin(), cand.end(), [&](int32_t a, int32_t b) {
                return hkey[a] < hkey[b] || (hkey[a] == hkey[b] && a < b); });
            size_t a = 0;
            while (a < cand.size()) {
                size_t b = a + 1;
                while (b < cand.size() && hkey[cand[b]] == hkey[cand[a]]) b++;
                for (size_t x = a; x < b; ++x) {
                    int32_t i = cand[x];
                    if (S.nv[i] <= 0) continue;
                    // mark i's adjacency
                    S.tag++;
                    int32_t t2 = S.tag;
                    for (int32_t e : S.adjE[i]) S.mark[e] = t2;
                    for (int32_t j : S.adjV[i]) S.mark[j] = t2;
                    for (size_t y = x + 1; y < b; ++y) {
                        int32_t j = cand[y];
                        if (S.nv[j] <= 0) continue;
                        if (S.adjE[j].size() != S.adjE[i].size() ||
                            S.adjV[j].size() != S.adjV[i].size()) continue;
                        bool same = true;
                        for (int32_t e : S.adjE[j]) if (S.mark[e] != t2) { same = false; break; }
                        if (same) for (int32_t v : S.adjV[j]) if (S.mark[v] != t2) { same = false; break; }
                        if (!same) continue;
                        // merge j into i
                        S.nv[i] += S.nv[j];
                        S.degree[i] = std::max(0, S.degree[i] - S.nv[j]);
                        S.nv[j] = 0; S.state[j] = 2;
                        S.merged_next[S.merged_tail[i]] = j;
                        S.merged_tail[i] = S.merged_tail[j];
                        std::vector<int32_t>().swap(S.adjV[j]);
                        std::vector<int32_t>().swap(S.adjE[j]);
                    }
                }
                a = b;
            }
        }
        // ---- finalise element p and re-insert the survivors
        auto& ev = S.evars[p];
        ev.clear();
        int32_t dm = 0;
        for (int32_t i : Lp) if (S.nv[i] > 0) { ev.push_back(i); dm += S.nv[i]; }
        S.elen_deg[p] = dm;
        for (int32_t i : ev) {
            int32_t d = std::min(S.degree[i], std::max(0, nleft - S.nv[i]));
            S.degree[i] = d;
            S.list_insert(i);
        }
        if (ev.empty()) S.state[p] = 2;
        S.wflg = wflg + (int64_t)n + 1;      // exceeds every w[e] set in this step
        emit(p);
    }
    // dense nodes last, by increasing degree
    std::sort(dense_nodes.begin(), dense_nodes.end(), [&](int32_t a, int32_t b) {
        int64_t da = xadj[a + 1] - xadj[a], db = xadj[b + 1] - xadj[b];
        return da < db || (da == db && a < b); });
    for (int32_t i : dense_nodes) order.push_back(i);
    for (int32_t k = 0; k < n; ++k) perm_out[k] = order[k];
}


// ------------------------------------------------------------------------------------------
// Nested dissection with BFS level-structure separators (George's automatic ND) over AMD
// leaves.  Rationale: the GPU factorization schedules fronts level by level, so the depth of
// the assembly tree is a latency term; minimum-degree orderings on banded / chain-like KKT
// graphs give trees of depth O(N).  ND bounds the depth by O(log N) + leaf depth and exposes
// the independent subtrees that the multi-GPU split uses.  Falls back to AMD on pieces where
// no small separator exists (expander-like graphs such as factor models).
namespace {

struct NDCtx {
    int32_t n;                                  // vertices of the (possibly compressed) graph
    const int64_t* xadj; const int32_t* adj;
    // clique blocks: vertex v of this graph stands for the original vertices mem[mem_ptr[v]..) and
    // weighs wt[v]; without blocks the graph is the original one (compressed == false)
    bool compressed = false;
    std::vector<int32_t> wt, mem_ptr, mem, comp_of;
    const int64_t* oxadj = nullptr; const int32_t* oadj = nullptr; int32_t on = 0;
    std::vector<int32_t> olocal;
    std::vector<int32_t> label;      // current piece id of each vertex (-1 = already ordered)
    std::vector<int64_t> level;
    std::vector<int32_t> local;
    std::atomic<int32_t> next_label{1};
    int32_t leaf_size;
    double dense_scale;
    // Sub-pieces are vertex-disjoint, so independent pieces are ordered on separate host threads;
    // every per-vertex array is only written at the piece's own vertices.  label[] is also READ at
    // neighbours that may belong to a piece another thread is relabelling: labels are never reused,
    // so either value compares unequal to this piece's label (relaxed atomics keep that well defined).
    std::atomic<int32_t> live_threads{1};
    int32_t max_threads = 1;
    static constexpr size_t PAR_MIN_VERTS = 20000;
    int32_t lab_get(int32_t v) const { return __atomic_load_n(&label[v], __ATOMIC_RELAXED); }
    void lab_set(int32_t v, int32_t l) { __atomic_store_n(&label[v], l, __ATOMIC_RELAXED); }

    // BFS inside piece `lab` from `root`; fills queue (visit order) and level[]; returns #levels
    int32_t bfs(int32_t root, int32_t lab, std::vector<int32_t>& q, int64_t stamp_base) {
        q.clear(); q.push_back(root); level[root] = stamp_base;
        size_t h = 0; int64_t maxl = stamp_base;
        while (h < q.size()) {
            int32_t v = q[h++];
            for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                int32_t u = adj[p];
                if (lab_get(u) != lab || level[u] >= stamp_base) continue;
                level[u] = level[v] + 1; maxl = std::max(maxl, level[u]); q.push_back(u);
            }
        }
        return (int32_t)(maxl - stamp_base + 1);
    }

    int64_t weight_of(const std::vector<int32_t>& verts) const {
        if (!compressed) return (int64_t)verts.size();
        int64_t w = 0; for (int32_t v : verts) w += wt[v];
        return w;
    }

    void amd_leaf(const std::vector<int32_t>& verts, std::vector<int32_t>& order) {
        int32_t lab = lab_get(verts[0]);
        if (compressed) {
            // expand to original vertices and order the induced original subgraph
            std::vector<int32_t> ov;
            for (int32_t v : verts) for (int32_t q = mem_ptr[v]; q < mem_ptr[v + 1]; ++q) ov.push_back(mem[q]);
            const int32_t k = (int32_t)ov.size();
            if (k <= 2) { for (int32_t v : ov) order.push_back(v); for (int32_t v : verts) lab_set(v, -1); return; }
            for (int32_t i = 0; i < k; ++i) olocal[ov[i]] = i;
            std::vector<int64_t> lx(k + 1, 0); std::vector<int32_t> la;
            for (int32_t i = 0; i < k; ++i) {
                const int32_t v = ov[i];
                for (int64_t p = oxadj[v]; p < oxadj[v + 1]; ++p)
                    if (lab_get(comp_of[oadj[p]]) == lab) la.push_back(olocal[oadj[p]]);
                lx[i + 1] = (int64_t)la.size();
            }
            std::vector<int32_t> lp(k);
            cb200::amd_order_graph(k, lx.data(), la.data(), dense_scale, lp.data());
            for (int32_t i = 0; i < k; ++i) order.push_back(ov[lp[i]]);
            for (int32_t v : verts) lab_set(v, -1);
            return;
        }
        int32_t k = (int32_t)verts.size();
        if (k <= 2) { for (int32_t v : verts) { order.push_back(v); lab_set(v, -1); } return; }
        for (int32_t i = 0; i < k; ++i) local[verts[i]] = i;
        std::vector<int64_t> lx(k + 1, 0); std::vector<int32_t> la;
        for (int32_t i = 0; i < k; ++i) {
            int32_t v = verts[i];
            for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p)
                if (lab_get(adj[p]) == lab) la.push_back(local[adj[p]]);
            lx[i + 1] = (int64_t)la.size();
        }
        std::vector<int32_t> lp(k);
        cb200::amd_order_graph(k, lx.data(), la.data(), dense_scale, lp.data());
        for (int32_t i = 0; i < k; ++i) order.push_back(verts[lp[i]]);
        for (int32_t v : verts) lab_set(v, -1);
    }

    void emit_vertex(int32_t v, std::vector<int32_t>& order) {   // separator vertex -> its original members
        if (compressed) for (int32_t q = mem_ptr[v]; q < mem_ptr[v + 1]; ++q) order.push_back(mem[q]);
        else order.push_back(v);
        lab_set(v, -1);
    }

    // When the level structure of the whole graph offers no separator (small-world graphs such as
    // block-angular problems with random linking rows), the result would be the AMD-class ordering
    // of everything: the caller can ask to be told instead of paying for it twice.
    bool skip_unsplit = false, unsplit = false;
    size_t root_size = 0;
    void leaf_or_skip(const std::vector<int32_t>& verts, std::vector<int32_t>& order) {
        if (skip_unsplit && verts.size() == root_size) { unsplit = true; return; }
        amd_leaf(verts, order);
    }

    struct Piece { std::vector<int32_t>* verts; bool leaf; };

    void run_one(const Piece& pc, std::vector<int32_t>& order, int64_t stamp) {
        if (pc.verts->empty()) return;
        if (pc.leaf) amd_leaf(*pc.verts, order); else dissect(*pc.verts, order, stamp);
    }

    // Order independent pieces and concatenate their orderings in list order.  Large pieces get a
    // thread of their own while the thread budget lasts; the result does not depend on the budget.
    void run_pieces(std::vector<Piece>& pieces, std::vector<int32_t>& order, int64_t stamp) {
        const size_t np = pieces.size();
        size_t nbig = 0;
        for (auto& pc : pieces) nbig += (!pc.leaf && pc.verts->size() >= PAR_MIN_VERTS);
        if (nbig < 2 || live_threads.load() >= max_threads) {
            for (auto& pc : pieces) run_one(pc, order, stamp);
            return;
        }
        std::vector<std::vector<int32_t>> outs(np);
        std::vector<std::exception_ptr> errs(np);
        std::vector<std::thread> threads;
        std::vector<size_t> mine;
        size_t big_left = nbig;
        for (size_t i = 0; i < np; ++i) {
            bool spawned = false;
            const bool big = !pieces[i].leaf && pieces[i].verts->size() >= PAR_MIN_VERTS;
            if (big && --big_left > 0) {                      // the last big piece stays on this thread
                int32_t cur = live_threads.load();
                while (cur < max_threads && !spawned)
                    if (live_threads.compare_exchange_weak(cur, cur + 1)) {
                        threads.emplace_back([this, &pieces, &outs, &errs, i, stamp] {
                            try { run_one(pieces[i], outs[i], stamp); } catch (...) { errs[i] = std::current_exception(); }
                            live_threads.fetch_sub(1);
                        });
                        spawned = true;
                    }
            }
            if (!spawned) mine.push_back(i);
        }
        for (size_t i : mine) {
            try { run_one(pieces[i], outs[i], stamp); } catch (...) { errs[i] = std::current_exception(); break; }
        }
        for (auto& t : threads) t.join();
        for (auto& e : errs) if (e) std::rethrow_exception(e);
        for (size_t i = 0; i < np; ++i) {
            order.insert(order.end(), outs[i].begin(), outs[i].end());
            std::vector<int32_t>().swap(outs[i]);
        }
    }

    // level stamps grow monotonically along every root-to-leaf path of the recursion (stamp is
    // passed by value), so level[] never needs clearing
    void dissect(std::vector<int32_t>& verts, std::vector<int32_t>& order, int64_t stamp) {
        // verts all carry the same label
        if (weight_of(verts) <= leaf_size || verts.size() == 1) { leaf_or_skip(verts, order); return; }
        int32_t lab = lab_get(verts[0]);
        // ---- connected components (each handled independently: no separator needed)
        std::vector<int32_t> q;
        {
            stamp += 2 * n + 4;
            int64_t base = stamp;
            bfs(verts[0], lab, q, base);
            if (q.size() < verts.size()) {
                // split into components
                std::vector<std::vector<int32_t>> comps;
                comps.emplace_back(q);
                for (int32_t v : verts)
                    if (level[v] < base) { bfs(v, lab, q, base); comps.emplace_back(q); }
                std::vector<int32_t>().swap(verts);
                // small components are batched together into one AMD leaf to limit overhead;
                // pieces keep their discovery order
                std::deque<std::vector<int32_t>> smalls;          // stable addresses
                std::vector<int32_t> small;
                std::vector<Piece> pieces;
                for (auto& c : comps) {
                    if (weight_of(c) <= leaf_size) {
                        small.insert(small.end(), c.begin(), c.end());
                        std::vector<int32_t>().swap(c);
                        if (weight_of(small) > leaf_size) {
                            smalls.emplace_back(std::move(small)); small.clear();
                            pieces.push_back({&smalls.back(), true});
                        }
                    } else pieces.push_back({&c, false});
                }
                if (!small.empty()) { smalls.emplace_back(std::move(small)); pieces.push_back({&smalls.back(), true}); }
                for (auto& pc : pieces) { const int32_t nl = next_label++; for (int32_t v : *pc.verts) lab_set(v, nl); }
                run_pieces(pieces, order, stamp);
                return;
            }
        }
        // ---- pseudo-peripheral root: repeat BFS from a min-degree vertex of the last level
        int32_t root = q.back(), nlev = 0;
        for (int it = 0; it < 4; ++it) {
            stamp += 2 * n + 4;
            int32_t nl = bfs(root, lab, q, stamp);
            if (nl <= nlev) { nlev = std::max(nlev, nl); break; }
            nlev = nl;
            int64_t last_level = level[q.back()];
            int32_t best = q.back(); int64_t bd = INT64_MAX;
            for (size_t i = q.size(); i-- > 0 && level[q[i]] == last_level;) {
                int64_t d = xadj[q[i] + 1] - xadj[q[i]];
                if (d < bd) { bd = d; best = q[i]; }
            }
            if (best == root) break;
            root = best;
        }
        stamp += 2 * n + 4;
        nlev = bfs(root, lab, q, stamp);
        int64_t base = stamp;
        if (nlev < 5) { leaf_or_skip(verts, order); return; }
        // ---- choose the smallest level in the middle half (by cumulative vertex count)
        std::vector<int64_t> lsize(nlev, 0);
        int64_t tot = 0;
        for (int32_t v : q) { const int64_t w = compressed ? wt[v] : 1; lsize[level[v] - base] += w; tot += w; }
        int64_t cum = 0;
        int32_t best = -1; double bestscore = 1e300;
        for (int32_t l = 0; l < nlev; ++l) {
            int64_t before = cum; cum += lsize[l];
            int64_t after = tot - cum;
            if (l == 0 || l == nlev - 1) continue;
            double bal = (double)std::min(before, after) / (double)tot;
            if (bal < 0.2) continue;
            double score = (double)lsize[l] / (0.1 + bal);
            if (score < bestscore) { bestscore = score; best = l; }
        }
        if (best < 0 || (double)lsize[best] > 0.25 * (double)tot) { leaf_or_skip(verts, order); return; }
        // ---- vertex separator from the edge cut between levels `best` and `best+1`: a minimum
        // vertex cover of the bipartite boundary graph (Koenig: maximum matching by Hopcroft-Karp,
        // then alternating reachability from the unmatched left vertices).  Never larger than the
        // one-sided choice "level-`best` vertices that touch level best+1".
        std::vector<int32_t> A, B, Sp;
        {
            std::vector<int32_t> X, Y;                       // boundary vertices of the two levels
            for (int32_t v : q) {
                const int32_t l = (int32_t)(level[v] - base);
                if (l == best || l == best + 1) local[v] = -1;
            }
            for (int32_t v : q) {
                const int32_t l = (int32_t)(level[v] - base);
                if (l != best) continue;
                bool touches = false;
                for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                    const int32_t u = adj[p];
                    if (lab_get(u) == lab && level[u] - base == best + 1) {
                        touches = true;
                        if (local[u] < 0) { local[u] = (int32_t)Y.size(); Y.push_back(u); }
                    }
                }
                if (touches) { local[v] = (int32_t)X.size(); X.push_back(v); }
            }
            const int32_t nx = (int32_t)X.size(), ny = (int32_t)Y.size();
            std::vector<int32_t> mx(nx, -1), my(ny, -1), dist(nx);
            auto ynbr = [&](int32_t xv, auto&& fn) {        // iterate Y-neighbours (local ids) of X[xv]
                const int32_t v = X[xv];
                for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                    const int32_t u = adj[p];
                    if (lab_get(u) == lab && level[u] - base == best + 1) if (!fn(local[u])) return;
                }
            };
            // Hopcroft-Karp
            std::vector<int32_t> bq;
            while (true) {
                bq.clear();
                for (int32_t i = 0; i < nx; ++i) { if (mx[i] < 0) { dist[i] = 0; bq.push_back(i); } else dist[i] = -1; }
                bool found = false;
                for (size_t h = 0; h < bq.size(); ++h) {
                    const int32_t i = bq[h];
                    ynbr(i, [&](int32_t yj) {
                        const int32_t i2 = my[yj];
                        if (i2 < 0) found = true;
                        else if (dist[i2] < 0) { dist[i2] = dist[i] + 1; bq.push_back(i2); }
                        return true;
                    });
                }
                if (!found) break;
                int32_t augmented = 0;
                // layered DFS (iterative) from every free left vertex
                std::vector<int64_t> itp(nx);
                std::vector<uint8_t> seen(nx, 0);
                for (int32_t i = 0; i < nx; ++i) itp[i] = xadj[X[i]];
                for (int32_t r = 0; r < nx; ++r) {
                    if (mx[r] >= 0) continue;
                    std::vector<int32_t> path{r};
                    while (!path.empty()) {
                        const int32_t i = path.back();
                        const int32_t v = X[i];
                        bool advanced = false;
                        while (itp[i] < xadj[v + 1]) {
                            const int32_t u = adj[itp[i]++];
                            if (!(lab_get(u) == lab && level[u] - base == best + 1)) continue;
                            const int32_t yj = local[u];
                            const int32_t i2 = my[yj];
                            if (i2 < 0) {
                                // augment along the path: path[k] takes the Y vertex it advanced through
                                int32_t cur_y = yj;
                                for (size_t k = path.size(); k-- > 0;) {
                                    const int32_t xi = path[k];
                                    const int32_t prev_y = mx[xi];
                                    mx[xi] = cur_y; my[cur_y] = xi;
                                    cur_y = prev_y;
                                }
                                path.clear(); advanced = true; ++augmented; break;
                            } else if (!seen[i2] && dist[i2] == dist[i] + 1) {
                                seen[i2] = 1;                // visit once per phase
                                path.push_back(i2); advanced = true; break;
                            }
                        }
                        if (!advanced && !path.empty()) path.pop_back();
                    }
                }
                if (augmented == 0) break;                   // safety: no progress in this phase
            }
            // Koenig: Z = reachable from free X by alternating paths ; cover = (X \ Z) u (Y n Z)
            std::vector<uint8_t> zx(nx, 0), zy(ny, 0);
            bq.clear();
            for (int32_t i = 0; i < nx; ++i) if (mx[i] < 0) { zx[i] = 1; bq.push_back(i); }
            for (size_t h = 0; h < bq.size(); ++h) {
                const int32_t i = bq[h];
                ynbr(i, [&](int32_t yj) {
                    if (!zy[yj]) {
                        zy[yj] = 1;
                        const int32_t i2 = my[yj];
                        if (i2 >= 0 && !zx[i2]) { zx[i2] = 1; bq.push_back(i2); }
                    }
                    return true;
                });
            }
            for (int32_t v : q) {
                const int32_t l = (int32_t)(level[v] - base);
                if (l < best) A.push_back(v);
                else if (l > best + 1) B.push_back(v);
                else if (l == best) {
                    const int32_t i = local[v];
                    if (i >= 0 && !zx[i]) Sp.push_back(v); else A.push_back(v);
                } else {
                    const int32_t j = local[v];
                    if (j >= 0 && zy[j]) Sp.push_back(v); else B.push_back(v);
                }
            }
        }
        std::vector<int32_t>().swap(verts);
        int32_t la = next_label++, lb = next_label++;
        for (int32_t v : A) lab_set(v, la);
        for (int32_t v : B) lab_set(v, lb);
        for (int32_t v : Sp) lab_set(v, -2);            // taken out of both halves
        std::vector<Piece> pieces{{&A, false}, {&B, false}};
        run_pieces(pieces, order, stamp);
        for (int32_t v : Sp) emit_vertex(v, order);
    }
};

}  // namespace

void nd_order_graph(int32_t n, const int64_t* xadj, const int32_t* adj, double dense_scale,
                    int32_t leaf_size, int32_t* perm_out) {
    nd_order_graph_blocks(n, xadj, adj, dense_scale, leaf_size, nullptr, perm_out);
}

// block_id (optional, length n): vertices sharing a block id >= 0 form a dense clique (a PSD or
// dense SOC cone block of the KKT matrix) that no separator may cut: they are contracted to one
// weighted vertex for the dissection and expanded again for the leaf orderings.
bool nd_order_graph_blocks(int32_t n, const int64_t* xadj, const int32_t* adj, double dense_scale,
                           int32_t leaf_size, const int32_t* block_id, int32_t* perm_out,
                           bool skip_unsplit) {
    if (n == 0) return true;
    NDCtx C; C.leaf_size = std::max(8, leaf_size); C.dense_scale = dense_scale;
    std::vector<int64_t> cx; std::vector<int32_t> ca;
    bool any_block = false;
    if (block_id) for (int32_t i = 0; i < n && !any_block; ++i) any_block = block_id[i] >= 0;
    if (any_block) {
        C.compressed = true; C.oxadj = xadj; C.oadj = adj; C.on = n;
        C.comp_of.assign(n, -1); C.olocal.assign(n, 0);
        int32_t maxb = -1;
        for (int32_t i = 0; i < n; ++i) maxb = std::max(maxb, block_id[i]);
        std::vector<int32_t> block_comp(maxb + 1, -1);
        int32_t nc = 0;
        for (int32_t i = 0; i < n; ++i) {
            const int32_t bid = block_id[i];
            if (bid >= 0) { if (block_comp[bid] < 0) block_comp[bid] = nc++; C.comp_of[i] = block_comp[bid]; }
            else C.comp_of[i] = nc++;
        }
        C.wt.assign(nc, 0); C.mem_ptr.assign(nc + 1, 0);
        for (int32_t i = 0; i < n; ++i) { C.wt[C.comp_of[i]]++; C.mem_ptr[C.comp_of[i] + 1]++; }
        for (int32_t c = 0; c < nc; ++c) C.mem_ptr[c + 1] += C.mem_ptr[c];
        C.mem.resize(n);
        { std::vector<int32_t> pos(C.mem_ptr.begin(), C.mem_ptr.end() - 1);
          for (int32_t i = 0; i < n; ++i) C.mem[pos[C.comp_of[i]]++] = i; }
        // compressed adjacency (deduplicated with a marker)
        cx.assign(nc + 1, 0);
        std::vector<int32_t> mark(nc, -1);
        for (int32_t c = 0; c < nc; ++c) {
            mark[c] = c;
            for (int32_t q = C.mem_ptr[c]; q < C.mem_ptr[c + 1]; ++q) {
                const int32_t v = C.mem[q];
                for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                    const int32_t cu = C.comp_of[adj[p]];
                    if (mark[cu] != c) { mark[cu] = c; ca.push_back(cu); }
                }
            }
            cx[c + 1] = (int64_t)ca.size();
        }
        C.n = nc; C.xadj = cx.data(); C.adj = ca.data();
    } else {
        C.n = n; C.xadj = xadj; C.adj = adj;
    }
    const int32_t gn = C.n;
    C.label.assign(gn, 0); C.level.assign(gn, -1); C.local.assign(gn, 0);
    std::vector<int32_t> order; order.reserve(n);
    {
        int32_t hw = (int32_t)std::thread::hardware_concurrency();
        C.max_threads = std::max(1, std::min(hw, 8));
        if (const char* e = getenv("CB200_ND_THREADS")) C.max_threads = std::max(1, atoi(e));
    }
    double dthr = dense_scale * 10.0 * std::sqrt((double)n);
    int64_t dense = (int64_t)std::max(16.0, std::min(dthr, (double)n));
    std::vector<int32_t> dense_nodes, verts;
    for (int32_t i = 0; i < gn; ++i) {
        const bool is_block = C.compressed && C.wt[i] > 1;
        if (!is_block && C.xadj[i + 1] - C.xadj[i] > dense) { dense_nodes.push_back(i); C.label[i] = -1; }
        else verts.push_back(i);
    }
    C.skip_unsplit = skip_unsplit; C.root_size = verts.size();
    if (!verts.empty()) C.dissect(verts, order, 0);
    if (C.unsplit) return false;
    std::sort(dense_nodes.begin(), dense_nodes.end(), [&](int32_t a, int32_t b) {
        int64_t da = C.xadj[a + 1] - C.xadj[a], db = C.xadj[b + 1] - C.xadj[b];
        return da < db || (da == db && a < b); });
    for (int32_t v : dense_nodes) C.emit_vertex(v, order);
    for (int32_t k = 0; k < n; ++k) perm_out[k] = order[k];
    return true;
}

// ------------------------------------------------------------------------------------------
// Ordering for KKT systems with dense cone blocks (PSD cones: cliques of n(n+1)/2 rows).
//   phase 1: every vertex outside the blocks (the primal variables, the rows of diagonal cones) in
//            the AMD-class order of their induced subgraph.  Late in the IP iteration a PSD block
//            Hs = (RR') (x)s (RR') has a dynamic range > 1e10; eliminating the variables it is
//            coupled to FIRST turns the block into the (negative definite, far better conditioned)
//            Schur complement -Hs - A P^-1 A' before any of its pivots is taken - that is what the
//            reference's AMD order does implicitly and what keeps the pivots' signs (DESIGN.md 5).
//   phase 2: the blocks themselves in a nested-dissection order of the block quotient graph (two
//            blocks are adjacent if a connected piece of the phase-1 vertices touches both), whole
//            blocks as separators, natural order inside a block.  The elimination of a definite
//            matrix is stable in any order, so phase 2 is free to trade flops for tree shape: a
//            chain of k coupled cones becomes a tree of depth log2 k whose fronts batch per level,
//            instead of a k-level chain of single large fronts (C4: 1463 levels -> 21).
// Returns false (perm_out untouched) when the structure does not fit: fewer than `min_blocks`
// blocks, or a phase-1 component that touches too many blocks (the quotient graph would be dense).
bool order_blocks_last_nd(int32_t n, const int64_t* xadj, const int32_t* adj, double dense_scale,
                          const int32_t* block_id, int32_t min_blocks, int32_t* perm_out) {
    if (!block_id || n == 0) return false;
    int32_t nb = 0;
    for (int32_t i = 0; i < n; ++i) nb = std::max(nb, block_id[i] + 1);
    if (nb < min_blocks) return false;
    std::vector<std::vector<int32_t>> members(nb);
    std::vector<int32_t> loc(n, -1), free_v;
    for (int32_t i = 0; i < n; ++i) {
        if (block_id[i] >= 0) members[block_id[i]].push_back(i);
        else { loc[i] = (int32_t)free_v.size(); free_v.push_back(i); }
    }
    const int32_t k = (int32_t)free_v.size();
    // ---- phase 1: AMD-class order of the induced subgraph of the free vertices
    std::vector<int32_t> order1(k);
    {
        std::vector<int64_t> lx(k + 1, 0); std::vector<int32_t> la;
        for (int32_t i = 0; i < k; ++i) {
            const int32_t v = free_v[i];
            for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) if (loc[adj[p]] >= 0) la.push_back(loc[adj[p]]);
            lx[i + 1] = (int64_t)la.size();
        }
        if (k > 0) amd_order_graph(k, lx.data(), la.data(), dense_scale, order1.data());
    }
    // ---- block quotient graph through the connected pieces of the free vertices
    std::vector<std::vector<int32_t>> H(nb);
    {
        std::vector<int32_t> comp(k, -1), stack, touched;
        std::vector<int32_t> mark(nb, -1);
        int32_t nc = 0;
        for (int32_t r = 0; r < k; ++r) {
            if (comp[r] >= 0) continue;
            touched.clear(); stack.assign(1, r); comp[r] = nc;
            while (!stack.empty()) {
                const int32_t u = stack.back(); stack.pop_back();
                const int32_t v = free_v[u];
                for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                    const int32_t w = adj[p];
                    if (loc[w] >= 0) { if (comp[loc[w]] < 0) { comp[loc[w]] = nc; stack.push_back(loc[w]); } }
                    else { const int32_t b = block_id[w]; if (mark[b] != nc) { mark[b] = nc; touched.push_back(b); } }
                }
            }
            if (touched.size() > 64) return false;
            for (size_t a = 0; a < touched.size(); ++a)
                for (size_t c = a + 1; c < touched.size(); ++c) { H[touched[a]].push_back(touched[c]); H[touched[c]].push_back(touched[a]); }
            ++nc;
        }
        for (int32_t b = 0; b < nb; ++b)                      // direct block-block entries
            for (int32_t v : members[b])
                for (int64_t p = xadj[v]; p < xadj[v + 1]; ++p) {
                    const int32_t b2 = block_id[adj[p]];
                    if (b2 >= 0 && b2 != b) H[b].push_back(b2);
                }
        for (auto& l : H) { std::sort(l.begin(), l.end()); l.erase(std::unique(l.begin(), l.end()), l.end()); }
    }
    // ---- phase 2: nested dissection of the quotient graph (weights = block sizes)
    std::vector<int32_t> border; border.reserve(nb);
    std::vector<int32_t> piece(nb, 0), lev(nb, -1);
    int32_t next_piece = 1;
    struct Rec {
        std::vector<std::vector<int32_t>>& H; std::vector<std::vector<int32_t>>& members;
        std::vector<int32_t>& piece; std::vector<int32_t>& lev; int32_t& next_piece; std::vector<int32_t>& out;
        void bfs(int32_t root, int32_t lab, std::vector<int32_t>& q) {
            q.assign(1, root); lev[root] = 0;
            for (size_t h = 0; h < q.size(); ++h)
                for (int32_t u : H[q[h]]) if (piece[u] == lab && lev[u] < 0) { lev[u] = lev[q[h]] + 1; q.push_back(u); }
        }
        void run(std::vector<int32_t> verts) {
            if (verts.empty()) return;
            if (verts.size() <= 2) { for (int32_t v : verts) { out.push_back(v); piece[v] = -1; } return; }
            const int32_t lab = piece[verts[0]];
            std::vector<int32_t> q;
            for (int32_t v : verts) lev[v] = -1;
            bfs(verts[0], lab, q);
            if (q.size() < verts.size()) {                    // disconnected: every component on its own
                std::vector<std::vector<int32_t>> comps; comps.push_back(q);
                for (int32_t v : verts) if (lev[v] < 0) { bfs(v, lab, q); comps.push_back(q); }
                for (auto& c : comps) { const int32_t nl = next_piece++; for (int32_t v : c) piece[v] = nl; }
                for (auto& c : comps) run(c);
                return;
            }
            int32_t root = q.back();                          // pseudo-peripheral: two more sweeps
            for (int it = 0; it < 2; ++it) { for (int32_t v : verts) lev[v] = -1; bfs(root, lab, q); root = q.back(); }
            for (int32_t v : verts) lev[v] = -1;
            bfs(root, lab, q);
            const int32_t nlev = lev[q.back()] + 1;
            if (nlev < 3) { for (int32_t v : q) { out.push_back(v); piece[v] = -1; } return; }
            std::vector<int64_t> lw(nlev, 0); int64_t tot = 0;
            for (int32_t v : q) { lw[lev[v]] += (int64_t)members[v].size(); tot += (int64_t)members[v].size(); }
            int32_t best = -1; double bs = 1e300; int64_t cum = 0;
            for (int32_t l = 0; l < nlev; ++l) {
                const int64_t before = cum; cum += lw[l];
                if (l == 0 || l == nlev - 1) continue;
                const double bal = (double)std::min(before, tot - cum) / (double)tot;
                const double score = (double)lw[l] / (0.05 + bal);
                if (score < bs) { bs = score; best = l; }
            }
            std::vector<int32_t> A, B, Sp;
            for (int32_t v : q) (lev[v] < best ? A : (lev[v] > best ? B : Sp)).push_back(v);
            const int32_t la = next_piece++, lb = next_piece++;
            for (int32_t v : A) piece[v] = la;
            for (int32_t v : B) piece[v] = lb;
            for (int32_t v : Sp) piece[v] = -2;
            run(A); run(B);
            for (int32_t v : Sp) { out.push_back(v); piece[v] = -1; }
        }
    } rec{H, members, piece, lev, next_piece, border};
    {
        std::vector<int32_t> all(nb); std::iota(all.begin(), all.end(), 0);
        rec.run(all);
    }
    if ((int32_t)border.size() != nb) return false;
    int32_t pos = 0;
    for (int32_t i = 0; i < k; ++i) perm_out[pos++] = free_v[order1[i]];
    for (int32_t b : border) for (int32_t v : members[b]) perm_out[pos++] = v;
    return pos == n;
}

}  // namespace cb200

extern "C" int32_t cb200_order_amd(int64_t n, const int64_t* colptr, const int64_t* rowval,
                                   double dense_scale, int64_t* perm) {
    if (n < 0 || n > 2000000000LL) return -1;
    std::vector<int64_t> xadj; std::vector<int32_t> adj;
    cb200::build_sym_graph(n, colptr, rowval, xadj, adj);
    std::vector<int32_t> p32(n);
    cb200::amd_order_graph((int32_t)n, xadj.data(), adj.data(), dense_scale, p32.data());
    for (int64_t i = 0; i < n; ++i) perm[i] = p32[i];
    return 0;
}

extern "C" int32_t cb200_order_nd(int64_t n, const int64_t* colptr, const int64_t* rowval,
                                  double dense_scale, int64_t leaf_size, int64_t* perm) {
    if (n < 0 || n > 2000000000LL) return -1;
    std::vector<int64_t> xadj; std::vector<int32_t> adj;
    cb200::build_sym_graph(n, colptr, rowval, xadj, adj);
    std::vector<int32_t> p32(n);
    cb200::nd_order_graph((int32_t)n, xadj.data(), adj.data(), dense_scale, (int32_t)leaf_size,
                          p32.data());
    for (int64_t i = 0; i < n; ++i) perm[i] = p32[i];
    return 0;
}
