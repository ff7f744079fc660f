// Supernodal multifrontal symbolic analysis (see symbolic.h).
#include "symbolic.h"
#include "ordering.h"

#include <algorithm>
#include <numeric>
#include <cstring>
#include <stdexcept>
#include <thread>
#include <exception>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>

namespace cb200 {

namespace {

// Elimination tree of the permuted matrix given its *upper* pattern by columns
// (Liu's algorithm with path compression).
void etree_upper(int32_t n, const std::vector<int64_t>& up, const std::vector<int32_t>& ui,
                 std::vector<int32_t>& parent) {
    parent.assign(n, -1);
    std::vector<int32_t> anc(n, -1);
    for (int32_t j = 0; j < n; ++j)
        for (int64_t p = up[j]; p < up[j + 1]; ++p) {
            int32_t i = ui[p];
            while (i != -1 && i < j) {
                int32_t nx = anc[i];
                anc[i] = j;
                if (nx == -1) parent[i] = j;
                i = nx;
            }
        }
}


// Factor cost (sum of squared column lengths) of the ordering ip (ip[orig] = position), with an
// early exit once `limit` is exceeded.  Used to arbitrate between the nested-dissection and the
// AMD-class ordering: BFS level-structure separators are poor on expander-like KKT graphs.
double ordering_cost(int32_t N, const int64_t* colptr, const int64_t* rowval,
                     const std::vector<int32_t>& ip, double limit, bool* aborted) {
    std::vector<int64_t> up(N + 1, 0), lp(N + 1, 0);
    for (int32_t j = 0; j < N; ++j)
        for (int64_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t a = ip[rowval[p]], b = ip[j];
            if (a == b) continue;
            up[std::max(a, b) + 1]++; lp[std::min(a, b) + 1]++;
        }
    for (int32_t j = 0; j < N; ++j) { up[j + 1] += up[j]; lp[j + 1] += lp[j]; }
    std::vector<int32_t> ui(up[N]), li(lp[N]);
    {
        std::vector<int64_t> pu(up.begin(), up.end() - 1), pl(lp.begin(), lp.end() - 1);
        for (int32_t j = 0; j < N; ++j)
            for (int64_t p = colptr[j]; p < colptr[j + 1]; ++p) {
                int32_t a = ip[rowval[p]], b = ip[j];
                if (a == b) continue;
                int32_t lo = std::min(a, b), hi = std::max(a, b);
                ui[pu[hi]++] = lo; li[pl[lo]++] = hi;
            }
    }
    std::vector<int32_t> parent;
    etree_upper(N, up, ui, parent);
    std::vector<int32_t> cptr(N + 1, 0), clist(N);
    for (int32_t j = 0; j < N; ++j) if (parent[j] >= 0) cptr[parent[j] + 1]++;
    for (int32_t j = 0; j < N; ++j) cptr[j + 1] += cptr[j];
    { std::vector<int32_t> pos(cptr.begin(), cptr.end() - 1);
      for (int32_t j = 0; j < N; ++j) if (parent[j] >= 0) clist[pos[parent[j]]++] = j; }
    std::vector<std::vector<int32_t>> lists(N);
    std::vector<int32_t> mark(N, -1);
    double flops = 0;
    *aborted = false;
    for (int32_t j = 0; j < N; ++j) {
        auto& L = lists[j];
        mark[j] = j;
        for (int64_t p = lp[j]; p < lp[j + 1]; ++p) { int32_t i = li[p]; if (mark[i] != j) { mark[i] = j; L.push_back(i); } }
        for (int32_t q = cptr[j]; q < cptr[j + 1]; ++q) {
            auto& C = lists[clist[q]];
            for (int32_t i : C) if (mark[i] != j) { mark[i] = j; L.push_back(i); }
            std::vector<int32_t>().swap(C);
        }
        const double c = (double)L.size() + 1.0;
        flops += c * c;
        if (flops > limit) { *aborted = true; return flops; }
        if (parent[j] < 0) std::vector<int32_t>().swap(L);
    }
    return flops;
}

}  // namespace

void symbolic_analyze(int64_t N64, const int64_t* colptr, const int64_t* rowval,
                      const SymbolicOptions& opt, const int64_t* user_perm, Symbolic& S) {
    if (N64 > 2000000000LL) throw std::runtime_error("N too large for int32 indices");
    const int32_t N = (int32_t)N64;
    const int64_t nnzK = colptr[N];
    S.N = N; S.nnzK = nnzK;
    const bool verbose = getenv("CB200_SYM_VERBOSE") != nullptr;     // phase times on stderr
    auto t_last = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        if (!verbose) return;
        auto t = std::chrono::steady_clock::now();
        fprintf(stderr, "[cb200 symbolic] %-28s %8.3f s\n", what, std::chrono::duration<double>(t - t_last).count());
        t_last = t;
    };

    // ---------------------------------------------------------------- 1. fill-reducing order
    std::vector<int32_t> p0(N);
    if (user_perm) {
        for (int32_t i = 0; i < N; ++i) p0[i] = (int32_t)user_perm[i];
        S.ordering_used = 3;
    } else if (opt.ordering == 2) {
        std::iota(p0.begin(), p0.end(), 0);
        S.ordering_used = 2;
    } else {
        S.ordering_used = 0;
        std::vector<int64_t> xadj; std::vector<int32_t> adj;
        build_sym_graph(N, colptr, rowval, xadj, adj);
        bool has_blocks = false;
        if (opt.block_id) for (int32_t i = 0; i < N && !has_blocks; ++i) has_blocks = opt.block_id[i] >= 0;
        if (opt.ordering != 1) {
            amd_order_graph(N, xadj.data(), adj.data(), opt.dense_scale, p0.data());
        } else if (has_blocks) {
            // dense cone blocks (PSD): their coupled variables first, then the blocks by nested
            // dissection of the block graph; the AMD-class order when that structure does not fit.
            // The generic vertex dissection below is never used here (it may eliminate a block before
            // the variables it is coupled to: wrong-sign pivots late in the iteration, DESIGN.md 5).
            if (order_blocks_last_nd(N, xadj.data(), adj.data(), opt.dense_scale, opt.block_id, opt.min_cone_blocks, p0.data()))
                S.ordering_used = 4;
            else
                amd_order_graph(N, xadj.data(), adj.data(), opt.dense_scale, p0.data());
        } else {
            // auto: nested dissection (shallow, wide trees for the level-scheduled kernels and the
            // multi-GPU split) unless it costs more than nd_max_cost_ratio x the AMD-class ordering.
            // The two orderings are independent, so they run on two host threads.
            std::vector<int32_t> pn(N), ipa(N), ipn(N);
            bool ab = false;
            double fa = 0;
            std::exception_ptr err;
            std::atomic<bool> want_cost{true};
            std::thread amd_thread([&] {
                try {
                    amd_order_graph(N, xadj.data(), adj.data(), opt.dense_scale, p0.data());
                    if (!want_cost.load()) return;
                    for (int32_t k = 0; k < N; ++k) ipa[p0[k]] = k;
                    bool dummy = false;
                    fa = ordering_cost(N, colptr, rowval, ipa, 1e300, &dummy);
                } catch (...) { err = std::current_exception(); }
            });
            bool split = false;
            try {
                split = nd_order_graph_blocks(N, xadj.data(), adj.data(), opt.dense_scale, opt.nd_leaf,
                                              opt.block_id, pn.data(), /*skip_unsplit=*/true);
            } catch (...) { amd_thread.join(); throw; }
            if (!split) want_cost.store(false);              // nothing to arbitrate: AMD it is
            lap("  nested dissection");
            amd_thread.join();
            lap("  wait for amd thread");
            if (err) std::rethrow_exception(err);
            if (split) {
                for (int32_t k = 0; k < N; ++k) ipn[pn[k]] = k;
                ordering_cost(N, colptr, rowval, ipn, opt.nd_max_cost_ratio * fa, &ab);
                if (!ab) { p0.swap(pn); S.ordering_used = 1; }
                lap("  nd cost + arbitration");
            }
        }
    }
    lap("ordering");
    std::vector<int32_t> ip0(N);
    for (int32_t k = 0; k < N; ++k) ip0[p0[k]] = k;

    // permuted pattern as upper-by-column (row < col) == lower-by-row; also lower-by-column
    auto build_patterns = [&](const std::vector<int32_t>& ip, std::vector<int64_t>& up,
                              std::vector<int32_t>& ui, std::vector<int64_t>& lp,
                              std::vector<int32_t>& li) {
        up.assign(N + 1, 0); lp.assign(N + 1, 0);
        for (int32_t j = 0; j < N; ++j)
            for (int64_t p = colptr[j]; p < colptr[j + 1]; ++p) {
                int32_t a = ip[rowval[p]], b = ip[j];
                if (a == b) continue;
                int32_t lo = std::min(a, b), hi = std::max(a, b);
                up[hi + 1]++; lp[lo + 1]++;
            }
        for (int32_t j = 0; j < N; ++j) { up[j + 1] += up[j]; lp[j + 1] += lp[j]; }
        ui.resize(up[N]); li.resize(lp[N]);
        std::vector<int64_t> pu(up.begin(), up.end() - 1), pl(lp.begin(), lp.end() - 1);
        for (int32_t j = 0; j < N; ++j)
            for (int64_t p = colptr[j]; p < colptr[j + 1]; ++p) {
                int32_t a = ip[rowval[p]], b = ip[j];
                if (a == b) continue;
                int32_t lo = std::min(a, b), hi = std::max(a, b);
                ui[pu[hi]++] = lo; li[pl[lo]++] = hi;
            }
    };
    std::vector<int64_t> up, lp; std::vector<int32_t> ui, li;
    build_patterns(ip0, up, ui, lp, li);

    // ---------------------------------------------------------------- 2. etree + column counts
    std::vector<int32_t> parent;
    etree_upper(N, up, ui, parent);
    std::vector<int32_t> cptr(N + 1, 0), clist(N);
    auto build_children = [&](const std::vector<int32_t>& par) {
        std::fill(cptr.begin(), cptr.end(), 0);
        for (int32_t j = 0; j < N; ++j) if (par[j] >= 0) cptr[par[j] + 1]++;
        for (int32_t j = 0; j < N; ++j) cptr[j + 1] += cptr[j];
        std::vector<int32_t> pos(cptr.begin(), cptr.end() - 1);
        for (int32_t j = 0; j < N; ++j) if (par[j] >= 0) clist[pos[par[j]]++] = j;
    };
    build_children(parent);
    // column structures by list merging (children are always numbered below their parent)
    std::vector<int32_t> count(N, 0);
    {
        std::vector<std::vector<int32_t>> lists(N);
        std::vector<int32_t> mark(N, -1);
        for (int32_t j = 0; j < N; ++j) {
            auto& L = lists[j];
            mark[j] = j;
            for (int64_t p = lp[j]; p < lp[j + 1]; ++p) {
                int32_t i = li[p];
                if (mark[i] != j) { mark[i] = j; L.push_back(i); }
            }
            for (int32_t q = cptr[j]; q < cptr[j + 1]; ++q) {
                auto& C = lists[clist[q]];
                for (int32_t i : C) if (mark[i] != j) { mark[i] = j; L.push_back(i); }
                std::vector<int32_t>().swap(C);
            }
            count[j] = (int32_t)L.size();
            if (parent[j] < 0) std::vector<int32_t>().swap(L);
        }
    }

    lap("etree + column counts");
    // ---------------------------------------------------------------- 3. postorder (big child last)
    std::vector<int32_t> post(N), ipost(N);
    {
        // sort each child list by count ascending so the heaviest child is visited last
        for (int32_t j = 0; j < N; ++j)
            std::sort(clist.begin() + cptr[j], clist.begin() + cptr[j + 1],
                      [&](int32_t a, int32_t b) { return count[a] < count[b] || (count[a] == count[b] && a < b); });
        std::vector<int32_t> stack, it(N, 0);
        int32_t k = 0;
        for (int32_t r = 0; r < N; ++r) {
            if (parent[r] >= 0) continue;
            stack.push_back(r);
            while (!stack.empty()) {
                int32_t v = stack.back();
                if (cptr[v] + it[v] < cptr[v + 1]) { stack.push_back(clist[cptr[v] + it[v]++]); }
                else { post[k++] = v; stack.pop_back(); }
            }
        }
        for (int32_t q = 0; q < N; ++q) ipost[post[q]] = q;
    }
    S.perm.resize(N); S.iperm.resize(N);
    for (int32_t q = 0; q < N; ++q) S.perm[q] = p0[post[q]];
    for (int32_t q = 0; q < N; ++q) S.iperm[S.perm[q]] = q;
    {   // relabel parent / count into postorder
        std::vector<int32_t> par2(N), cnt2(N);
        for (int32_t q = 0; q < N; ++q) {
            int32_t v = post[q];
            par2[q] = parent[v] >= 0 ? ipost[parent[v]] : -1;
            cnt2[q] = count[v];
        }
        parent.swap(par2); count.swap(cnt2);
    }
    build_patterns(S.iperm, up, ui, lp, li);
    std::vector<int64_t>().swap(up); std::vector<int32_t>().swap(ui);

    // ---------------------------------------------------------------- 4. maximal supernodes
    std::vector<int32_t> first;      // first column of each (fundamental/maximal) supernode
    first.push_back(0);
    for (int32_t j = 1; j < N; ++j)
        if (!(parent[j - 1] == j && count[j - 1] == count[j] + 1)) first.push_back(j);
    int32_t nsn = (int32_t)first.size();
    if (N == 0) { nsn = 0; first.clear(); }
    first.push_back(N);
    std::vector<int32_t> snof(N);
    for (int32_t s = 0; s < nsn; ++s) for (int32_t j = first[s]; j < first[s + 1]; ++j) snof[j] = s;
    // supernodal tree
    std::vector<int32_t> spar(nsn, -1);
    for (int32_t s = 0; s < nsn; ++s) {
        int32_t last = first[s + 1] - 1;
        spar[s] = parent[last] >= 0 ? snof[parent[last]] : -1;
    }
    // ---------------------------------------------------------------- 5. relaxed amalgamation
    // Merge supernode c into its parent p when c is p's immediately preceding sibling-free
    // neighbour in postorder (first[c+1] == first[p]) and the padding zeros stay small.
    std::vector<int32_t> merged_into(nsn, -1);         // c -> p
    {
        std::vector<int64_t> zeros(nsn, 0);
        std::vector<int32_t> width(nsn), below(nsn), head(nsn);   // head: first column after merges
        for (int32_t s = 0; s < nsn; ++s) {
            width[s] = first[s + 1] - first[s];
            below[s] = count[first[s + 1] - 1];      // rows below the supernode's last column
            head[s] = first[s];
        }
        // 5a. subtree collapse: the bottom of the tree consists of millions of 1-8 column supernodes
        // (a leaf column and its few neighbours).  A subtree whose merged front is tiny is stored and
        // processed as ONE dense supernode: the columns of a subtree are contiguous in postorder, the
        // rows below are those of its root, and the padding zeros cost less than the index traffic
        // and the per-supernode latency they replace.
        if (opt.collapse_nf > 0) {
            std::vector<int32_t> sub_sn(nsn, 1);
            std::vector<int64_t> sub_cols(nsn), sub_true(nsn);
            for (int32_t s = 0; s < nsn; ++s) {
                sub_cols[s] = width[s];
                int64_t t = 0;
                for (int32_t j = first[s]; j < first[s + 1]; ++j) t += (int64_t)count[j] + 1;
                sub_true[s] = t;
            }
            for (int32_t s = 0; s < nsn; ++s) if (spar[s] >= 0) {
                sub_sn[spar[s]] += sub_sn[s]; sub_cols[spar[s]] += sub_cols[s]; sub_true[spar[s]] += sub_true[s];
            }
            for (int32_t p = nsn - 1; p >= 0; --p) {
                if (merged_into[p] >= 0 || sub_sn[p] == 1) continue;
                const int64_t w = sub_cols[p];
                if (w + below[p] > opt.collapse_nf || w > opt.max_width) continue;
                for (int32_t d = p - sub_sn[p] + 1; d < p; ++d) merged_into[d] = p;
                width[p] = (int32_t)w; head[p] = first[p - sub_sn[p] + 1];
                zeros[p] = w * (w + 1) / 2 + w * (int64_t)below[p] - sub_true[p];
            }
        }
        for (int32_t p = 0; p < nsn; ++p) {
            if (merged_into[p] >= 0) continue;      // inside a collapsed subtree
            // candidate: the supernode ending right before head[p] whose parent is p
            while (true) {
                if (head[p] == 0) break;
                int32_t c = snof[head[p] - 1];
                while (merged_into[c] >= 0) c = merged_into[c];   // representative (never p itself)
                if (c == p || spar[c] != p) break;
                int32_t wc = width[c], wp = width[p];
                int32_t w = wc + wp;
                if (w > opt.max_width) break;
                int64_t newz = (int64_t)wc * ((int64_t)wp + below[p] - below[c]);
                int64_t z = zeros[c] + zeros[p] + newz;
                double total = (double)w * (w + 1) / 2.0 + (double)w * below[p];
                double frac = (double)z / total;
                bool ok = (w <= opt.relax_small) ||
                          (w <= 32 && frac < opt.relax_z1) ||
                          (w <= 96 && frac < opt.relax_z2) || (frac < opt.relax_z3);
                if (!ok) break;
                merged_into[c] = p;
                zeros[p] = z; width[p] = w; head[p] = head[c];
                // c's children now hang off p
            }
        }
    }
    // final supernodes: survivors, with their merged column ranges
    std::vector<int32_t> rep(nsn);
    for (int32_t s = 0; s < nsn; ++s) {
        int32_t r = s;
        while (merged_into[r] >= 0) r = merged_into[r];
        rep[s] = r;
    }
    std::vector<int32_t> newid(nsn, -1);
    S.sn_first.clear();
    int32_t ns2 = 0;
    for (int32_t s = 0; s < nsn; ++s) {
        // a merged group is contiguous and ends with its representative; its first member is
        // the first s with rep[s] == r
        if (s == 0 || rep[s] != rep[s - 1]) { S.sn_first.push_back(first[s]); newid[rep[s]] = ns2++; }
    }
    S.sn_first.push_back(N);
    S.nsuper = ns2;
    S.sn_of_col.resize(N);
    for (int32_t s = 0; s < ns2; ++s)
        for (int32_t j = S.sn_first[s]; j < S.sn_first[s + 1]; ++j) S.sn_of_col[j] = s;
    S.sn_parent.assign(ns2, -1);
    for (int32_t s = 0; s < ns2; ++s) {
        int32_t last = S.sn_first[s + 1] - 1;
        S.sn_parent[s] = parent[last] >= 0 ? S.sn_of_col[parent[last]] : -1;
    }
    S.child_ptr.assign(ns2 + 1, 0);
    for (int32_t s = 0; s < ns2; ++s) if (S.sn_parent[s] >= 0) S.child_ptr[S.sn_parent[s] + 1]++;
    for (int32_t s = 0; s < ns2; ++s) S.child_ptr[s + 1] += S.child_ptr[s];
    S.child_list.resize(S.child_ptr[ns2]);
    {
        std::vector<int32_t> pos(S.child_ptr.begin(), S.child_ptr.end() - 1);
        for (int32_t s = 0; s < ns2; ++s) if (S.sn_parent[s] >= 0) S.child_list[pos[S.sn_parent[s]]++] = s;
    }

    lap("postorder + supernodes");
    // ---------------------------------------------------------------- 6. supernodal row structures
    S.rows_ptr.assign(ns2 + 1, 0);
    {
        std::vector<std::vector<int32_t>> R(ns2);
        std::vector<int32_t> mark(N, -1);
        for (int32_t s = 0; s < ns2; ++s) {
            int32_t f = S.sn_first[s], l = S.sn_first[s + 1] - 1;
            auto& L = R[s];
            for (int32_t j = f; j <= l; ++j)
                for (int64_t p = lp[j]; p < lp[j + 1]; ++p) {
                    int32_t i = li[p];
                    if (i > l && mark[i] != s) { mark[i] = s; L.push_back(i); }
                }
            for (int32_t q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q)
                for (int32_t i : R[S.child_list[q]])
                    if (i > l && mark[i] != s) { mark[i] = s; L.push_back(i); }
            std::sort(L.begin(), L.end());
            S.rows_ptr[s + 1] = S.rows_ptr[s] + (int64_t)L.size();
        }
        S.rows.resize(S.rows_ptr[ns2]);
        for (int32_t s = 0; s < ns2; ++s)
            std::copy(R[s].begin(), R[s].end(), S.rows.begin() + S.rows_ptr[s]);
    }
    // parent consistency: the assembly parent must own the first below-row
    for (int32_t s = 0; s < ns2; ++s) {
        if (S.nr(s) > 0) {
            int32_t ps = S.sn_of_col[S.rows[S.rows_ptr[s]]];
            if (ps != S.sn_parent[s]) S.sn_parent[s] = ps;   // (amalgamation keeps this equal)
        } else S.sn_parent[s] = -1;
    }
    // rebuild children in case the loop above changed anything
    std::fill(S.child_ptr.begin(), S.child_ptr.end(), 0);
    for (int32_t s = 0; s < ns2; ++s) if (S.sn_parent[s] >= 0) S.child_ptr[S.sn_parent[s] + 1]++;
    for (int32_t s = 0; s < ns2; ++s) S.child_ptr[s + 1] += S.child_ptr[s];
    S.child_list.resize(S.child_ptr[ns2]);
    {
        std::vector<int32_t> pos(S.child_ptr.begin(), S.child_ptr.end() - 1);
        for (int32_t s = 0; s < ns2; ++s) if (S.sn_parent[s] >= 0) S.child_list[pos[S.sn_parent[s]]++] = s;
    }

    lap("row structures");
    // ---------------------------------------------------------------- 7. storage + maps
    S.panel_off.assign(ns2 + 1, 0); S.upd_off.assign(ns2 + 1, 0); S.panel_ld.assign(ns2, 0);
    S.nnzL = 0; S.flops = 0; S.max_front = 0; S.max_width = 0;
    {
        int64_t off = 0;
        for (int32_t s = 0; s < ns2; ++s) {
            const int64_t w = S.ns(s), nf = w + S.nr(s);
            int64_t ld = nf;
            if (front_is_large(opt, (int)nf, (int)w)) {
                ld = (nf + LD_ALIGN - 1) / LD_ALIGN * LD_ALIGN;
                off = (off + LD_ALIGN - 1) / LD_ALIGN * LD_ALIGN;
            }
            S.panel_ld[s] = (int32_t)ld;
            S.panel_off[s] = off;
            off += ld * w;
        }
        S.panel_off[ns2] = off;
    }
    for (int32_t s = 0; s < ns2; ++s) {
        int64_t w = S.ns(s), r = S.nr(s), nf = w + r;
        S.upd_off[s + 1] = S.upd_off[s] + r * r;
        S.nnzL += w * (w - 1) / 2 + w * r;
        for (int64_t k = 0; k < w; ++k) { double c = (double)(nf - k); S.flops += c * c; }
        S.max_front = std::max<int32_t>(S.max_front, (int32_t)nf);
        S.max_width = std::max<int32_t>(S.max_width, (int32_t)w);
    }
    S.upd_total = S.upd_off[ns2];
    // relative indices of R_s in the parent's front
    S.rel.resize(S.rows.size());
    for (int32_t s = 0; s < ns2; ++s) {
        int32_t p = S.sn_parent[s];
        if (p < 0) continue;
        int32_t pf = S.sn_first[p], pl = S.sn_first[p + 1] - 1, pw = pl - pf + 1;
        const int32_t* PR = S.rows.data() + S.rows_ptr[p];
        int32_t pnr = S.nr(p);
        int32_t cur = 0;
        for (int64_t q = S.rows_ptr[s]; q < S.rows_ptr[s + 1]; ++q) {
            int32_t r = S.rows[q];
            if (r <= pl) { S.rel[q] = r - pf; }
            else {
                while (cur < pnr && PR[cur] < r) cur++;
                if (cur >= pnr || PR[cur] != r) throw std::runtime_error("symbolic: child row not in parent front");
                S.rel[q] = pw + cur;
            }
        }
    }
    // destination-owner assembly maps
    {
        S.front_ptr.assign(ns2 + 1, 0); S.asm_base.assign(ns2 + 1, 0);
        for (int32_t s = 0; s < ns2; ++s) {
            int64_t nf = (int64_t)S.ns(s) + S.nr(s);
            S.front_ptr[s + 1] = S.front_ptr[s] + nf + 1;
            int64_t cnt = 0;
            for (int32_t q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) cnt += S.nr(S.child_list[q]);
            S.asm_base[s + 1] = S.asm_base[s] + cnt;
        }
        if (S.asm_base[ns2] > 2000000000LL || (int64_t)S.rows.size() > 2000000000LL)
            throw std::runtime_error("symbolic: assembly map exceeds int32 indexing");
        S.asm_colptr.assign(S.front_ptr[ns2], 0);
        S.asm_src.resize(S.asm_base[ns2]); S.asm_child.resize(S.asm_base[ns2]);
        for (int32_t s = 0; s < ns2; ++s) {
            int32_t* cp = S.asm_colptr.data() + S.front_ptr[s];
            const int64_t nf = (int64_t)S.ns(s) + S.nr(s);
            for (int32_t q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
                int32_t c = S.child_list[q];
                for (int64_t r = S.rows_ptr[c]; r < S.rows_ptr[c + 1]; ++r) cp[S.rel[r] + 1]++;
            }
            for (int64_t d = 0; d < nf; ++d) cp[d + 1] += cp[d];
            std::vector<int32_t> pos(cp, cp + nf);
            for (int32_t q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
                int32_t c = S.child_list[q];
                for (int64_t r = S.rows_ptr[c]; r < S.rows_ptr[c + 1]; ++r) {
                    int64_t e = S.asm_base[s] + pos[S.rel[r]]++;
                    S.asm_src[e] = (int32_t)r; S.asm_child[e] = c;
                }
            }
        }
        S.kids.resize(S.child_list.size());
        for (size_t q = 0; q < S.child_list.size(); ++q) {
            const int32_t c = S.child_list[q];
            S.kids[q] = {S.upd_off[c], S.rows_ptr[c], S.nr(c), 0};
        }
    }
    // scatter map of the original K entries into the panels
    S.a_map.resize(nnzK);
    for (int32_t j = 0; j < N; ++j)
        for (int64_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t a = S.iperm[rowval[p]], b = S.iperm[j];
            int32_t c = std::min(a, b), r = std::max(a, b);
            int32_t s = S.sn_of_col[c];
            int32_t f = S.sn_first[s], l = S.sn_first[s + 1] - 1, w = l - f + 1;
            int64_t nf = S.panel_ld[s];
            int64_t lr;
            if (r <= l) lr = r - f;
            else {
                const int32_t* Rb = S.rows.data() + S.rows_ptr[s];
                const int32_t* Re = Rb + S.nr(s);
                const int32_t* it = std::lower_bound(Rb, Re, r);
                if (it == Re || *it != r) throw std::runtime_error("symbolic: K entry outside front");
                lr = w + (it - Rb);
            }
            S.a_map[p] = S.panel_off[s] + (int64_t)(c - f) * nf + lr;
        }

    lap("storage + maps");
    // ---------------------------------------------------------------- 8. level sets
    S.sn_level.assign(ns2, 0);
    int32_t nl = 0;
    for (int32_t s = 0; s < ns2; ++s) {          // children precede parents
        int32_t p = S.sn_parent[s];
        if (p >= 0) S.sn_level[p] = std::max(S.sn_level[p], S.sn_level[s] + 1);
        nl = std::max(nl, S.sn_level[s] + 1);
    }
    S.nlevels = nl;
    S.level_ptr.assign(nl + 1, 0);
    for (int32_t s = 0; s < ns2; ++s) S.level_ptr[S.sn_level[s] + 1]++;
    for (int32_t l = 0; l < nl; ++l) S.level_ptr[l + 1] += S.level_ptr[l];
    S.level_list.resize(ns2);
    {
        std::vector<int32_t> pos(S.level_ptr.begin(), S.level_ptr.end() - 1);
        for (int32_t s = 0; s < ns2; ++s) S.level_list[pos[S.sn_level[s]]++] = s;
    }
}

void partition_subtrees(const Symbolic& S, int32_t nranks, std::vector<int32_t>& owner,
                        std::vector<int8_t>& is_top, std::vector<double>* rank_load) {
    const int32_t n = S.nsuper;
    owner.assign(n, 0); is_top.assign(n, 0);
    if (rank_load) rank_load->assign(std::max(1, nranks), 0.0);
    if (n == 0) return;
    // subtree weights (factor flops of the front, accumulated upwards; children precede parents)
    std::vector<double> wself(n), wsub(n);
    for (int32_t s = 0; s < n; ++s) {
        const double w = S.ns(s), nf = w + S.nr(s);
        wself[s] = w * nf * nf + 1.0;
        wsub[s] = wself[s];
    }
    for (int32_t s = 0; s < n; ++s) if (S.sn_parent[s] >= 0) wsub[S.sn_parent[s]] += wsub[s];
    double total = 0;
    std::vector<int32_t> cand;                       // roots of the current subtree forest
    for (int32_t s = 0; s < n; ++s) if (S.sn_parent[s] < 0) { cand.push_back(s); total += wsub[s]; }
    if (nranks <= 1) return;
    // Grow the top set: repeatedly move the heaviest candidate root into it (exposing its children)
    // until there are enough subtrees to balance: heaviest <= total / (2 * nranks) or nothing to split.
    auto heavier = [&](int32_t a, int32_t b) { return wsub[a] < wsub[b]; };
    std::make_heap(cand.begin(), cand.end(), heavier);
    double top_w = 0;
    while (!cand.empty()) {
        const int32_t h = cand.front();
        const bool need_more = (int32_t)cand.size() < 2 * nranks;
        const bool too_heavy = wsub[h] > (total - top_w) / (1.5 * nranks);
        if (!(need_more || too_heavy)) break;
        if (S.child_ptr[h + 1] == S.child_ptr[h]) break;        // a leaf: cannot split further
        if (top_w + wself[h] > 0.5 * total && !need_more) break; // do not replicate most of the work
        std::pop_heap(cand.begin(), cand.end(), heavier); cand.pop_back();
        is_top[h] = 1; top_w += wself[h];
        for (int32_t q = S.child_ptr[h]; q < S.child_ptr[h + 1]; ++q) {
            cand.push_back(S.child_list[q]);
            std::push_heap(cand.begin(), cand.end(), heavier);
        }
    }
    // LPT assignment of whole subtrees
    std::sort(cand.begin(), cand.end(), [&](int32_t a, int32_t b) { return wsub[a] > wsub[b] || (wsub[a] == wsub[b] && a < b); });
    std::vector<double> load(nranks, 0.0);
    std::vector<int32_t> root_owner(n, -1);
    for (int32_t r : cand) {
        int32_t best = 0;
        for (int32_t k = 1; k < nranks; ++k) if (load[k] < load[best]) best = k;
        root_owner[r] = best; load[best] += wsub[r];
    }
    // propagate ownership down (parents have larger indices than children)
    for (int32_t s = n - 1; s >= 0; --s) {
        if (is_top[s]) { owner[s] = -1; continue; }
        if (root_owner[s] >= 0) owner[s] = root_owner[s];
        else owner[s] = owner[S.sn_parent[s]];
    }
    if (rank_load) *rank_load = load;
}

void build_tile_lists(const Symbolic& S, const int32_t* fronts, int32_t n, int32_t T, bool schur,
                      bool gather, const int8_t* active, std::vector<TileEntry>& tiles,
                      std::vector<TileRect>& rects) {
    std::vector<int32_t> bnd;                        // per child: first child row at or below each tile boundary
    for (int32_t k = 0; k < n; ++k) {
        const int32_t s = fronts[k];
        const int32_t ns = S.ns(s), nf = ns + S.nr(s);
        const int32_t c0 = S.child_ptr[s], nch = S.child_ptr[s + 1] - c0;
        const bool gathers = gather && nch <= MANY_CHILDREN;
        if (schur ? nf == ns : (nch > MANY_CHILDREN || nch == 0)) continue;
        const int32_t nt = (nf - 1) / T + 1;          // tiles per side
        const int32_t nb = nt + 2;                    // boundaries 0..nt, then lower_bound(ns)
        const bool with_rects = !schur || gathers;
        if (with_rects) {
            bnd.assign((size_t)nch * nb, 0);
            for (int32_t q = 0; q < nch; ++q) {
                const int32_t c = S.child_list[c0 + q];
                if (active && !active[c]) continue;
                const int32_t* relc = S.rel.data() + S.rows_ptr[c];
                const int32_t nrc = S.nr(c);
                int32_t* b = bnd.data() + (size_t)q * nb;
                for (int32_t t = 0, i = 0; t <= nt; ++t) {
                    while (i < nrc && relc[i] < t * T) ++i;
                    b[t] = i;
                }
                b[nt + 1] = (int32_t)(std::lower_bound(relc, relc + nrc, ns) - relc);
            }
        }
        const int32_t chi = schur ? nf : (gathers ? ns : nf);      // columns [clo, chi) are assembled here
        const int32_t clo = schur ? ns : 0;
        for (int32_t tj = clo / T; tj * T < chi; ++tj)
            for (int32_t ti = tj; ti < nt; ++ti) {
                const size_t r0 = rects.size();
                if (with_rects)
                    for (int32_t q = 0; q < nch; ++q) {
                        if (active && !active[S.child_list[c0 + q]]) continue;
                        const int32_t* b = bnd.data() + (size_t)q * nb;
                        const int32_t nrc = S.nr(S.child_list[c0 + q]);
                        const int32_t ja = std::max(b[tj], schur ? b[nt + 1] : 0);
                        const int32_t ia = b[ti], ib = b[ti + 1];
                        const int32_t jb = std::min({b[tj + 1], ib, chi == ns ? b[nt + 1] : nrc});
                        if (ja < jb && ia < ib) rects.push_back({S.child_list[c0 + q], ja, jb, ia, ib, {0, 0, 0}});
                    }
                if (schur || rects.size() > r0) tiles.push_back({k, ti, tj, (int32_t)r0});
            }
    }
}

}  // namespace cb200
