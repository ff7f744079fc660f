// Supernodal multifrontal symbolic analysis of the permuted KKT pattern (host, setup-time).
// Replaces the symbolic half of QDLDL.qdldl(...; logical=true) at the reference call site
// src/kktsolvers/direct-ldl/directldl_qdldl.jl:18-25 (F0 in SURVEY.md section 8a): ordering,
// elimination tree, supernodes, front structures, assembly (extend-add) maps, level sets.
#pragma once
#include <cstdint>
#include <vector>

namespace cb200 {

struct SymbolicOptions {
    int32_t ordering = 1;        // 0 = AMD, 1 = auto (nested dissection unless much costlier than AMD), 2 = natural
    double dense_scale = 0.3;    // AMD dense-row threshold multiplier (reference: 1.5; rows above
                                 // 10*scale*sqrt(N) are ordered last, where they end up anyway)
    int32_t nd_leaf = 96;        // ND leaf size
    double nd_max_cost_ratio = 3.0;  // ordering 1: keep ND only if flops <= ratio * AMD flops
    int32_t relax_small = 8;     // always merge a last child when merged width <= this
    double relax_z1 = 0.50;      // allowed zero fraction for merged width <= 32
    double relax_z2 = 0.20;      // ... <= 96
    double relax_z3 = 0.05;      // otherwise
    int32_t max_width = 512;     // never merge beyond this many pivot columns
    int32_t collapse_nf = 32;    // a whole subtree whose merged front (all its columns + the rows below its
                                 // root) has at most this many rows becomes ONE dense supernode (0 = off)
    const int32_t* block_id = nullptr;   // optional [N]: rows sharing an id >= 0 form a dense cone block
                                         // (clique): ordering 1 then eliminates everything else first and
                                         // dissects the block graph (order_blocks_last_nd)
    int32_t min_cone_blocks = 8;         // fewer blocks than this: AMD-class order
    // Size classes of the numeric factorisation (the large-front path pads its panels, so the
    // symbolic layout has to know which fronts take it): panel-in-smem kernel for
    // panel_min_nf < nf <= panel_max_nf (if it fits), shared-memory front kernel up to small_max_nf,
    // large (pivot-block + TMA GEMM) path above.
    int32_t panel_min_nf = 64, panel_max_nf = 152, small_max_nf = 152;
    bool use_panel_kernel = true;
};

// fronts handled by k_factor_panel (panel + scratch in one CTA's shared memory)
inline bool front_to_panel(const SymbolicOptions& o, int nf, int ns) {
    return o.use_panel_kernel && nf > o.panel_min_nf && nf <= o.panel_max_nf && ns <= 150 &&
           ((int64_t)nf * ns + (int64_t)nf * 25) <= 27000;
}
// fronts on the large path: their panels are stored with a padded leading dimension (multiple of
// LD_ALIGN doubles, panel start aligned likewise) so that TMA can address them
inline bool front_is_large(const SymbolicOptions& o, int nf, int ns) {
    return nf > o.small_max_nf && !front_to_panel(o, nf, ns);
}
constexpr int32_t LD_ALIGN = 8;
constexpr int MANY_CHILDREN = 2048;   // large fronts with more children are assembled by k_assemble_atomic

struct Symbolic {
    int64_t N = 0, nnzK = 0;
    std::vector<int32_t> perm;      // perm[k]  = original index of permuted position k
    std::vector<int32_t> iperm;     // iperm[i] = permuted position of original index i
    int32_t nsuper = 0;
    std::vector<int32_t> sn_first;  // [nsuper+1] first permuted column of each supernode
    std::vector<int32_t> sn_of_col; // [N]
    std::vector<int64_t> rows_ptr;  // [nsuper+1] into rows / rel
    std::vector<int32_t> rows;      // below-block row indices R_s (permuted, ascending)
    std::vector<int32_t> rel;       // position of R_s[i] inside the parent's front
    std::vector<int32_t> sn_parent; // [nsuper] assembly-tree parent (-1 = root)
    std::vector<int32_t> child_ptr; // [nsuper+1]
    std::vector<int32_t> child_list;
    std::vector<int64_t> panel_off; // [nsuper+1] doubles; panel s is nf x ns column-major with leading
                                    // dimension panel_ld[s] (= nf, or nf rounded up to LD_ALIGN for large fronts)
    std::vector<int32_t> panel_ld;  // [nsuper]
    std::vector<int64_t> upd_off;   // [nsuper+1] doubles; update block s is nr x nr, ld = nr
    std::vector<int64_t> a_map;     // [nnzK] K nz (original order) -> offset in panel storage
    // Destination-owner form of the extend-add: for front s and front-local index d (column of
    // the front for the factorisation, row of the work vector for the solves) the sources are
    // asm_src[asm_base[s] + asm_colptr[front_ptr[s] + d] ...) ; each source is a global index q
    // into rows/rel (child c = asm_child[.], child-local index j = q - rows_ptr[c]).  Sources of
    // one destination are ordered by child, so sums are deterministic without atomics and a
    // front with thousands of children is assembled in parallel over destinations.
    std::vector<int64_t> front_ptr; // [nsuper+1] prefix sum of (nf+1)
    std::vector<int64_t> asm_base;  // [nsuper+1]
    std::vector<int32_t> asm_colptr;// [front_ptr.back()]
    std::vector<int32_t> asm_src;   // [rows_total minus roots]
    std::vector<int32_t> asm_child; // same length
    // Per-front child lists of the shared-memory front kernel (k_factor_small): kids[child_ptr[s] + q]
    // describes child child_list[child_ptr[s] + q] (its update block at Ust + uoff, nrc x nrc, and its
    // rel at rel + roff).  rel is ascending, so a child adds the lower triangle of its update block to
    // the rows and columns rel[] of the front; adding the children one after the other in this order
    // sums every destination in the order of the destination-owner maps above.
    struct KidEntry { int64_t uoff, roff; int32_t nrc, pad; };
    std::vector<KidEntry> kids;     // [child_list.size()]
    std::vector<int32_t> sn_level;  // [nsuper]
    int32_t nlevels = 0;
    std::vector<int32_t> level_ptr; // [nlevels+1]
    std::vector<int32_t> level_list;// supernodes grouped by level (ascending size inside level)
    int64_t nnzL = 0;               // strictly-lower entries of L incl. amalgamation zeros
    double flops = 0;               // sum over pivot columns of (col length incl. diag)^2
    int64_t upd_total = 0;          // doubles in update storage
    int32_t max_front = 0, max_width = 0;
    int32_t ordering_used = 0;      // 0 = AMD-class, 1 = nested dissection, 2 = natural, 3 = caller's permutation,
                                    // 4 = cone-block dissection (variables first, PSD blocks by ND of the block graph)
    inline int32_t ns(int32_t s) const { return sn_first[s + 1] - sn_first[s]; }
    inline int32_t nr(int32_t s) const { return (int32_t)(rows_ptr[s + 1] - rows_ptr[s]); }
};

// Per-tile source lists of the large-front extend-add.  A child's rel is ascending, so what it adds
// to a T x T tile (rows r0.., columns c0..) of its parent is a rectangle of its update block: child
// columns [ja, jb), and rows [max(ia, j), ib) of column j.  A tile entry names the front (its slot in
// the batch), the tile and its first rectangle; its rectangles end where the next entry's begin (the
// lists end with a sentinel entry).  Rectangles of a tile are in child_list order, so adding them one
// after the other sums every entry in the order of the destination-owner maps.
struct TileEntry { int32_t slot, ti, tj, rect; };
struct TileRect { int32_t child, ja, jb, ia, ib, pad[3]; };
// Appends the tiles of the batch fronts[0..n) to `tiles` / `rects` (slot = position in fronts).
//   schur: every tile (ti >= tj) of columns [ns, nf) of the fronts with nr > 0 - the Schur GEMM's tiles.
//          Only fronts that gather their update block (gather and at most MANY_CHILDREN children)
//          get rectangles, restricted to columns >= ns; the others are updated in place.
//   else:  the tiles of columns [0, ns) (gather) or [0, nf) (pre-assembled fronts) that some child
//          reaches; fronts with more than MANY_CHILDREN children are left to k_assemble_atomic.
// active (multi-GPU, nullptr = all): per-supernode mask of the children whose contributions this
// rank assembles; the other children get no rectangles.
// The caller appends the sentinel {0, 0, 0, rects.size()} after the last batch.
void build_tile_lists(const Symbolic& S, const int32_t* fronts, int32_t n, int32_t T, bool schur,
                      bool gather, const int8_t* active, std::vector<TileEntry>& tiles,
                      std::vector<TileRect>& rects);

// Multi-GPU partition of the assembly tree (SURVEY.md section 8e): an upward-closed "top" set of
// supernodes (root separator fronts) is replicated on every rank; the subtrees hanging below it
// are independent and are assigned whole to ranks (longest-processing-time-first on factor flops).
//   owner[s] in [0, nranks) for subtree supernodes, -1 for top supernodes ; is_top[s] in {0,1}
void partition_subtrees(const Symbolic& S, int32_t nranks, std::vector<int32_t>& owner,
                        std::vector<int8_t>& is_top, std::vector<double>* rank_load = nullptr);

// colptr/rowval: upper-triangular CSC pattern (0-based) of the N x N KKT matrix.
// user_perm (optional, length N): use this ordering instead of computing one.
void symbolic_analyze(int64_t N, const int64_t* colptr, const int64_t* rowval,
                      const SymbolicOptions& opt, const int64_t* user_perm, Symbolic& S);

}  // namespace cb200
