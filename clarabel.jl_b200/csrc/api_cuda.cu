// C-ABI implementation of the device-resident KKT solver (include/clarabel_b200.h).
// Host orchestration only: every numeric operation is a kernel from kernels.cuh.  There is no
// CPU fallback: if CUDA is unavailable every entry point returns a negative status.
#include "../../include/clarabel_b200.h"
#include "symbolic.h"
#include "api_common.h"
#include "kernels.cuh"
#include "kernels_multi.cuh"
#include "kernels_scaling.cuh"

#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <string>
#include <vector>

namespace cb200 {

#define CUDA_OK(call)                                                                     \
    do {                                                                                  \
        cudaError_t _e = (call);                                                          \
        if (_e != cudaSuccess) {                                                          \
            set_error(std::string(#call) + ": " + cudaGetErrorString(_e));                \
            return -100 - (int)_e;                                                        \
        }                                                                                 \
    } while (0)

template <class T> struct DevBuf {
    T* p = nullptr; size_t n = 0;
    // New device buffers are zero-filled: cudaMalloc hands back whatever an earlier owner of the pages left
    // there, and a solver created late in a long-lived process must behave like one in a fresh process.
    // CB200_POISON=1 fills with 0xFF instead (NaN doubles, -1 indices: any read-before-write that matters
    // becomes a loud failure; the GPU suite is run once per round that way), CB200_POISON=2 leaves the
    // memory untouched (for compute-sanitizer --tool initcheck).
    static int fill_mode() {
        static const int m = [] { const char* e = getenv("CB200_POISON"); return e ? atoi(e) : 0; }();
        return m;
    }
    cudaError_t alloc(size_t count, bool fill = true) {
        free(); n = count;
        if (count == 0) return cudaSuccess;
        cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
        if (e != cudaSuccess) return e;
        const int m = fill_mode();
        if (m == 2 || !fill) return cudaSuccess;
        e = cudaMemset(p, m == 1 ? 0xFF : 0, count * sizeof(T));
        if (e != cudaSuccess) return e;
        return cudaDeviceSynchronize();      // the fill runs on the NULL stream, the solver's streams do not wait for it
    }
    cudaError_t upload(const std::vector<T>& v, cudaStream_t st = 0) {
        cudaError_t e = alloc(v.size(), /*fill=*/false);
        if (e != cudaSuccess || v.empty()) return e;
        return cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    void free() { if (p) cudaFree(p); p = nullptr; n = 0; }
    ~DevBuf() { free(); }
};

struct Batch { int32_t off = 0, cnt = 0, maxnf = 0, maxns = 0, maxnr = 0, maxpanel = 0; bool many_children = false;
               bool pre_assembled = false;    // large: some front has more than MANY_CHILDREN children (k_assemble_atomic)
               // large: the batch's slices of the Schur and assembly tile lists (build_tile_lists)
               int32_t schur_off = 0, nschur = 0, asm_off = 0, nasm = 0;
               int32_t src_per_row = 0;
               // big solve class: the 64-blocks of L11 (forward ticket order, then backward) and the 64-row
               // tiles of L21 in d_bigwork, and the tickets + ready flags in d_bigsync (build_plans)
               int32_t work_off = 0, nwork = 0, tile_off = 0, ntile = 0; int64_t sync_off = 0;
               bool all_padded = true;
               std::vector<int32_t> ns_desc;  // large batches are sorted by pivot width (descending): the fronts still
                                              // active at pivot column kb are the first active(kb) of the batch
               int active(int kb) const { int c = 0; while (c < (int)ns_desc.size() && ns_desc[c] > kb) ++c; return c; } };     // every front of the batch is on the padded (TMA-addressable) layout     // max over the fronts of (assembly sources / front rows)      // max over the fronts of the number of update-block tiles per side

constexpr int NSMALL = 6;
static const int kSmallNf[NSMALL] = {16, 32, 64, 96, 128, 152};
constexpr int NPANEL = 4;
static const int kPanelDoubles[NPANEL] = {4096, 9000, 16000, 1 << 30};   // smem need classes (doubles)
constexpr int NSOLVE = 6;      // 0: single-column leaves, 1: warp (16 < ns <= 32), 2: CTA per supernode, 3: multi-CTA (big),
                               // 4: 8 lanes (tiny), 5: warp, ns <= 16 (half the registers, twice the warps in flight)

struct LevelPlan {
    Batch small[NSMALL];
    Batch panel[NPANEL];       // 64 < nf <= 152: panel-in-smem kernel, classes by panel size
    Batch large;
    Batch solve[NSOLVE];
    Batch topf, tops;          // multi-GPU: replicated top fronts of this level (factor / solve)
    int64_t wtotal = 0;        // doubles of W workspace needed by the large batch
};

struct Timers {
    enum { CONE = 0, FACTOR = 1, SOLVE = 2, SPMV = 3, SCHUR = 4, PANEL = 5, SMALL = 6, ASM = 7, NCOARSE = 8 };
    // per-kernel-class segments, recorded only in detail mode 2 (cb200_get_fine_timers)
    enum { F_SMALL0 = 0, F_PANEL0 = 6, F_ZERO = 10, F_ASM = 11, F_DIAG = 12, F_ROWS = 13, F_SCHUR = 14, F_FINISH = 15,
           F_PROLOGUE = 16, F_FWD_LEAF = 17, F_FWD_SUB = 18, F_FWD_WARP = 19, F_FWD_CTA = 20, F_FWD_BIG_ASM = 21,
           F_FWD_BIG_TRI = 22, F_FWD_BIG_GEMV = 23, F_BWD_LEAF = 24, F_BWD_SUB = 25, F_BWD_WARP = 26, F_BWD_CTA = 27,
           F_BWD_BIG_GEMV = 28, F_BWD_BIG_TRI = 29, F_PERMUTE = 30, F_COMM = 31, F_PANELUPD = 32, NFINE = 33 };
    static constexpr int NPH = NCOARSE + NFINE;
    double ms[NPH] = {};
    double nfactor = 0, nsolve = 0, nlaunch = 0;
    std::vector<cudaEvent_t> pool;
    struct Seg { int ph; cudaEvent_t a, b; bool closed; };
    std::vector<Seg> open;
    size_t used = 0;
    cudaEvent_t get() {
        if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); }
        return pool[used++];
    }
    void begin(int ph, cudaStream_t st) { Seg s{ph, get(), get(), false}; cudaEventRecord(s.a, st); open.push_back(s); }
    void end(cudaStream_t st) {        // closes the most recently opened, still open segment (segments nest)
        for (size_t i = open.size(); i-- > 0;) if (!open[i].closed) { cudaEventRecord(open[i].b, st); open[i].closed = true; return; }
    }
    void collect() {      // call after a stream synchronise
        for (auto& s : open) { float t = 0; if (s.closed && cudaEventElapsedTime(&t, s.a, s.b) == cudaSuccess) ms[s.ph] += t; }
        open.clear(); used = 0;
    }
    ~Timers() { for (auto e : pool) cudaEventDestroy(e); }
};

// NCCL is bound at run time (dlsym): the library loads without NCCL for single-GPU use, and under
// torchrun it resolves to the NCCL that torch already loaded.
struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
    bool load() {
        if (ok) return true;
        void* hd = RTLD_DEFAULT;
        auto sym = [&](const char* n) { return dlsym(hd, n); };
        if (!sym("ncclAllReduce")) {
            const char* names[] = {"libnccl.so.2", "libnccl.so"};
            hd = nullptr;
            for (const char* n : names) { hd = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (hd) break; }
            if (!hd) return false;
        }
        GetUniqueId = (decltype(GetUniqueId))sym("ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))sym("ncclCommInitRank");
        AllReduce = (decltype(AllReduce))sym("ncclAllReduce");
        GroupStart = (decltype(GroupStart))sym("ncclGroupStart");
        GroupEnd = (decltype(GroupEnd))sym("ncclGroupEnd");
        CommDestroy = (decltype(CommDestroy))sym("ncclCommDestroy");
        GetErrorString = (decltype(GetErrorString))sym("ncclGetErrorString");
        ok = GetUniqueId && CommInitRank && AllReduce && GroupStart && GroupEnd && CommDestroy;
        return ok;
    }
};
static NcclApi g_nccl;

#define NCCL_OK(call)                                                                      \
    do {                                                                                   \
        ncclResult_t _r = (call);                                                          \
        if (_r != ncclSuccess) {                                                           \
            set_error(std::string(#call) + ": " +                                          \
                      (g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "nccl error")); \
            return -200 - (int)_r;                                                         \
        }                                                                                  \
    } while (0)

struct GraphExec {
    cudaGraphExec_t exec = nullptr;
    double nlaunch = 0;
    bool failed = false;
    ~GraphExec() { if (exec) cudaGraphExecDestroy(exec); }
};

}  // namespace cb200

using namespace cb200;

struct cb200_handle {
    cb200_settings st;
    Symbolic S;
    int64_t N = 0, nnzK = 0, base = 0;
    cudaStream_t stream = nullptr;
    // K (original order, upper CSC) + row-wise index for the symmetric product
    DevBuf<int64_t> d_cp; DevBuf<int32_t> d_ri; DevBuf<double> d_nz;
    DevBuf<int64_t> d_tp; DevBuf<int32_t> d_tc; DevBuf<int64_t> d_tpos;
    DevBuf<int64_t> d_amap, d_diagidx;
    DevBuf<int32_t> d_long_rows; int32_t n_long_rows = 0;
    DevBuf<int8_t> d_dsign_perm, d_dsign_orig;
    DevBuf<int32_t> d_perm;
    // symbolic
    DevBuf<int32_t> d_sn_first, d_rows, d_rel, d_child_ptr, d_child_list, d_batches, d_ld;
    DevBuf<SolveDesc> d_sdesc;          // one packed descriptor per batch entry (same indexing as d_batches)
    DevBuf<int64_t> d_rows_ptr, d_panel_off, d_upd_off, d_woff, d_front_ptr, d_asm_base;
    DevBuf<int32_t> d_asm_colptr, d_asm_src, d_asm_child;
    DevBuf<Symbolic::KidEntry> d_kids;
    // numeric
    DevBuf<double> d_L, d_U, d_W, d_D, d_Dinv, d_uvec, d_partial;
    DevBuf<BigItem> d_bigwork;
    DevBuf<unsigned> d_bigsync;         // [0]: error word of the current solve call, then per big batch: tickets, flags
    DevBuf<double> d_b, d_x, d_e, d_dx, d_y, d_rx, d_rz;
    DevBuf<double> d_eps; DevBuf<unsigned long long> d_scal;   // [0] max|diag|, [1] normb, [2] norme
    DevBuf<unsigned int> d_nreg; DevBuf<int32_t> d_reglog;
    std::vector<LevelPlan> plan;
    std::vector<int32_t> h_batches;
    bool have_diag = false;
    // fused (outer) boundary state
    bool maps_set = false;
    int64_t n = 0, m = 0, p = 0;
    DevBuf<int64_t> d_mapP, d_mapA;
    // diagonal Hs entries
    int64_t ndiag = 0;
    DevBuf<int8_t> d_dg_kind; DevBuf<int32_t> d_dg_midx, d_dg_cone; DevBuf<int64_t> d_dg_map;
    // dense SOC
    int32_t nsocd = 0;
    DevBuf<int32_t> d_sd_moff, d_sd_dim, d_sd_socid; DevBuf<int64_t> d_sd_hoff;
    DevBuf<int64_t> d_mapHs;
    // sparse SOC expansion
    int64_t nexp = 0; int32_t nsocs = 0;
    DevBuf<int32_t> d_ex_src, d_ex_cone, d_exD_cone; DevBuf<int64_t> d_mapu, d_mapv, d_mapD;
    // PSD
    int32_t npsd = 0, psd_maxn = 0;
    DevBuf<int32_t> d_psd_side; DevBuf<int64_t> d_psd_roff, d_psd_hoff;
    DevBuf<double> d_psd_R, d_psd_A;
    int64_t psd_rtotal = 0;
    // cone state
    int64_t nsoc = 0, nsocrows = 0;
    DevBuf<double> d_w, d_eta, d_socd, d_socu, d_socv;
    double last_eps = 0;
    bool resident = false;
    int detail = 0;            // 1: per-phase event timing, 2: also per kernel class (both disable graph replay)
    // size-class boundaries of the factorisation plan (tuning knobs, environment variables
    // CB200_PANEL_MIN_NF / CB200_PANEL_MAX_NF / CB200_SMALL_MAX_NF / CB200_NO_PANEL, read once into the
    // symbolic options because the large path pads its panels): panel kernel for
    // panel_min_nf < nf <= panel_max_nf, shared-memory front kernel up to small_max_nf, pivot-block
    // (large) path above
    SymbolicOptions opt;
    bool to_panel(int nf, int ns) const { return front_to_panel(opt, nf, ns); }
    bool to_large(int nf, int ns) const { return front_is_large(opt, nf, ns); }
    // TMA descriptors of the large-front panels (one CUtensorMap per large front)
    bool use_tma = false; int tma_kmajor = 1;
    int reduce_blocks = 1;            // grid cap of the grid-stride max-reductions: 8 CTAs per SM of the device
    int tma_tile = 64;                // CTA tile of the TMA GEMM: 64 (3 CTAs per SM, 64 KB of shared memory each; the
                                      // fastest on the H100, DESIGN.md section 4), 128 (1 CTA per SM, spills on sm_90a),
                                      // or 0 = by front size (CB200_TMA_TILE)
    DevBuf<CUtensorMap> d_tmaps, d_tmaps64; DevBuf<int32_t> d_tmap_of;
    // per-tile source lists of the large fronts, all batches (build_tile_lists)
    DevBuf<TileEntry> d_schur_tiles, d_asm_tiles; DevBuf<TileRect> d_schur_rects, d_asm_rects;
    int64_t n_schur_tiles = 0, n_schur_rects = 0, n_asm_tiles = 0, n_asm_rects = 0;
    // multi-GPU state
    bool dist = false; int rank = 0, nranks = 1;
    ncclComm_t comm = nullptr;
    std::vector<int32_t> owner; std::vector<int8_t> is_top;
    std::vector<int8_t> h_active;       // host copy of d_active (DevSym::active)
    std::vector<int32_t> h_top_list;
    std::vector<std::vector<int32_t>> h_top_by_level;
    DevBuf<int8_t> d_active, d_keepcol, d_topcolkeep;
    DevBuf<int32_t> d_top_list;
    GraphExec g_factor[2], g_solve;     // CUDA graphs: factor (without/with static reg), solve sweeps
    // Fork/join streams: the kernel classes of one tree level are independent of each other (small
    // fronts vs the pivot-block chain of the large fronts; leaf / warp / CTA / big solve classes),
    // most of them are latency-bound and leave SMs idle, so they run as parallel branches (captured
    // as such into the CUDA graphs).  CB200_MULTISTREAM=0 serialises them again.
    cudaStream_t side[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[3] = {nullptr, nullptr, nullptr};
    bool multi_stream = true;
    bool sort_batches = true;          // CB200_SORT_BATCHES=0: keep the size order of the level lists
    bool merged_rows = true;           // 16-column warp solve kernels fetch the triangle and the first L21 chunk in ONE batch
                                       // of loads (one dependent round trip less; 80 registers, 3 CTAs/SM).
                                       // CB200_MERGED_ROWS=0: two-phase loads.
    // bottom subtrees of narrow supernodes solved by one CTA each (k_fwd_subtree / k_bwd_subtree)
    bool use_subtree = false;          // CB200_SUBTREE=1 turns them on.  Slower than the level-scheduled kernels
                                       // - with only L streamed from HBM but metadata still fetched per
                                       // supernode, 16 warps per SM are too few to hide the dependent round trips.  Kept as
                                       // the base of a version that bulk-prefetches the (contiguous) subtree panels.
    int32_t nsub = 0, sub_nlev = 0, sub_maxcols = 0, sub_maxrows = 0;
    DevBuf<int32_t> d_sub_sn0, d_sub_sn1, d_sub_order, d_sub_lvl;
    DevBuf<int64_t> d_sub_optr;
    bool ms_on() const { return multi_stream && detail == 0; }
    void fork(int n) {            // side[0..n) start after everything issued so far on `stream`
        cudaEventRecord(ev_fork, stream);
        for (int i = 0; i < n; ++i) cudaStreamWaitEvent(side[i], ev_fork, 0);
    }
    void join(int n) {            // `stream` continues after side[0..n)
        for (int i = 0; i < n; ++i) { cudaEventRecord(ev_join[i], side[i]); cudaStreamWaitEvent(stream, ev_join[i], 0); }
    }
    // grow-only device staging for the inner-boundary uploads (update_values!/scale_values!/update_P/A):
    // no cudaMalloc / cudaFree per call and no stream sync for pageable caller buffers
    DevBuf<int64_t> d_stage_idx; DevBuf<double> d_stage_val;
    size_t stage_idx_cap = 0, stage_val_cap = 0;
    Timers tm;
    // multi-right-hand-side state (cb200_solve_multi / cb200_solve_ir_multi): grow-only, allocated by the first
    // multi call, so a caller that never uses those entry points pays no memory
    int multi_w = 0;                                // widest sweep (1, 2 or 4; shared memory can cap it), 0: not allocated
    DevBuf<double> d_my, d_muvec, d_mpartial;       // interleaved sweep vectors (R > 1; R = 1 uses d_y, d_uvec, d_partial)
    DevBuf<double> d_mb, d_mx, d_mdx, d_me;         // interleaved refinement vectors, N x multi_w
    DevBuf<double> d_mstage, d_mrx, d_mrz;          // column-major staging of one chunk of the caller's columns
    DevBuf<double> d_msol; int64_t msol_cols = 0;   // solutions of the last cb200_solve_ir_multi (download selector 8)
    DevBuf<unsigned long long> d_mscal;             // [0, 4): ||b_r||_inf, [4, 8): ||e_r||_inf (bits)
    GraphExec g_msolve[2];                          // sweep graphs of width 2 and 4 (width 1 is g_solve)
    int64_t partial_len = 1;                        // doubles of d_partial (one column)
    double n_multi_sweeps = 0, n_percol = 0;        // cb200_get_stats 21 / 22
    // device NT scaling (cb200_update_scaling, G10): tables and outputs built by the first call
    std::vector<int32_t> h_ctype; std::vector<int64_t> h_cdim;      // the cone table of cb200_set_maps
    bool scale_ready = false;
    int64_t nnn = 0, psd_ltotal = 0;
    int32_t nsoc_warp = 0, nsoc_cta = 0, npsd_smem = 0, npsd_glob = 0;
    size_t psd_smem_bytes = 0;                                      // dynamic shared memory of k_scale_psd<true>
    DevBuf<int32_t> d_nn_rows;                                      // m-space rows of the NN cones
    DevBuf<int32_t> d_soc_list, d_soc_dim; DevBuf<int64_t> d_soc_moff, d_soc_srow;   // list: warp class, then CTA class
    DevBuf<int32_t> d_psd_list; DevBuf<int64_t> d_psd_moff, d_psd_loff, d_psd_woff;  // list: shared-memory, then global
    DevBuf<double> d_lam, d_psd_Rinv, d_psd_lam, d_psd_ws, d_ss, d_sz;
    DevBuf<int> d_scale_flags;                                      // [0] failure, [1] max Jacobi sweeps
    cudaEvent_t ev_scale[2] = {nullptr, nullptr};
    double scale_ms = 0, last_sweeps = 0;                           // cb200_get_timers 11, cb200_get_stats 25
};

namespace {

DevSym devsym(cb200_handle* h) {
    DevSym d;
    d.sn_first = h->d_sn_first.p; d.rows_ptr = h->d_rows_ptr.p; d.rows = h->d_rows.p; d.rel = h->d_rel.p;
    d.child_ptr = h->d_child_ptr.p; d.child_list = h->d_child_list.p;
    d.panel_off = h->d_panel_off.p; d.upd_off = h->d_upd_off.p; d.dsign = h->d_dsign_perm.p; d.ld = h->d_ld.p;
    d.front_ptr = h->d_front_ptr.p; d.asm_base = h->d_asm_base.p; d.asm_colptr = h->d_asm_colptr.p;
    d.asm_src = h->d_asm_src.p; d.asm_child = h->d_asm_child.p; d.kids = h->d_kids.p;
    d.active = h->dist ? h->d_active.p : nullptr;
    return d;
}

inline int nblk(int64_t n, int t) { return (int)((n + t - 1) / t); }

#define LAUNCH(h) ((h)->tm.nlaunch += 1)

// times the launches issued while it is alive under one kernel class (detail mode 2 only)
struct FineScope {
    cb200_handle* h; bool on;
    FineScope(cb200_handle* h_, int cls) : h(h_), on(h_->detail >= 2) { if (on) h->tm.begin(Timers::NCOARSE + cls, h->stream); }
    ~FineScope() { if (on) h->tm.end(h->stream); }
};

// G threads per front, FPC fronts per CTA, each with an nf x nf front in shared memory
template <int G, int FPC>
int launch_small(cb200_handle* h, const Batch& b, int cls, RegParams rp, cudaStream_t st) {
    if (b.cnt == 0) return 0;
    FineScope fs(h, Timers::F_SMALL0 + cls);
    const int fstride = b.maxnf * b.maxnf;
    const size_t sm = (size_t)FPC * fstride * sizeof(double);
    k_factor_small<G, FPC><<<nblk(b.cnt, FPC), G * FPC, sm, st>>>(devsym(h), h->d_batches.p + b.off, b.cnt, fstride,
                                                                  h->d_L.p, h->d_U.p, h->d_D.p, h->d_Dinv.p, rp, h->d_nreg.p);
    LAUNCH(h);
    return 0;
}

// The work vectors of one sweep: R = 1 the single-column buffers, R > 1 the interleaved multi-RHS ones
struct SweepBufs { double* y; double* uvec; double* partial; };
// the single-column kernel for R = 1, its R-wide form (kernels_multi.cuh) otherwise; both take the same arguments
#define PICK(R, single, multi) ([] { if constexpr (R == 1) return single; else return multi; }())

template <int R>
void launch_fwd_level(cb200_handle* h, const LevelPlan& P, int lv, const SweepBufs& V) {
    DevSym ds = devsym(h);
    // classes of a level are independent: leaf + tiny on side[0], warp on side[1], CTA on side[2], big on the
    // main stream (fork/join only when a second class has work)
    const bool big_work = P.solve[3].cnt || P.tops.cnt;
    const int nclass = (P.solve[0].cnt || P.solve[4].cnt) + (P.solve[1].cnt != 0 || P.solve[5].cnt != 0) + (P.solve[2].cnt != 0) + big_work;
    const bool ms = h->ms_on() && nclass > 1;
    cudaStream_t s_leaf = ms ? h->side[0] : h->stream, s_warp = ms ? h->side[1] : h->stream,
                 s_cta = ms ? h->side[2] : h->stream;
    if (ms) h->fork(3);
    const Batch& b0 = P.solve[0];
    if (b0.cnt) {
        { FineScope fs(h, Timers::F_FWD_LEAF);
        PICK(R, k_fwd_leaf, k_fwd_leaf_multi<R>)<<<nblk(b0.cnt, 128), 128, 0, s_leaf>>>(ds, h->d_batches.p + b0.off, b0.cnt, h->d_L.p,
                                                             V.y, V.uvec);
        LAUNCH(h);
        }
    }
    const Batch& b1 = P.solve[1];
    if (b1.cnt) {
        FineScope fs(h, Timers::F_FWD_WARP);
        PICK(R, (k_fwd_warp<32, false>), (k_fwd_warp_multi<32, R>))<<<nblk(b1.cnt, WPB), WPB * 32, fwd_warp_smem(b1.maxnf, R), s_warp>>>(
            ds, h->d_sdesc.p + b1.off, b1.cnt, b1.maxnf, h->d_L.p, V.y, V.uvec);
        LAUNCH(h);
    }
    const Batch& b5 = P.solve[5];
    if (b5.cnt) {
        FineScope fs(h, Timers::F_FWD_WARP);
        auto k = R > 1 ? PICK(R, (k_fwd_warp<16, true>), (k_fwd_warp_multi<16, R>))
                       : h->merged_rows ? k_fwd_warp<16, true> : k_fwd_warp<16, false>;
        k<<<nblk(b5.cnt, WPB), WPB * 32, fwd_warp_smem(b5.maxnf, R), s_warp>>>(
            ds, h->d_sdesc.p + b5.off, b5.cnt, b5.maxnf, h->d_L.p, V.y, V.uvec);
        LAUNCH(h);
    }
    const Batch& b2 = P.solve[2];
    if (b2.cnt) {
        { FineScope fs(h, Timers::F_FWD_CTA);
        PICK(R, k_fwd_cta, k_fwd_cta_multi<R>)<<<b2.cnt, 256, (size_t)b2.maxnf * R * sizeof(double), s_cta>>>(
            ds, h->d_sdesc.p + b2.off, h->d_L.p, V.y, V.uvec);
        LAUNCH(h);
        }
    }
    for (int pass = 0; pass < 2; ++pass) {
        const Batch& b3 = pass == 0 ? P.solve[3] : P.tops;
        if (!b3.cnt) continue;
        const int32_t* bl = h->d_batches.p + b3.off;
        { FineScope fs(h, Timers::F_FWD_BIG_ASM);
        if (b3.src_per_row >= 512)
            PICK(R, k_big_asm_fwd<256>, (k_big_asm_fwd_multi<256, R>))<<<dim3(b3.maxnf, b3.cnt), 256, 0, h->stream>>>(ds, bl, V.y, V.uvec);
        else if (b3.many_children)
            PICK(R, k_big_asm_fwd<32>, (k_big_asm_fwd_multi<32, R>))<<<dim3(nblk((int64_t)b3.maxnf * 32, 256), b3.cnt), 256, 0, h->stream>>>(ds, bl, V.y, V.uvec);
        else
            PICK(R, k_big_asm_fwd<1>, (k_big_asm_fwd_multi<1, R>))<<<dim3(nblk(b3.maxnf, 256), b3.cnt), 256, 0, h->stream>>>(ds, bl, V.y, V.uvec);
        LAUNCH(h);
        }
        if (pass == 1 && h->dist) {
            // sum the per-rank partial right-hand sides of the replicated top fronts
            FineScope fs(h, Timers::F_COMM);
            const Symbolic& S = h->S;
            g_nccl.GroupStart();
            for (int32_t sn : h->h_top_by_level[lv]) {
                double* yt = V.y + (int64_t)S.sn_first[sn] * R;
                g_nccl.AllReduce(yt, yt, (size_t)S.ns(sn) * R, ncclDouble, ncclSum, h->comm, h->stream);
                if (S.nr(sn) > 0) {
                    double* ut = V.uvec + S.rows_ptr[sn] * R;
                    g_nccl.AllReduce(ut, ut, (size_t)S.nr(sn) * R, ncclDouble, ncclSum, h->comm, h->stream);
                }
            }
            g_nccl.GroupEnd();
        }
        {
            FineScope fs(h, Timers::F_FWD_BIG_TRI);
            unsigned* sy = h->d_bigsync.p + b3.sync_off;
            PICK(R, k_big_tri_fwd, k_big_tri_fwd_multi<R>)<<<b3.nwork, 256, 0, h->stream>>>(ds, h->d_bigwork.p + b3.work_off, sy, sy + 2, h->d_bigsync.p,
                                                            h->d_L.p, V.y);
            LAUNCH(h);
        }
        if (b3.ntile) {
            FineScope fs(h, Timers::F_FWD_BIG_GEMV);
            PICK(R, k_big_gemv_fwd, k_big_gemv_fwd_multi<R>)<<<b3.ntile, 256, 0, h->stream>>>(ds, h->d_bigwork.p + b3.tile_off, h->d_L.p, V.y, V.uvec);
            LAUNCH(h);
        }
    }
    if (ms) h->join(3);
}
template <int R>
void launch_bwd_level(cb200_handle* h, const LevelPlan& P, const SweepBufs& V) {
    DevSym ds = devsym(h);
    const bool big_work = P.solve[3].cnt || P.tops.cnt;
    const int nclass = (P.solve[0].cnt || P.solve[4].cnt) + (P.solve[1].cnt != 0 || P.solve[5].cnt != 0) + (P.solve[2].cnt != 0) + big_work;
    const bool ms = h->ms_on() && nclass > 1;
    cudaStream_t s_leaf = ms ? h->side[0] : h->stream, s_warp = ms ? h->side[1] : h->stream,
                 s_cta = ms ? h->side[2] : h->stream;
    if (ms) h->fork(3);
    for (int pass = 0; pass < 2; ++pass) {
        const Batch& b3 = pass == 0 ? P.tops : P.solve[3];
        if (!b3.cnt) continue;
        if (b3.ntile) {
            FineScope fs(h, Timers::F_BWD_BIG_GEMV);
            PICK(R, k_big_gemvT_bwd, k_big_gemvT_bwd_multi<R>)<<<b3.ntile, 256, 0, h->stream>>>(ds, h->d_bigwork.p + b3.tile_off, h->d_L.p, V.y,
                                                              V.partial);
            LAUNCH(h);
        }
        FineScope fs(h, Timers::F_BWD_BIG_TRI);
        unsigned* sy = h->d_bigsync.p + b3.sync_off;
        PICK(R, k_big_tri_bwd, k_big_tri_bwd_multi<R>)<<<b3.nwork, 256, 0, h->stream>>>(ds, h->d_bigwork.p + b3.work_off + b3.nwork, sy + 1,
                                                        sy + 2 + b3.nwork, h->d_bigsync.p, h->d_L.p, h->d_Dinv.p,
                                                        V.partial, V.y);
        LAUNCH(h);
    }
    const Batch& b2 = P.solve[2];
    if (b2.cnt) {
        { FineScope fs(h, Timers::F_BWD_CTA);
        PICK(R, k_bwd_cta, k_bwd_cta_multi<R>)<<<b2.cnt, 256, R == 1 ? (size_t)b2.maxnf * sizeof(double) : bwd_cta_smem(b2.maxnf, R), s_cta>>>(
            ds, h->d_batches.p + b2.off, h->d_L.p, h->d_Dinv.p, V.y);
        LAUNCH(h);
        }
    }
    const Batch& b1 = P.solve[1];
    if (b1.cnt) {
        FineScope fs(h, Timers::F_BWD_WARP);
        PICK(R, (k_bwd_warp<32, false>), (k_bwd_warp_multi<32, R>))<<<nblk(b1.cnt, WPB), WPB * 32, bwd_warp_smem(b1.maxnf, 32, R), s_warp>>>(
            ds, h->d_sdesc.p + b1.off, b1.cnt, b1.maxnf, h->d_L.p, h->d_Dinv.p, V.y);
        LAUNCH(h);
    }
    const Batch& b5 = P.solve[5];
    if (b5.cnt) {
        FineScope fs(h, Timers::F_BWD_WARP);
        auto k = R > 1 ? PICK(R, (k_bwd_warp<16, true>), (k_bwd_warp_multi<16, R>))
                       : h->merged_rows ? k_bwd_warp<16, true> : k_bwd_warp<16, false>;
        k<<<nblk(b5.cnt, WPB), WPB * 32, bwd_warp_smem(b5.maxnf, 16, R), s_warp>>>(
            ds, h->d_sdesc.p + b5.off, b5.cnt, b5.maxnf, h->d_L.p, h->d_Dinv.p, V.y);
        LAUNCH(h);
    }
    const Batch& b0 = P.solve[0];
    if (b0.cnt) {
        { FineScope fs(h, Timers::F_BWD_LEAF);
        PICK(R, k_bwd_leaf, k_bwd_leaf_multi<R>)<<<nblk(b0.cnt, 128), 128, 0, s_leaf>>>(ds, h->d_batches.p + b0.off, b0.cnt, h->d_L.p,
                                                             h->d_Dinv.p, V.y);
        LAUNCH(h);
        }
    }
    if (ms) h->join(3);
}


// One CUtensorMap per large front: the nf x ns panel (leading dimension ld, a multiple of 8) viewed
// as a 3-D tensor so that one TMA box is a 128-row x 16-k operand tile in a DMMA-friendly layout
// (see k_ldl_update_tma).  The encoder lives in libcuda; it is fetched through the runtime
// (cudaGetDriverEntryPoint) so that the library has no link-time dependency on the driver.
// CB200_NO_TMA=1 selects the LDG fallback kernel.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
int build_tensor_maps(cb200_handle* h) {
    const Symbolic& S = h->S;
    h->use_tma = false;
    if (const char* e = getenv("CB200_NO_TMA")) if (e[0] == '1') return 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || !fn) { cudaGetLastError(); return 0; }
    EncodeTiledFn encode = (EncodeTiledFn)fn;
    if (const char* e = getenv("CB200_TMA_TILE")) h->tma_tile = atoi(e);
    std::vector<int32_t> map_of(S.nsuper, -1);
    std::vector<CUtensorMap> maps, maps64;
    int kmajor = 1;
    if (const char* e = getenv("CB200_TMA_NATURAL")) if (e[0] == '1') kmajor = 0;
    for (int attempt = 0; attempt < 2; ++attempt) {
        maps.clear(); maps64.clear(); std::fill(map_of.begin(), map_of.end(), -1);
        bool ok = true;
        for (int32_t sn = 0; sn < S.nsuper && ok; ++sn) {
            const int ns = S.ns(sn), nf = ns + S.nr(sn);
            if (!h->to_large(nf, ns)) continue;
            const cuuint64_t ld = (cuuint64_t)S.panel_ld[sn];
            CUtensorMap m;
            cuuint64_t dims[3], strides[2]; cuuint32_t box[3], estr[3] = {1, 1, 1};
            if (kmajor) { dims[0] = 8; dims[1] = (cuuint64_t)ns; dims[2] = ld / 8; strides[0] = ld * 8; strides[1] = 64;
                          box[0] = 8; box[1] = TK; box[2] = TB / 8; }
            else        { dims[0] = 8; dims[1] = ld / 8; dims[2] = (cuuint64_t)ns; strides[0] = 64; strides[1] = ld * 8;
                          box[0] = 8; box[1] = TB / 8; box[2] = TK; }
            CUresult r = encode(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)(h->d_L.p + S.panel_off[sn]), dims, strides,
                                box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { ok = false; break; }
            CUtensorMap m64;                              // same view, box of 64 rows for the small tile
            if (kmajor) box[2] = 64 / 8; else box[1] = 64 / 8;
            r = encode(&m64, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)(h->d_L.p + S.panel_off[sn]), dims, strides,
                       box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { ok = false; break; }
            map_of[sn] = (int32_t)maps.size(); maps.push_back(m); maps64.push_back(m64);
        }
        if (ok) { h->use_tma = true; h->tma_kmajor = kmajor; break; }
        if (kmajor == 0) break;
        kmajor = 0;                              // retry with the natural dimension order
    }
    if (!h->use_tma) return 0;
    if (maps.empty()) { maps.resize(1); maps64.resize(1); }
    CUDA_OK(h->d_tmaps.alloc(maps.size())); CUDA_OK(h->d_tmaps64.alloc(maps64.size()));
    CUDA_OK(cudaMemcpyAsync(h->d_tmaps.p, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, h->stream));
    CUDA_OK(cudaMemcpyAsync(h->d_tmaps64.p, maps64.data(), maps64.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, h->stream));
    CUDA_OK(h->d_tmap_of.upload(map_of, h->stream));
    CUDA_OK(cudaStreamSynchronize(h->stream));
    return 0;
}

// Builds the per-level launch plans.  In multi-GPU mode a rank only schedules the supernodes it
// owns plus the replicated top fronts (which always take the large-front / big-solve paths so
// that assembly, all-reduce and factorisation are separate steps).
int build_plans(cb200_handle* h) {
    const Symbolic& S = h->S;
    cudaStream_t s = h->stream;
    h->plan.assign(S.nlevels, LevelPlan());
    std::vector<int32_t> batches; std::vector<int64_t> woff;
    int64_t wmax = 0;
    auto add_batch = [&](Batch& b, std::vector<int32_t> v, bool large, LevelPlan& P) {
        b = Batch();
        if (large) {
            std::stable_sort(v.begin(), v.end(), [&](int32_t x, int32_t y) { return S.ns(x) > S.ns(y); });
            for (int32_t sn : v) b.ns_desc.push_back(S.ns(sn));
        } else if (h->sort_batches) {
            // memory order: panels, update blocks and solution slices of consecutive supernodes are
            // adjacent in HBM (postorder layout), so neighbouring warps / CTAs touch neighbouring DRAM
            // pages instead of random ones (the level lists come sorted by front size)
            std::sort(v.begin(), v.end());
        }
        b.off = (int32_t)batches.size(); b.cnt = (int32_t)v.size();
        int64_t w = 0;
        for (int32_t sn : v) {
            int nf = S.ns(sn) + S.nr(sn);
            b.maxnf = std::max(b.maxnf, nf); b.maxns = std::max(b.maxns, S.ns(sn));
            b.maxnr = std::max(b.maxnr, S.nr(sn));
            b.maxpanel = std::max(b.maxpanel, nf * S.ns(sn) + 25 * nf);      // smem need of k_factor_panel
            if (S.child_ptr[sn + 1] - S.child_ptr[sn] > 64) b.many_children = true;
            if (S.child_ptr[sn + 1] - S.child_ptr[sn] > MANY_CHILDREN) b.pre_assembled = true;
            b.src_per_row = std::max<int32_t>(b.src_per_row, (int32_t)((S.asm_base[sn + 1] - S.asm_base[sn]) / std::max(1, nf)));
            if (large && !h->to_large(nf, S.ns(sn))) b.all_padded = false;   // multi-GPU: small top fronts on the large path
            batches.push_back(sn);
            woff.push_back(large ? w : 0);
            if (large) w += (int64_t)nblk(S.ns(sn), PB) * PB * PB;   // parked diagonal blocks
        }
        if (large) { P.wtotal += w; wmax = std::max(wmax, w); }
    };
    // ---- bottom subtrees for the solves: complete subtrees whose supernodes are all narrow (ns <= 32,
    // nf <= SUB_MAXNF) and whose columns / contribution rows fit a shared-memory window
    std::vector<int8_t> in_sub(S.nsuper, 0);
    h->nsub = 0;
    if (h->use_subtree && S.nsuper > 0) {
        constexpr int64_t MAXCOLS = 2048, MAXROWS = 6144, MAXPANEL = 131072;
        constexpr int32_t MINSN = 16;
        const int32_t n = S.nsuper;
        std::vector<int8_t> ok(n, 1);
        std::vector<int64_t> wc(n), wr(n), wp(n); std::vector<int32_t> cnt(n, 1);
        for (int32_t sn = 0; sn < n; ++sn) {            // children precede parents
            const int64_t ns = S.ns(sn), nr = S.nr(sn);
            wc[sn] += ns; wr[sn] += nr; wp[sn] += (ns + nr) * ns;
            bool self = ns <= 32 && ns + nr <= SUB_MAXNF;
            if (h->dist) self = self && !h->is_top[sn] && h->owner[sn] == h->rank;
            if (!self || wc[sn] > MAXCOLS || wr[sn] > MAXROWS || wp[sn] > MAXPANEL) ok[sn] = 0;
            const int32_t p = S.sn_parent[sn];
            if (p >= 0) { wc[p] += wc[sn]; wr[p] += wr[sn]; wp[p] += wp[sn]; cnt[p] += cnt[sn]; if (!ok[sn]) ok[p] = 0; }
        }
        std::vector<int32_t> sn0, sn1, order, lvl; std::vector<int64_t> optr(1, 0);
        int32_t maxl = 0;
        std::vector<int32_t> roots;
        for (int32_t sn = 0; sn < n; ++sn) {
            const int32_t p = S.sn_parent[sn];
            if (ok[sn] && (p < 0 || !ok[p]) && cnt[sn] >= MINSN) { roots.push_back(sn); maxl = std::max(maxl, S.sn_level[sn] + 1); }
        }
        h->sub_nlev = maxl; h->sub_maxcols = 1; h->sub_maxrows = 1;
        for (int32_t r : roots) {
            const int32_t a = r - cnt[r] + 1;
            sn0.push_back(a); sn1.push_back(r);
            h->sub_maxcols = std::max<int32_t>(h->sub_maxcols, (int32_t)wc[r]);
            h->sub_maxrows = std::max<int32_t>(h->sub_maxrows, (int32_t)wr[r]);
            std::vector<int32_t> off(maxl + 1, 0);
            for (int32_t q = a; q <= r; ++q) { in_sub[q] = 1; off[S.sn_level[q] + 1]++; }
            for (int32_t l = 0; l < maxl; ++l) off[l + 1] += off[l];
            const size_t base = order.size();
            order.resize(base + (size_t)cnt[r]);
            { std::vector<int32_t> pos(off.begin(), off.end() - 1);
              for (int32_t q = a; q <= r; ++q) order[base + pos[S.sn_level[q]]++] = q; }
            lvl.insert(lvl.end(), off.begin(), off.end());
            optr.push_back((int64_t)order.size());
        }
        h->nsub = (int32_t)roots.size();
        if (h->nsub) {
            CUDA_OK(h->d_sub_sn0.upload(sn0, s)); CUDA_OK(h->d_sub_sn1.upload(sn1, s));
            CUDA_OK(h->d_sub_order.upload(order, s)); CUDA_OK(h->d_sub_lvl.upload(lvl, s));
            CUDA_OK(h->d_sub_optr.upload(optr, s));
        }
    }
    for (int lv = 0; lv < S.nlevels; ++lv) {
        std::vector<int32_t> cls[NSMALL + 1], scl[NSOLVE], pcl[NPANEL], top;
        for (int32_t q = S.level_ptr[lv]; q < S.level_ptr[lv + 1]; ++q) {
            int32_t sn = S.level_list[q];
            if (h->dist) {
                if (h->is_top[sn]) { top.push_back(sn); continue; }
                if (h->owner[sn] != h->rank) continue;
            }
            int nf = S.ns(sn) + S.nr(sn);
            int c = 0; while (c < NSMALL && nf > kSmallNf[c]) ++c;
            if (h->to_large(nf, S.ns(sn)) || nf > kSmallNf[NSMALL - 1]) c = NSMALL;
            if (h->to_panel(nf, S.ns(sn))) {
                int pc = 0; while (nf * S.ns(sn) + 25 * nf > kPanelDoubles[pc]) ++pc;
                pcl[pc].push_back(sn);
            } else cls[c].push_back(sn);
            const bool leaf = (S.ns(sn) == 1 && S.child_ptr[sn + 1] == S.child_ptr[sn]);
            const bool big = (int64_t)nf * S.ns(sn) >= 65536 && S.ns(sn) > 32;
            // (the 8-lane kernels for tiny supernodes are gone: the 16-column warp kernel takes them)
            static const bool warp16 = !(getenv("CB200_WARP16") && getenv("CB200_WARP16")[0] == '0');    // debugging aid
            const int d = leaf ? 0 : ((S.ns(sn) <= 32 && nf <= 192) ? (S.ns(sn) <= 16 && warp16 ? 5 : 1) : (big ? 3 : 2));
            if (!in_sub[sn]) scl[d].push_back(sn);
        }
        LevelPlan& P = h->plan[lv];
        P.wtotal = 0;
        for (int c = 0; c < NSMALL; ++c) add_batch(P.small[c], cls[c], false, P);
        for (int c = 0; c < NPANEL; ++c) add_batch(P.panel[c], pcl[c], false, P);
        add_batch(P.large, cls[NSMALL], true, P);
        for (int d = 0; d < NSOLVE; ++d) add_batch(P.solve[d], scl[d], false, P);
        add_batch(P.topf, top, true, P);
        add_batch(P.tops, top, false, P);
    }
    h->h_batches = batches;
    CUDA_OK(h->d_batches.upload(batches, s)); CUDA_OK(h->d_woff.upload(woff, s));
    {
        std::vector<SolveDesc> sd(batches.size());
        for (size_t i = 0; i < batches.size(); ++i) {
            const int32_t sn = batches[i];
            SolveDesc& d = sd[i];
            d.f = S.sn_first[sn]; d.ns = S.ns(sn); d.nr = S.nr(sn); d.ld = S.panel_ld[sn];
            d.nchild = S.child_ptr[sn + 1] - S.child_ptr[sn]; d.pad = 0; d.pad2 = 0;
            d.panel_off = S.panel_off[sn]; d.rows_ptr = S.rows_ptr[sn]; d.front_ptr = S.front_ptr[sn]; d.asm_base = S.asm_base[sn];
        }
        CUDA_OK(h->d_sdesc.alloc(std::max<size_t>(1, sd.size())));
        if (!sd.empty()) CUDA_OK(cudaMemcpyAsync(h->d_sdesc.p, sd.data(), sd.size() * sizeof(SolveDesc), cudaMemcpyHostToDevice, s));
        CUDA_OK(cudaStreamSynchronize(s));
    }
    CUDA_OK(h->d_W.alloc((size_t)std::max<int64_t>(1, wmax)));
    // big-solve work lists, per batch: the 64-blocks of L11 block-major across the fronts, ascending
    // (forward) then descending (backward) - every block of a front is ticketed before the blocks that
    // wait on it - then the 64-row tiles of L21.  d_bigsync per batch: forward ticket, backward ticket,
    // forward flags, backward flags (one per block).
    std::vector<BigItem> work;
    int64_t nsync = 1, pmax = 1;
    for (LevelPlan& P : h->plan)
        for (Batch* b3 : {&P.solve[3], &P.tops}) {
            if (!b3->cnt) continue;
            std::vector<int32_t> nbk(b3->cnt), fbase(b3->cnt);
            std::vector<int64_t> pbase(b3->cnt);
            int32_t nflag = 0, maxnb = 0;
            int64_t psz = 0;
            for (int32_t k = 0; k < b3->cnt; ++k) {
                const int32_t sn = batches[b3->off + k];
                nbk[k] = nblk(S.ns(sn), SB); fbase[k] = nflag; nflag += nbk[k]; maxnb = std::max(maxnb, nbk[k]);
                pbase[k] = psz; psz += (int64_t)nblk(S.nr(sn), BRT) * S.ns(sn);
            }
            if (psz > std::numeric_limits<int32_t>::max()) { set_error("build_plans: big-solve partial sums exceed 2^31"); return -3; }
            b3->sync_off = nsync; nsync += 2 + 2 * (int64_t)nflag;
            b3->work_off = (int32_t)work.size(); b3->nwork = nflag;
            for (int dir = 0; dir < 2; ++dir)
                for (int32_t m = 0; m < maxnb; ++m)
                    for (int32_t k = 0; k < b3->cnt; ++k)
                        if (m < nbk[k]) work.push_back({batches[b3->off + k], dir == 0 ? m : nbk[k] - 1 - m, fbase[k], (int32_t)pbase[k]});
            b3->tile_off = (int32_t)work.size();
            for (int32_t k = 0; k < b3->cnt; ++k) {
                const int32_t sn = batches[b3->off + k];
                for (int32_t t = 0; t * BRT < S.nr(sn); ++t)
                    work.push_back({sn, S.ns(sn) + t * BRT, 0, (int32_t)(pbase[k] + (int64_t)t * S.ns(sn))});
            }
            b3->ntile = (int32_t)work.size() - b3->tile_off;
            pmax = std::max(pmax, psz);
        }
    CUDA_OK(h->d_bigwork.upload(work, s));
    CUDA_OK(h->d_bigsync.alloc((size_t)nsync));
    CUDA_OK(h->d_partial.alloc((size_t)pmax));
    h->partial_len = pmax;
    CUDA_OK(cudaStreamSynchronize(s));
    return 0;
}

// CTA tile of a large batch's GEMMs: 64 for the LDG kernel, else CB200_TMA_TILE (0: by front size)
int gemm_tile(const cb200_handle* h, const Batch& B) {
    if (!(h->use_tma && B.all_padded)) return GBM;
    return h->tma_tile == 64 || h->tma_tile == 128 ? h->tma_tile : (B.maxnf >= 1024 ? 128 : 64);
}

// Schur and assembly tile lists of every large batch (the Schur list for the batch's GEMM tile), after
// build_plans and build_tensor_maps.  They depend on the symbolic structure only.
int upload_tile_lists(cb200_handle* h) {
    const Symbolic& S = h->S;
    std::vector<TileEntry> st, at; std::vector<TileRect> sr, ar;
    // multi-GPU: the children this rank does not assemble get no rectangles (DevSym::active)
    const int8_t* act = h->dist ? h->h_active.data() : nullptr;
    for (LevelPlan& P : h->plan)
        for (Batch* B : {&P.large, &P.topf}) {
            if (!B->cnt) continue;
            const bool gather = B == &P.large;
            const int32_t* fr = h->h_batches.data() + B->off;
            B->schur_off = (int32_t)st.size();
            build_tile_lists(S, fr, B->cnt, gemm_tile(h, *B), true, gather, act, st, sr);
            B->nschur = (int32_t)st.size() - B->schur_off;
            B->asm_off = (int32_t)at.size();
            build_tile_lists(S, fr, B->cnt, ASM_T, false, gather, act, at, ar);
            B->nasm = (int32_t)at.size() - B->asm_off;
        }
    h->n_schur_tiles = (int64_t)st.size(); h->n_schur_rects = (int64_t)sr.size();
    h->n_asm_tiles = (int64_t)at.size(); h->n_asm_rects = (int64_t)ar.size();
    st.push_back({0, 0, 0, (int32_t)sr.size()}); at.push_back({0, 0, 0, (int32_t)ar.size()});
    if (sr.empty()) sr.resize(1);
    if (ar.empty()) ar.resize(1);
    cudaStream_t s = h->stream;
    CUDA_OK(h->d_schur_tiles.upload(st, s)); CUDA_OK(h->d_schur_rects.upload(sr, s));
    CUDA_OK(h->d_asm_tiles.upload(at, s)); CUDA_OK(h->d_asm_rects.upload(ar, s));
    CUDA_OK(cudaStreamSynchronize(s));
    return 0;
}

// all-reduce (sum) of the panel and update block of every front of a batch, one NCCL group
int allreduce_fronts(cb200_handle* h, const Batch& B, const std::vector<int32_t>& list) {
    const Symbolic& S = h->S;
    NCCL_OK(g_nccl.GroupStart());
    for (int32_t k = 0; k < B.cnt; ++k) {
        const int32_t sn = list[k];
        const int64_t ns = S.ns(sn), nr = S.nr(sn), ld = S.panel_ld[sn];
        double* Lp = h->d_L.p + S.panel_off[sn];
        NCCL_OK(g_nccl.AllReduce(Lp, Lp, (size_t)(ld * ns), ncclDouble, ncclSum, h->comm, h->stream));
        if (nr > 0) {
            double* Us = h->d_U.p + S.upd_off[sn];
            NCCL_OK(g_nccl.AllReduce(Us, Us, (size_t)(nr * nr), ncclDouble, ncclSum, h->comm, h->stream));
        }
    }
    NCCL_OK(g_nccl.GroupEnd());
    return 0;
}

// zero the update blocks of the pre-assembled large fronts of one level (kernels.cuh, G6)
__global__ void k_zero_upd(DevSym S, const int32_t* batch, int gather, double* Ust) {
    const int s = batch[blockIdx.y];
    if (gathers_update(S, s, gather)) return;
    const int64_t nr = S.rows_ptr[s + 1] - S.rows_ptr[s];
    double* U = Ust + S.upd_off[s];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nr * nr;
         i += (int64_t)gridDim.x * blockDim.x) U[i] = 0.0;
}

// numeric factorisation of whatever is in d_nz (+ optional on-device static regularisation)
// Replays `body` (a fixed sequence of stream operations on h->stream) through a CUDA graph: the
// launch sequence of a factorisation / solve sweep only depends on the symbolic structure, so it
// is captured once and relaunched with one call per IP iteration.
template <class F> int run_captured(cb200_handle* h, GraphExec& g, F body, int bit = 1) {
    // use_cuda_graph is a bit mask: 1 = solve sweeps, 2 = factorisation
    if (!(h->st.use_cuda_graph & bit) || g.failed || h->detail) return body();
    if (!g.exec) {
        const double l0 = h->tm.nlaunch;
        cudaGraph_t graph = nullptr;
        if (cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
            cudaGetLastError(); g.failed = true; return body();
        }
        int rc = body();
        cudaError_t e = cudaStreamEndCapture(h->stream, &graph);
        g.nlaunch = h->tm.nlaunch - l0; h->tm.nlaunch = l0;
        if (rc != 0 || e != cudaSuccess || !graph) {
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError(); g.failed = true;
            return rc != 0 ? rc : body();
        }
        e = cudaGraphInstantiate(&g.exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) { cudaGetLastError(); g.exec = nullptr; g.failed = true; return body(); }
    }
    CUDA_OK(cudaGraphLaunch(g.exec, h->stream));
    h->tm.nlaunch += g.nlaunch;
    return 0;
}

int factor_body(cb200_handle* h, bool static_reg) {
    cudaStream_t st = h->stream;
    const auto& S = h->S;
    if (h->detail >= 2) h->tm.begin(Timers::NCOARSE + Timers::F_PROLOGUE, st);
    CUDA_OK(cudaMemsetAsync(h->d_L.p, 0, h->d_L.n * sizeof(double), st));
    CUDA_OK(cudaMemsetAsync(h->d_nreg.p, 0, sizeof(unsigned int), st));
    if (h->nnzK) { k_scatter<<<nblk(h->nnzK, 256), 256, 0, st>>>(h->d_nz.p, h->d_amap.p, h->nnzK, h->d_L.p); LAUNCH(h); }
    if (static_reg && h->st.static_regularization_enable && h->N) {
        CUDA_OK(cudaMemsetAsync(h->d_scal.p, 0, sizeof(unsigned long long), st));
        k_diag_absmax<<<std::min(nblk(h->N, 256), h->reduce_blocks), 256, 0, st>>>(h->d_nz.p, h->d_diagidx.p, h->N, h->d_scal.p);
        k_compute_eps<<<1, 1, 0, st>>>(h->d_scal.p, h->st.static_regularization_constant,
                                       h->st.static_regularization_proportional, h->d_eps.p);
        k_shift_diag<<<nblk(h->N, 256), 256, 0, st>>>(h->d_nz.p, h->d_diagidx.p, h->d_amap.p,
                                                      h->d_dsign_orig.p, h->d_eps.p, h->N, h->d_L.p);
        h->tm.nlaunch += 3;
    }
    RegParams rp{h->st.dynamic_regularization_eps, h->st.dynamic_regularization_delta,
                 h->st.dynamic_regularization_enable, h->d_reglog.p};
    DevSym ds = devsym(h);
    if (h->dist && h->rank != 0 && !h->h_top_list.empty()) {
        // the original entries of the replicated top fronts are contributed by rank 0 only
        k_zero_panels<<<dim3(32, (unsigned)h->h_top_list.size()), 256, 0, st>>>(ds, h->d_top_list.p, h->d_L.p);
        LAUNCH(h);
    }
    if (h->detail >= 2) h->tm.end(st);
    for (int lv = 0; lv < S.nlevels; ++lv) {
        const LevelPlan& P = h->plan[lv];
        bool small_work = false;
        for (int c = 0; c < NSMALL; ++c) small_work |= P.small[c].cnt != 0;
        for (int c = 0; c < NPANEL; ++c) small_work |= P.panel[c].cnt != 0;
        // the small-front kernels of a level run beside the pivot-block chain of its large fronts
        const bool ms = h->ms_on() && small_work && (P.large.cnt || P.topf.cnt);
        cudaStream_t ss = ms ? h->side[0] : st;
        if (ms) h->fork(1);
        if (h->detail) h->tm.begin(Timers::SMALL, st);
        launch_small<32, 8>(h, P.small[0], 0, rp, ss);     // size classes kSmallNf[0..5]: a warp per front
        launch_small<64, 1>(h, P.small[1], 1, rp, ss);     // up to nf 16, a CTA per front above
        launch_small<128, 1>(h, P.small[2], 2, rp, ss);
        launch_small<256, 1>(h, P.small[3], 3, rp, ss);
        launch_small<256, 1>(h, P.small[4], 4, rp, ss);
        launch_small<256, 1>(h, P.small[5], 5, rp, ss);
        for (int c = 0; c < NPANEL; ++c) {
            const Batch& b = P.panel[c];
            if (!b.cnt) continue;
            const size_t sm = (size_t)b.maxpanel * sizeof(double);
            FineScope fs(h, Timers::F_PANEL0 + c);
            k_factor_panel<<<b.cnt, 256, sm, ss>>>(ds, h->d_batches.p + b.off, b.maxpanel, b.maxnf, h->d_L.p, h->d_U.p,
                                                   h->d_D.p, h->d_Dinv.p, rp, h->d_nreg.p);
            LAUNCH(h);
        }
        if (h->detail) h->tm.end(st);
        for (int pass = 0; pass < 2; ++pass) {
            const Batch& B = pass == 0 ? P.large : P.topf;
            if (!B.cnt) continue;
            const bool is_top = pass == 1;
            const int32_t* bl = h->d_batches.p + B.off;
            const int64_t* wo = h->d_woff.p + B.off;
            // the update blocks of the replicated top fronts are summed over the GPUs before their Schur
            // update, so they are pre-assembled; other fronts gather theirs in the Schur epilogue
            const int gather = is_top ? 0 : 1;
            if (h->detail) h->tm.begin(Timers::ASM, st);
            if (!gather || B.pre_assembled) {
              FineScope fs(h, Timers::F_ZERO);
              k_zero_upd<<<dim3(std::max(1, std::min(64, nblk((int64_t)B.maxnr * B.maxnr, 1024))), B.cnt), 256, 0, st>>>(ds, bl, gather, h->d_U.p);
              LAUNCH(h); }
            { FineScope fs(h, Timers::F_ASM);
              if (B.nasm) {
                  k_assemble_tiles<<<B.nasm, 256, 0, st>>>(ds, bl, h->d_asm_tiles.p + B.asm_off, h->d_asm_rects.p, gather,
                                                           h->d_L.p, h->d_U.p);
                  LAUNCH(h);
              }
              for (int32_t k = 0; k < B.cnt; ++k) {
                  const int32_t sn = h->h_batches[B.off + k];
                  const int32_t nch = S.child_ptr[sn + 1] - S.child_ptr[sn];
                  if (nch > MANY_CHILDREN) { k_assemble_atomic<<<nch, 64, 0, st>>>(ds, sn, h->d_L.p, h->d_U.p); LAUNCH(h); }
              } }
            if (is_top && h->dist) {
                // root-front assembly across GPUs: every rank holds the contributions of its own
                // subtrees (rank 0 also the original entries); sum them over NVLink.
                FineScope fs(h, Timers::F_COMM);
                std::vector<int32_t> list(h->h_top_by_level[lv]);
                int rc = allreduce_fronts(h, B, list);
                if (rc) return rc;
            }
            if (h->detail) { h->tm.end(st); h->tm.begin(Timers::PANEL, st); }
            const size_t smrows = (size_t)(2 * PB * (PB + 1)) * sizeof(double);
            // one update launch (either version): mode 0 = panel step at pivot block J0, mode 1 = Schur
            // mode 1 runs over the batch's Schur tile list, which was built for this same tile size
            auto launch_update = [&](int mode, int J0) {
                const bool tma = h->use_tma && B.all_padded;
                const int T = gemm_tile(h, B);
                int gx, ny, na = 1;
                const TileEntry* tl = nullptr;
                if (mode == 0) {
                    const int tj0 = (J0 + PB) / T;
                    const int nbt = (B.maxns - 1) / T - tj0 + 1;          // panel column tiles still to update
                    na = (B.maxnf - 1) / T - tj0 + 1;
                    if (nbt <= 0 || na <= 0) return;
                    gx = nbt * na;
                    ny = B.active(J0 + PB);                                // fronts that still have panel columns to update
                } else {
                    gx = B.nschur; ny = 1;
                    tl = h->d_schur_tiles.p + B.schur_off;
                }
                if (gx <= 0 || ny <= 0) return;
                const TileRect* rc = h->d_schur_rects.p;
                if (tma && T == 128)
                    k_ldl_update_tma<128><<<dim3(gx, ny), tma_threads(128), tma_gemm_smem(128), st>>>(
                        ds, bl, tl, rc, h->d_tmaps.p, h->d_tmap_of.p, mode, J0, na, gather, h->tma_kmajor, h->d_L.p, h->d_U.p, h->d_D.p);
                else if (tma)
                    k_ldl_update_tma<64><<<dim3(gx, ny), tma_threads(64), tma_gemm_smem(64), st>>>(
                        ds, bl, tl, rc, h->d_tmaps64.p, h->d_tmap_of.p, mode, J0, na, gather, h->tma_kmajor, h->d_L.p, h->d_U.p, h->d_D.p);
                else
                    k_ldl_update_ldg<<<dim3(gx, ny), 256, 0, st>>>(ds, bl, tl, rc, mode, J0, na, gather, h->d_L.p, h->d_U.p, h->d_D.p);
                LAUNCH(h);
            };
            for (int kb = 0; kb < B.maxns; kb += PB) {
                const int nact = B.active(kb);
                if (nact <= 0) break;
                { FineScope fs(h, Timers::F_DIAG);
                  k_piv_diag<<<nact, 256, 0, st>>>(ds, bl, kb, h->d_L.p, h->d_W.p, wo, h->d_D.p, h->d_Dinv.p, rp, h->d_nreg.p);
                  LAUNCH(h); }
                const int rows_below = B.maxnf - kb - 1;
                if (rows_below > 0) {
                    FineScope fs(h, Timers::F_ROWS);
                    k_piv_rows<<<dim3(nblk(rows_below, GBM), nact), 256, smrows, st>>>(ds, bl, kb, h->d_L.p, h->d_W.p, wo, h->d_Dinv.p);
                    LAUNCH(h);
                }
                if (kb + PB < B.maxns) { FineScope fs(h, Timers::F_PANELUPD); launch_update(0, kb); }
            }
            if (h->detail) { h->tm.end(st); h->tm.begin(Timers::SCHUR, st); }
            { FineScope fs(h, Timers::F_SCHUR); launch_update(1, 0); }
            if (h->detail) h->tm.end(st);
            FineScope fs(h, Timers::F_FINISH);
            k_finish_large<<<dim3(nblk(B.maxns, PB), B.cnt), 256, 0, st>>>(ds, bl, h->d_L.p, h->d_W.p, wo);
            LAUNCH(h);
        }
        if (ms) h->join(1);
    }
    CUDA_OK(cudaGetLastError());
    return 0;
}

int factor(cb200_handle* h, bool static_reg) {
    h->tm.begin(Timers::FACTOR, h->stream);
    int rc = run_captured(h, h->g_factor[static_reg ? 1 : 0], [&]() { return factor_body(h, static_reg); }, 2);
    h->tm.end(h->stream);
    h->tm.nfactor += 1;
    return rc;
}

// y (permuted, in d_y) <- K^-1 : forward, diagonal, backward
SubTrees subtrees(cb200_handle* h) {
    SubTrees T;
    T.sn0 = h->d_sub_sn0.p; T.sn1 = h->d_sub_sn1.p; T.order = h->d_sub_order.p; T.order_ptr = h->d_sub_optr.p;
    T.lvl_off = h->d_sub_lvl.p; T.nlev = h->sub_nlev; T.maxcols = h->sub_maxcols; T.maxrows = h->sub_maxrows;
    return T;
}
size_t subtree_smem_fwd(const cb200_handle* h) { return ((size_t)h->sub_maxcols + h->sub_maxrows + 8 * SUB_MAXNF) * sizeof(double); }
size_t subtree_smem_bwd(const cb200_handle* h) { return ((size_t)h->sub_maxcols + 8 * (SUB_MAXNF + 32 * BT_LD)) * sizeof(double); }

template <int R>
int sweeps_body(cb200_handle* h, const SweepBufs& V) {
    const auto& S = h->S;
    // tickets and ready flags of the big-solve chains start from zero in every sweep (a memset node
    // of the captured graph); the error word [0] is reset per solve call
    if (h->d_bigsync.n > 1)
        CUDA_OK(cudaMemsetAsync(h->d_bigsync.p + 1, 0, (h->d_bigsync.n - 1) * sizeof(unsigned), h->stream));
    if (R == 1 && h->nsub) {  // the bottom subtrees first: everything above them depends on their contributions
        FineScope fs(h, Timers::F_FWD_SUB);
        k_fwd_subtree<<<h->nsub, 256, subtree_smem_fwd(h), h->stream>>>(devsym(h), subtrees(h), h->d_L.p, V.y, V.uvec);
        LAUNCH(h);
    }
    for (int lv = 0; lv < S.nlevels; ++lv) launch_fwd_level<R>(h, h->plan[lv], lv, V);
    for (int lv = S.nlevels - 1; lv >= 0; --lv) launch_bwd_level<R>(h, h->plan[lv], V);
    if (R == 1 && h->nsub) {
        FineScope fs(h, Timers::F_BWD_SUB);
        k_bwd_subtree<<<h->nsub, 256, subtree_smem_bwd(h), h->stream>>>(devsym(h), subtrees(h), h->d_L.p, h->d_Dinv.p, V.y);
        LAUNCH(h);
    }
    CUDA_OK(cudaGetLastError());
    return 0;
}

int tri_solve(cb200_handle* h, const double* d_rhs, double* d_sol) {
    cudaStream_t st = h->stream;
    h->tm.begin(Timers::SOLVE, st);
    {
        FineScope fs(h, Timers::F_PERMUTE);
        if (h->N) { k_pack_perm<<<nblk(h->N, 256), 256, 0, st>>>(d_rhs, h->d_perm.p, h->N, h->d_y.p); LAUNCH(h); }
        if (h->dist && h->N) {
            // top-front entries of the right-hand side are contributed by rank 0 only
            k_mask_vec<<<nblk(h->N, 256), 256, 0, st>>>(h->d_y.p, h->d_topcolkeep.p, h->N); LAUNCH(h);
        }
    }
    const SweepBufs V{h->d_y.p, h->d_uvec.p, h->d_partial.p};
    int rc = run_captured(h, h->g_solve, [&]() { return sweeps_body<1>(h, V); });
    if (rc) return rc;
    if (h->dist && h->N) {
        // every rank holds the solution on its own subtrees (+ the replicated top part): gather by
        // zeroing what a rank does not own and summing over NVLink
        FineScope fs(h, Timers::F_COMM);
        k_mask_vec<<<nblk(h->N, 256), 256, 0, st>>>(h->d_y.p, h->d_keepcol.p, h->N); LAUNCH(h);
        NCCL_OK(g_nccl.AllReduce(h->d_y.p, h->d_y.p, (size_t)h->N, ncclDouble, ncclSum, h->comm, st));
    }
    if (h->N) {
        FineScope fs(h, Timers::F_PERMUTE);
        k_unpack_perm<<<nblk(h->N, 256), 256, 0, st>>>(h->d_y.p, h->d_perm.p, h->N, d_sol); LAUNCH(h);
    }
    h->tm.end(st);
    h->tm.nsolve += 1;
    CUDA_OK(cudaGetLastError());
    return 0;
}

// e = b - K xi ; norm bits accumulated into d_scal[slot]
int residual(cb200_handle* h, const double* d_xi, double* d_e, int slot) {
    cudaStream_t st = h->stream;
    h->tm.begin(Timers::SPMV, st);
    CUDA_OK(cudaMemsetAsync(h->d_scal.p + slot, 0, sizeof(unsigned long long), st));
    if (h->N) {
        // lanes per row chosen from the mean row length of the symmetric matrix
        const double mean_row = 2.0 * (double)h->nnzK / (double)h->N;
        if (mean_row > 48.0)
            k_residual<32><<<nblk(h->N * 32, 256), 256, 0, st>>>(h->N, h->d_cp.p, h->d_ri.p, h->d_nz.p, h->d_tp.p,
                                                                 h->d_tc.p, h->d_tpos.p, d_xi, h->d_b.p, d_e,
                                                                 h->d_scal.p + slot);
        else
            k_residual<4><<<nblk(h->N * 4, 256), 256, 0, st>>>(h->N, h->d_cp.p, h->d_ri.p, h->d_nz.p, h->d_tp.p,
                                                               h->d_tc.p, h->d_tpos.p, d_xi, h->d_b.p, d_e,
                                                               h->d_scal.p + slot);
        if (h->n_long_rows) {
            k_residual_long<<<h->n_long_rows, 256, 0, st>>>(h->d_long_rows.p, h->d_cp.p, h->d_ri.p, h->d_nz.p,
                                                            h->d_tp.p, h->d_tc.p, h->d_tpos.p, d_xi, h->d_b.p,
                                                            d_e, h->d_scal.p + slot);
            LAUNCH(h);
        }
        LAUNCH(h);
    }
    h->tm.end(st);
    return 0;
}

// Error word of the big-solve chains (k_big_tri_*: a ready flag not set within the spin bound), one
// per solve call: reset before the first sweep, read back with the call's final synchronise.
int reset_chain_error(cb200_handle* h) {
    if (h->d_bigsync.n) CUDA_OK(cudaMemsetAsync(h->d_bigsync.p, 0, sizeof(unsigned), h->stream));
    return 0;
}
int read_chain_error(cb200_handle* h, unsigned* err) {
    if (h->d_bigsync.n) CUDA_OK(cudaMemcpyAsync(err, h->d_bigsync.p, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    return 0;
}

int read_scalars(cb200_handle* h, double* out, int first, int count) {
    unsigned long long bits[4];
    CUDA_OK(cudaMemcpyAsync(bits, h->d_scal.p + first, count * sizeof(unsigned long long),
                            cudaMemcpyDeviceToHost, h->stream));
    CUDA_OK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < count; ++i) { long long b = (long long)bits[i]; std::memcpy(&out[i], &b, 8); }
    return 0;
}


// ---- multi-right-hand-side sweeps (kernels_multi.cuh)
constexpr size_t kMaxDynSmem = 200 * 1024;     // leaves room for the kernels' static shared memory (227 KB per CTA)

template <int R> void set_multi_smem_attrs() {
    for (const void* k : {(const void*)k_fwd_warp_multi<32, R>, (const void*)k_fwd_warp_multi<16, R>,
                          (const void*)k_bwd_warp_multi<32, R>, (const void*)k_bwd_warp_multi<16, R>,
                          (const void*)k_fwd_cta_multi<R>, (const void*)k_bwd_cta_multi<R>})
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynSmem);
}

// Allocates the multi-RHS buffers on the first multi call.  The sweep width is 4 unless the shared memory
// of some warp- or CTA-class batch would not fit at that width (fronts of more than ~7000 rows solved by
// one CTA); it is then 2, or 1.
int ensure_multi(cb200_handle* h) {
    if (h->multi_w) return 0;
    auto fits = [&](int R) {
        for (const LevelPlan& P : h->plan) {
            const Batch &b1 = P.solve[1], &b5 = P.solve[5], &b2 = P.solve[2];
            if (b1.cnt && (fwd_warp_smem(b1.maxnf, R) > kMaxDynSmem || bwd_warp_smem(b1.maxnf, 32, R) > kMaxDynSmem)) return false;
            if (b5.cnt && (fwd_warp_smem(b5.maxnf, R) > kMaxDynSmem || bwd_warp_smem(b5.maxnf, 16, R) > kMaxDynSmem)) return false;
            if (b2.cnt && ((size_t)b2.maxnf * R * sizeof(double) > kMaxDynSmem || bwd_cta_smem(b2.maxnf, R) > kMaxDynSmem)) return false;
        }
        return true;
    };
    int w = 4;
    while (w > 1 && !fits(w)) w /= 2;
    const size_t N = (size_t)std::max<int64_t>(1, h->N);
    if (w > 1) {
        CUDA_OK(h->d_my.alloc(N * w));
        CUDA_OK(h->d_muvec.alloc(std::max<size_t>(1, h->S.rows.size()) * w));
        CUDA_OK(h->d_mpartial.alloc((size_t)h->partial_len * w));
        set_multi_smem_attrs<2>();
        if (w == 4) set_multi_smem_attrs<4>();
        CUDA_OK(cudaGetLastError());
    }
    for (DevBuf<double>* b : {&h->d_mb, &h->d_mx, &h->d_mdx, &h->d_me, &h->d_mstage}) {
        CUDA_OK(b->alloc(N * w));
        CUDA_OK(cudaMemsetAsync(b->p, 0, N * w * sizeof(double), h->stream));
    }
    CUDA_OK(h->d_mscal.alloc(8));
    h->multi_w = w;
    return 0;
}

// width of the next sweep for `rem` remaining columns: the full width, else the narrowest instantiated
// width that holds them (a short chunk carries zero padding columns)
int chunk_width(int w, int rem) {
    if (rem >= w) return w;
    return rem == 1 ? 1 : (rem == 2 ? 2 : 4);
}

// one R-wide sweep: column r < k of src (element i at src[i*rs + r*cs]) -> the same place of dst
int tri_solve_multi(cb200_handle* h, int R, int k, const double* src, int64_t rs, int64_t cs,
                    double* dst, int64_t drs, int64_t dcs) {
    cudaStream_t st = h->stream;
    const int64_t N = h->N;
    double* y = R == 1 ? h->d_y.p : h->d_my.p;
    h->tm.begin(Timers::SOLVE, st);
    {
        FineScope fs(h, Timers::F_PERMUTE);
        k_pack_perm_multi<<<nblk(N * R, 256), 256, 0, st>>>(src, rs, cs, k, R, h->d_perm.p, N, y); LAUNCH(h);
    }
    int rc;
    if (R == 1) {
        const SweepBufs V{h->d_y.p, h->d_uvec.p, h->d_partial.p};
        rc = run_captured(h, h->g_solve, [&]() { return sweeps_body<1>(h, V); });
    } else if (R == 2) {
        const SweepBufs V{h->d_my.p, h->d_muvec.p, h->d_mpartial.p};
        rc = run_captured(h, h->g_msolve[0], [&]() { return sweeps_body<2>(h, V); });
    } else {
        const SweepBufs V{h->d_my.p, h->d_muvec.p, h->d_mpartial.p};
        rc = run_captured(h, h->g_msolve[1], [&]() { return sweeps_body<4>(h, V); });
    }
    if (rc) return rc;
    {
        FineScope fs(h, Timers::F_PERMUTE);
        k_unpack_perm_multi<<<nblk(N * R, 256), 256, 0, st>>>(y, k, R, h->d_perm.p, N, dst, drs, dcs); LAUNCH(h);
    }
    h->tm.end(st);
    h->tm.nsolve += 1;
    h->n_multi_sweeps += 1;
    CUDA_OK(cudaGetLastError());
    return 0;
}

template <int R>
void launch_residual_multi(cb200_handle* h, const double* xi, double* e, unsigned long long* norms) {
    cudaStream_t st = h->stream;
    const double mean_row = 2.0 * (double)h->nnzK / (double)h->N;
    if (mean_row > 48.0)
        k_residual_multi<32, R><<<nblk(h->N * 32, 256), 256, 0, st>>>(h->N, h->d_cp.p, h->d_ri.p, h->d_nz.p, h->d_tp.p,
                                                                      h->d_tc.p, h->d_tpos.p, xi, h->d_mb.p, e, norms);
    else
        k_residual_multi<4, R><<<nblk(h->N * 4, 256), 256, 0, st>>>(h->N, h->d_cp.p, h->d_ri.p, h->d_nz.p, h->d_tp.p,
                                                                    h->d_tc.p, h->d_tpos.p, xi, h->d_mb.p, e, norms);
    LAUNCH(h);
    if (h->n_long_rows) {
        k_residual_long_multi<R><<<h->n_long_rows, 256, 0, st>>>(h->d_long_rows.p, h->d_cp.p, h->d_ri.p, h->d_nz.p,
                                                                 h->d_tp.p, h->d_tc.p, h->d_tpos.p, xi, h->d_mb.p, e, norms);
        LAUNCH(h);
    }
}
// e = b - K xi for R interleaved columns (b = d_mb); the norms go to d_mscal[4, 4 + R)
int residual_multi(cb200_handle* h, int R, const double* xi, double* e) {
    cudaStream_t st = h->stream;
    h->tm.begin(Timers::SPMV, st);
    CUDA_OK(cudaMemsetAsync(h->d_mscal.p + 4, 0, 4 * sizeof(unsigned long long), st));
    if (R == 1) launch_residual_multi<1>(h, xi, e, h->d_mscal.p + 4);
    else if (R == 2) launch_residual_multi<2>(h, xi, e, h->d_mscal.p + 4);
    else launch_residual_multi<4>(h, xi, e, h->d_mscal.p + 4);
    h->tm.end(st);
    return 0;
}
// max |v_r| of R interleaved columns into d_mscal[slot, slot + R)
int absmax_multi(cb200_handle* h, int R, const double* v, int slot) {
    cudaStream_t st = h->stream;
    CUDA_OK(cudaMemsetAsync(h->d_mscal.p + slot, 0, 4 * sizeof(unsigned long long), st));
    const int g = std::min(nblk(h->N, 256), h->reduce_blocks);
    if (R == 1) k_absmax_multi<1><<<g, 256, 0, st>>>(v, h->N, h->d_mscal.p + slot);
    else if (R == 2) k_absmax_multi<2><<<g, 256, 0, st>>>(v, h->N, h->d_mscal.p + slot);
    else k_absmax_multi<4><<<g, 256, 0, st>>>(v, h->N, h->d_mscal.p + slot);
    LAUNCH(h);
    return 0;
}
int read_mscal(cb200_handle* h, double* out, int first, int count) {
    unsigned long long bits[8];
    CUDA_OK(cudaMemcpyAsync(bits, h->d_mscal.p + first, count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CUDA_OK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < count; ++i) { long long b = (long long)bits[i]; std::memcpy(&out[i], &b, 8); }
    return 0;
}

// Solution, refinement rounds and status of R interleaved systems (b in d_mb, k real columns), with the
// per-column rules of cb200_solve_ir; the accepted iterates end in d_mx.
int solve_ir_chunk(cb200_handle* h, int R, int k, int32_t* rounds, int32_t* okc) {
    cudaStream_t st = h->stream;
    const int64_t N = h->N;
    const cb200_settings& S = h->st;
    int rc = absmax_multi(h, R, h->d_mb.p, 0); if (rc) return rc;
    rc = tri_solve_multi(h, R, R, h->d_mb.p, R, 1, h->d_mx.p, R, 1); if (rc) return rc;
    for (int c = 0; c < k; ++c) { rounds[c] = 0; okc[c] = 1; }
    if (!S.iterative_refinement_enable) {
        rc = absmax_multi(h, R, h->d_mx.p, 4); if (rc) return rc;
        double v[4];
        rc = read_mscal(h, v, 4, R); if (rc) return rc;
        for (int c = 0; c < k; ++c) okc[c] = std::isfinite(v[c]);
        return 0;
    }
    // _iterative_refinement (kktsolver_directldl.jl:389-449), per column
    rc = residual_multi(h, R, h->d_mx.p, h->d_me.p); if (rc) return rc;
    double sc[8];
    rc = read_mscal(h, sc, 0, 8); if (rc) return rc;
    double normb[4], norme[4], last[4];
    bool done[4];
    for (int c = 0; c < R; ++c) {
        normb[c] = sc[c]; norme[c] = sc[4 + c]; last[c] = 0;
        done[c] = c >= k;
        if (c < k && !std::isfinite(norme[c])) { okc[c] = 0; done[c] = true; }
    }
    for (int i = 0; i < S.iterative_refinement_max_iter; ++i) {
        bool act[4], any = false;
        for (int c = 0; c < R; ++c) {
            if (!done[c] && norme[c] <= S.iterative_refinement_abstol + S.iterative_refinement_reltol * normb[c]) done[c] = true;
            act[c] = !done[c]; any |= act[c];
            if (act[c]) last[c] = norme[c];
        }
        if (!any) break;
        rc = tri_solve_multi(h, R, R, h->d_me.p, R, 1, h->d_mdx.p, R, 1); if (rc) return rc;
        k_axpy_multi<<<nblk(N * R, 256), 256, 0, st>>>(h->d_mdx.p, h->d_mx.p, N * R); LAUNCH(h);
        rc = residual_multi(h, R, h->d_mdx.p, h->d_me.p); if (rc) return rc;
        rc = read_mscal(h, sc, 4, R); if (rc) return rc;
        unsigned take = 0;                         // columns whose new iterate replaces x (the single path's swap)
        for (int c = 0; c < R; ++c) {
            if (!act[c]) continue;
            norme[c] = sc[c];
            rounds[c]++;
            if (!std::isfinite(norme[c])) { okc[c] = 0; done[c] = true; continue; }
            const double ratio = last[c] / norme[c];
            if (ratio < S.iterative_refinement_stop_ratio) {
                if (ratio > 1.0) take |= 1u << c;
                done[c] = true;
            } else take |= 1u << c;
        }
        if (take) { k_select_cols<<<nblk(N * R, 256), 256, 0, st>>>(h->d_mx.p, h->d_mdx.p, N, R, take); LAUNCH(h); }
    }
    return 0;
}
}  // namespace

extern "C" {

int32_t cb200_create(int64_t N, const int64_t* colptr, const int64_t* rowval, const double* nzval,
                     const int64_t* Dsigns, const cb200_settings* stp, cb200_handle** out) {
    try {
        cb200_settings st;
        if (stp) st = *stp; else cb200_default_settings(&st);
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
            set_error("cb200_create: no CUDA device available (this backend has no CPU fallback)");
            return -3;
        }
        CUDA_OK(cudaSetDevice(st.device));
        auto* h = new cb200_handle();
        struct Guard { cb200_handle* h; ~Guard() { if (h) cb200_destroy(h); } } guard{h};   // error paths free everything
        h->st = st; h->N = N; h->base = st.index_base;
        const int64_t base = st.index_base;
        std::vector<int64_t> cp(N + 1), ri;
        for (int64_t i = 0; i <= N; ++i) cp[i] = colptr[i] - base;
        const int64_t nnz = cp[N];
        h->nnzK = nnz;
        ri.resize(nnz);
        for (int64_t i = 0; i < nnz; ++i) ri[i] = rowval[i] - base;
        if (!g_block_hint.empty() && (int64_t)g_block_hint.size() != N) g_block_hint.clear();
        h->opt = options_from_settings(&st);
        // ordering = 1 (auto) with dense cone blocks (PSD cones) in K: the blocks are detected here from the
        // pattern and Dsigns alone - a maximal run of columns of the (-,-) part in which column j holds ALL
        // earlier columns of the run as rows (a dense triangle; dense SOC blocks have at most 4 columns) - so
        // that every caller, the Julia shim included, gets the PSD-safe ordering without knowing about it:
        // coupled variables first, then the blocks by nested dissection of the block graph, or the
        // AMD-class order when there are only a few blocks (symbolic.cpp / ordering.cpp, DESIGN.md 5).
        std::vector<int32_t> detected;
        if (h->opt.ordering == 1 && Dsigns && !h->opt.block_id) {
            std::vector<int32_t> start(N, -1);                 // start[j] = first column of the run j belongs to
            for (int64_t j = 0; j < N; ++j) {
                if (Dsigns[j] >= 0) continue;
                start[j] = (int32_t)j;
                if (j == 0 || start[j - 1] < 0) continue;
                const int64_t want = j - start[j - 1];         // rows start[j-1] .. j-1 must all be present
                int64_t run = 0;
                for (int64_t p = cp[j + 1] - 1; p >= cp[j]; --p) {
                    const int64_t r = ri[p];
                    if (r == j) continue;
                    if (r == j - 1 - run) ++run; else if (r < j - 1 - run) break;
                    if (run == want) break;
                }
                if (run == want) start[j] = start[j - 1];
            }
            detected.assign(N, -1);
            int32_t nblk_found = 0;
            for (int64_t j = 0; j < N;) {
                if (start[j] < 0) { ++j; continue; }
                int64_t e = j; while (e + 1 < N && start[e + 1] == start[j]) ++e;
                if (e - j + 1 >= 5) { for (int64_t q = j; q <= e; ++q) detected[q] = nblk_found; ++nblk_found; }
                j = e + 1;
            }
            if (nblk_found > 0) h->opt.block_id = detected.data();
        }
        symbolic_analyze(N, cp.data(), ri.data(), h->opt, nullptr, h->S);
        h->opt.block_id = nullptr;
        g_block_hint.clear();
        const Symbolic& S = h->S;
        CUDA_OK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        { int nsm = 0; CUDA_OK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->st.device)); h->reduce_blocks = 8 * nsm; }
        for (int i = 0; i < 3; ++i) {
            CUDA_OK(cudaStreamCreateWithFlags(&h->side[i], cudaStreamNonBlocking));
            CUDA_OK(cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming));
        }
        CUDA_OK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
        if (const char* e = getenv("CB200_MULTISTREAM")) h->multi_stream = e[0] != '0';
        if (const char* e = getenv("CB200_SORT_BATCHES")) h->sort_batches = e[0] != '0';
        if (const char* e = getenv("CB200_SUBTREE")) h->use_subtree = e[0] == '1';
        if (const char* e = getenv("CB200_MERGED_ROWS")) h->merged_rows = e[0] != '0';
        cudaStream_t s = h->stream;
        // ---- K
        std::vector<int32_t> ri32(ri.begin(), ri.end());
        CUDA_OK(h->d_cp.upload(cp, s)); CUDA_OK(h->d_ri.upload(ri32, s));
        CUDA_OK(h->d_nz.alloc(nnz));
        if (nnz) CUDA_OK(cudaMemcpyAsync(h->d_nz.p, nzval, nnz * sizeof(double), cudaMemcpyHostToDevice, s));
        // row-wise index of the strictly-upper entries + diagonal positions
        std::vector<int64_t> tp(N + 1, 0), diagidx(N, -1);
        for (int64_t j = 0; j < N; ++j)
            for (int64_t p = cp[j]; p < cp[j + 1]; ++p) {
                if (ri[p] == j) diagidx[j] = p; else if (ri[p] < j) tp[ri[p] + 1]++;
            }
        for (int64_t j = 0; j < N; ++j) tp[j + 1] += tp[j];
        std::vector<int32_t> tc(tp[N]); std::vector<int64_t> tpos(tp[N]);
        {
            std::vector<int64_t> pos(tp.begin(), tp.end() - 1);
            for (int64_t j = 0; j < N; ++j)
                for (int64_t p = cp[j]; p < cp[j + 1]; ++p)
                    if (ri[p] < j) { int64_t q = pos[ri[p]]++; tc[q] = (int32_t)j; tpos[q] = p; }
        }
        CUDA_OK(h->d_tp.upload(tp, s)); CUDA_OK(h->d_tc.upload(tc, s)); CUDA_OK(h->d_tpos.upload(tpos, s));
        {
            std::vector<int32_t> longrows;
            for (int64_t j = 0; j < N; ++j)
                if ((cp[j + 1] - cp[j]) + (tp[j + 1] - tp[j]) > LONG_ROW) longrows.push_back((int32_t)j);
            h->n_long_rows = (int32_t)longrows.size();
            CUDA_OK(h->d_long_rows.upload(longrows, s));
        }
        h->have_diag = std::all_of(diagidx.begin(), diagidx.end(), [](int64_t v) { return v >= 0; });
        if (h->have_diag) CUDA_OK(h->d_diagidx.upload(diagidx, s));
        CUDA_OK(h->d_amap.upload(S.a_map, s));
        std::vector<int8_t> dsp(N), dso(N);
        for (int64_t k = 0; k < N; ++k) {
            dso[k] = (int8_t)(Dsigns ? (Dsigns[k] >= 0 ? 1 : -1) : 1);
        }
        for (int64_t k = 0; k < N; ++k) dsp[k] = dso[S.perm[k]];
        CUDA_OK(h->d_dsign_perm.upload(dsp, s)); CUDA_OK(h->d_dsign_orig.upload(dso, s));
        CUDA_OK(h->d_perm.upload(S.perm, s));
        // ---- symbolic
        CUDA_OK(h->d_sn_first.upload(S.sn_first, s)); CUDA_OK(h->d_rows_ptr.upload(S.rows_ptr, s));
        CUDA_OK(h->d_rows.upload(S.rows, s)); CUDA_OK(h->d_rel.upload(S.rel, s));
        CUDA_OK(h->d_child_ptr.upload(S.child_ptr, s)); CUDA_OK(h->d_child_list.upload(S.child_list, s));
        CUDA_OK(h->d_panel_off.upload(S.panel_off, s)); CUDA_OK(h->d_upd_off.upload(S.upd_off, s));
        CUDA_OK(h->d_ld.upload(S.panel_ld, s));
        CUDA_OK(h->d_front_ptr.upload(S.front_ptr, s)); CUDA_OK(h->d_asm_base.upload(S.asm_base, s));
        CUDA_OK(h->d_asm_colptr.upload(S.asm_colptr, s)); CUDA_OK(h->d_asm_src.upload(S.asm_src, s));
        CUDA_OK(h->d_asm_child.upload(S.asm_child, s)); CUDA_OK(h->d_kids.upload(S.kids, s));
        // ---- level plans (+ workspace sized for them)
        { int rcp = build_plans(h); if (rcp) return rcp; }
        // ---- numeric storage
        CUDA_OK(h->d_L.alloc((size_t)S.panel_off.back()));
        CUDA_OK(h->d_U.alloc((size_t)std::max<int64_t>(1, S.upd_total)));
        CUDA_OK(h->d_D.alloc(N)); CUDA_OK(h->d_Dinv.alloc(N));
        if (N) { CUDA_OK(cudaMemsetAsync(h->d_D.p, 0, N * sizeof(double), s)); CUDA_OK(cudaMemsetAsync(h->d_Dinv.p, 0, N * sizeof(double), s)); }
        CUDA_OK(h->d_uvec.alloc(std::max<size_t>(1, S.rows.size())));

        for (DevBuf<double>* b : {&h->d_b, &h->d_x, &h->d_e, &h->d_dx, &h->d_y}) {
            CUDA_OK(b->alloc(std::max<int64_t>(1, N)));
            CUDA_OK(cudaMemsetAsync(b->p, 0, std::max<int64_t>(1, N) * sizeof(double), s));
        }
        CUDA_OK(h->d_eps.alloc(1)); CUDA_OK(h->d_scal.alloc(4)); CUDA_OK(h->d_nreg.alloc(1)); CUDA_OK(h->d_reglog.alloc(64));
        CUDA_OK(cudaMemsetAsync(h->d_eps.p, 0, sizeof(double), s));
        CUDA_OK(cudaMemsetAsync(h->d_nreg.p, 0, sizeof(unsigned int), s));
        // opt in to large dynamic shared memory for the bigger small-front classes
        CUDA_OK(cudaFuncSetAttribute(k_factor_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_factor_small<256, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     152 * 152 * (int)sizeof(double)));
        CUDA_OK(cudaFuncSetAttribute(k_piv_rows, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (2 * PB * (PB + 1)) * (int)sizeof(double)));
        CUDA_OK(cudaFuncSetAttribute(k_ldl_update_tma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tma_gemm_smem(128)));
        CUDA_OK(cudaFuncSetAttribute(k_ldl_update_tma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tma_gemm_smem(64)));
        { int rct = build_tensor_maps(h); if (rct) return rct; }
        { int rcl = upload_tile_lists(h); if (rcl) return rcl; }
        CUDA_OK(cudaFuncSetAttribute(k_fwd_subtree, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_bwd_subtree, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_bwd_warp<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_bwd_warp<16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_bwd_warp<16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_fwd_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        CUDA_OK(cudaFuncSetAttribute(k_bwd_cta, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        if (S.max_front > 25000) { set_error("front too large for the single-CTA solve kernels"); return -4; }
        CUDA_OK(cudaStreamSynchronize(s));
        guard.h = nullptr;
        *out = h;
        return 0;
    } catch (const std::exception& e) { set_error(e.what()); return -1; }
}

void cb200_destroy(cb200_handle* h) {
    if (!h) return;
    if (h->stream) { cudaStreamSynchronize(h->stream); }
    // graphs captured with NCCL kernels inside hold references on the communicator: ncclCommDestroy waits
    // for them, so the executables go first (seen as a teardown hang with CB200_DIST_GRAPH=1)
    for (GraphExec* g : {&h->g_factor[0], &h->g_factor[1], &h->g_solve, &h->g_msolve[0], &h->g_msolve[1]})
        if (g->exec) { cudaGraphExecDestroy(g->exec); g->exec = nullptr; }
    if (h->comm && g_nccl.ok) { g_nccl.CommDestroy(h->comm); h->comm = nullptr; }
    cudaStream_t s = h->stream;
    for (int i = 0; i < 3; ++i) {
        if (h->side[i]) { cudaStreamSynchronize(h->side[i]); cudaStreamDestroy(h->side[i]); }
        if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
    }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    for (cudaEvent_t e : h->ev_scale) if (e) cudaEventDestroy(e);
    delete h;
    if (s) cudaStreamDestroy(s);
}

// Staging for the inner-boundary uploads.  The reference issues ~5 update_values!/scale_values! calls
// per sparse cone per iteration (directldl_datamaps.jl:61-79), so these calls must not allocate or
// synchronise: the device staging buffers only grow, and the stream is ordered, so the kernel of
// call k+1 cannot overtake the copy of call k.  The staging buffer is reused by the next call only
// after the previous kernel was enqueued behind its copy on the same stream; the H2D copies from
// pageable host memory return after the source has been staged by the driver, so the caller may
// overwrite `index` / `values` on return.
// Page-locked caller buffers make cudaMemcpyAsync truly asynchronous: then (and only then) the call
// must wait for the copy before returning, because the caller may overwrite its buffer.
static bool host_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

static int stage_reserve(cb200_handle* h, size_t nidx, size_t nval) {
    if (nidx > h->stage_idx_cap) {
        CUDA_OK(cudaStreamSynchronize(h->stream));          // the old buffer may still be in use
        size_t cap = std::max(nidx, std::max<size_t>(4096, 2 * h->stage_idx_cap));
        CUDA_OK(h->d_stage_idx.alloc(cap)); h->stage_idx_cap = cap;
    }
    if (nval > h->stage_val_cap) {
        CUDA_OK(cudaStreamSynchronize(h->stream));
        size_t cap = std::max(nval, std::max<size_t>(4096, 2 * h->stage_val_cap));
        CUDA_OK(h->d_stage_val.alloc(cap)); h->stage_val_cap = cap;
    }
    return 0;
}

int32_t cb200_update_values(cb200_handle* h, const int64_t* index, const double* values, int64_t len) {
    if (len <= 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    { int rc = stage_reserve(h, (size_t)len, (size_t)len); if (rc) return rc; }
    CUDA_OK(cudaMemcpyAsync(h->d_stage_idx.p, index, len * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
    CUDA_OK(cudaMemcpyAsync(h->d_stage_val.p, values, len * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    k_update_values<<<nblk(len, 256), 256, 0, h->stream>>>(h->d_nz.p, h->d_stage_idx.p, h->d_stage_val.p, len, h->base);
    LAUNCH(h);
    CUDA_OK(cudaGetLastError());
    if (host_is_pinned(index) || host_is_pinned(values)) CUDA_OK(cudaStreamSynchronize(h->stream));
    return 0;
}

int32_t cb200_scale_values(cb200_handle* h, const int64_t* index, int64_t len, double scale) {
    if (len <= 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    { int rc = stage_reserve(h, (size_t)len, 0); if (rc) return rc; }
    CUDA_OK(cudaMemcpyAsync(h->d_stage_idx.p, index, len * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
    k_scale_values<<<nblk(len, 256), 256, 0, h->stream>>>(h->d_nz.p, h->d_stage_idx.p, scale, len, h->base);
    LAUNCH(h);
    CUDA_OK(cudaGetLastError());
    if (host_is_pinned(index)) CUDA_OK(cudaStreamSynchronize(h->stream));
    return 0;
}

static int finish_factor(cb200_handle* h) {
    // success = all(isfinite, Dinv)   (directldl_qdldl.jl:79)
    CUDA_OK(cudaMemsetAsync(h->d_scal.p + 3, 0, sizeof(unsigned long long), h->stream));
    if (h->N) { k_absmax<<<std::min(nblk(h->N, 256), h->reduce_blocks), 256, 0, h->stream>>>(h->d_Dinv.p, h->N, h->d_scal.p + 3); LAUNCH(h); }
    if (h->dist) {
        // every rank must take the same success / failure branch: reduce the status over the ranks
        // (the value is the bit pattern of a non-negative double, so unsigned max == double max)
        NCCL_OK(g_nccl.AllReduce(h->d_scal.p + 3, h->d_scal.p + 3, 1, ncclUint64, ncclMax, h->comm, h->stream));
    }
    double v[1];
    int rc = read_scalars(h, v, 3, 1);
    if (rc) return rc;
    h->tm.collect();
    return std::isfinite(v[0]) ? 0 : 1;
}

int32_t cb200_refactor(cb200_handle* h) {
    CUDA_OK(cudaSetDevice(h->st.device));
    int rc = factor(h, /*static_reg=*/false);
    if (rc) return rc;
    return finish_factor(h);
}

int32_t cb200_solve(cb200_handle* h, double* x, const double* b) {
    const int64_t N = h->N;
    if (N == 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    CUDA_OK(cudaMemcpyAsync(h->d_b.p, b, N * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    int rc = reset_chain_error(h); if (rc) return rc;
    rc = tri_solve(h, h->d_b.p, h->d_x.p);
    if (rc) return rc;
    CUDA_OK(cudaMemcpyAsync(x, h->d_x.p, N * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    unsigned chain_err = 0;
    rc = read_chain_error(h, &chain_err); if (rc) return rc;
    CUDA_OK(cudaStreamSynchronize(h->stream));
    h->tm.collect();
    if (chain_err) { set_error("cb200_solve: a big-front solve chain timed out waiting for a block"); return -4; }
    return 0;
}

int32_t cb200_info(const cb200_handle* h, int64_t* nnzA, int64_t* nnzL, int32_t* ngpus) {
    if (nnzA) *nnzA = h->nnzK;
    if (nnzL) *nnzL = h->S.nnzL;
    if (ngpus) *ngpus = h->nranks;
    return 0;
}

int32_t cb200_set_maps(cb200_handle* h, int64_t n, int64_t m, int64_t p,
                       const int64_t* map_P, int64_t nnzP, const int64_t* map_A, int64_t nnzA,
                       const int64_t* map_Hs, int64_t nHs, const int64_t* map_diag_full,
                       int64_t ncones, const int32_t* cone_type, const int64_t* cone_dim,
                       const int64_t* map_soc_u, const int64_t* map_soc_v, const int64_t* map_soc_D) {
    try {
        if (n + m + p != h->N) { set_error("cb200_set_maps: n+m+p != N"); return -2; }
        CUDA_OK(cudaSetDevice(h->st.device));
        const int64_t base = h->base;
        cudaStream_t s = h->stream;
        h->n = n; h->m = m; h->p = p;
        auto rebased = [&](const int64_t* src, int64_t len) {
            std::vector<int64_t> v(len);
            for (int64_t i = 0; i < len; ++i) v[i] = src[i] - base;
            return v;
        };
        CUDA_OK(h->d_mapP.upload(rebased(map_P, nnzP), s));
        CUDA_OK(h->d_mapA.upload(rebased(map_A, nnzA), s));
        std::vector<int64_t> mapHs = rebased(map_Hs, nHs);
        CUDA_OK(h->d_mapHs.upload(mapHs, s));
        CUDA_OK(h->d_diagidx.upload(rebased(map_diag_full, h->N), s));
        h->have_diag = true;
        // cone tables
        std::vector<int8_t> dg_kind; std::vector<int32_t> dg_midx, dg_cone; std::vector<int64_t> dg_map;
        std::vector<int32_t> sd_moff, sd_dim, sd_socid; std::vector<int64_t> sd_hoff;
        std::vector<int32_t> ex_src, ex_cone, exD_cone;
        std::vector<int32_t> psd_side; std::vector<int64_t> psd_roff, psd_hoff;
        int64_t moff = 0, hoff = 0, socrow = 0, roff = 0;
        int32_t socid = 0;
        h->psd_maxn = 0;
        for (int64_t i = 0; i < ncones; ++i) {
            const int t = cone_type[i];
            const int64_t d = cone_dim[i];
            if (t == 0 || t == 1) {
                for (int64_t k = 0; k < d; ++k) {
                    dg_kind.push_back((int8_t)t); dg_midx.push_back((int32_t)(moff + k));
                    dg_cone.push_back(0); dg_map.push_back(mapHs[hoff + k]);
                }
                moff += d; hoff += d;
            } else if (t == 2) {
                if (d > 4) {
                    for (int64_t k = 0; k < d; ++k) {
                        dg_kind.push_back(k == 0 ? 3 : 2); dg_midx.push_back((int32_t)(moff + k));
                        dg_cone.push_back(socid); dg_map.push_back(mapHs[hoff + k]);
                        ex_src.push_back((int32_t)(socrow + k)); ex_cone.push_back(socid);
                    }
                    exD_cone.push_back(socid);
                    hoff += d;
                } else {
                    sd_moff.push_back((int32_t)moff); sd_dim.push_back((int32_t)d);
                    sd_socid.push_back(socid); sd_hoff.push_back(hoff);
                    hoff += d * (d + 1) / 2;
                }
                moff += d; socrow += d; socid++;
            } else if (t == 3) {
                const int64_t ne = d * (d + 1) / 2;
                psd_side.push_back((int32_t)d); psd_roff.push_back(roff); psd_hoff.push_back(hoff);
                roff += d * d; hoff += ne * (ne + 1) / 2; moff += ne;
                h->psd_maxn = std::max<int32_t>(h->psd_maxn, (int32_t)d);
            } else if (t == 4 || t == 5) {
                // exponential / power cone: dense 3x3 block whose values the caller computes
                // (coneops_expcone.jl:92-100) and sends through cb200_update_values before
                // cb200_update_cones; no cone kernel touches these entries
                if (d != 3) { set_error("cb200_set_maps: exponential / power cones have dimension 3"); return -2; }
                moff += 3; hoff += 6;
            } else if (t == 6) {
                // generalised power cone: diagonal block + expansion columns, all sent by the
                // caller through cb200_update_values (coneops_genpowcone.jl:91-108,
                // directldl_datamaps.jl:146-166)
                moff += d; hoff += d;
            } else { set_error("cb200_set_maps: unsupported cone type"); return -2; }
        }
        if (moff != m || hoff != nHs) { set_error("cb200_set_maps: cone table inconsistent with m / nHs"); return -2; }
        h->ndiag = (int64_t)dg_kind.size();
        CUDA_OK(h->d_dg_kind.upload(dg_kind, s)); CUDA_OK(h->d_dg_midx.upload(dg_midx, s));
        CUDA_OK(h->d_dg_cone.upload(dg_cone, s)); CUDA_OK(h->d_dg_map.upload(dg_map, s));
        h->nsocd = (int32_t)sd_dim.size();
        CUDA_OK(h->d_sd_moff.upload(sd_moff, s)); CUDA_OK(h->d_sd_dim.upload(sd_dim, s));
        CUDA_OK(h->d_sd_socid.upload(sd_socid, s)); CUDA_OK(h->d_sd_hoff.upload(sd_hoff, s));
        h->nexp = (int64_t)ex_src.size(); h->nsocs = (int32_t)exD_cone.size();
        CUDA_OK(h->d_ex_src.upload(ex_src, s)); CUDA_OK(h->d_ex_cone.upload(ex_cone, s));
        CUDA_OK(h->d_exD_cone.upload(exD_cone, s));
        CUDA_OK(h->d_mapu.upload(rebased(map_soc_u, h->nexp), s));
        CUDA_OK(h->d_mapv.upload(rebased(map_soc_v, h->nexp), s));
        CUDA_OK(h->d_mapD.upload(rebased(map_soc_D, 2 * (int64_t)h->nsocs), s));
        h->npsd = (int32_t)psd_side.size(); h->psd_rtotal = roff;
        CUDA_OK(h->d_psd_side.upload(psd_side, s)); CUDA_OK(h->d_psd_roff.upload(psd_roff, s));
        CUDA_OK(h->d_psd_hoff.upload(psd_hoff, s));
        CUDA_OK(h->d_psd_R.alloc(std::max<int64_t>(1, roff))); CUDA_OK(h->d_psd_A.alloc(std::max<int64_t>(1, roff)));
        h->nsoc = socid; h->nsocrows = socrow;
        CUDA_OK(h->d_w.alloc(std::max<int64_t>(1, m)));
        CUDA_OK(h->d_eta.alloc(std::max<int64_t>(1, h->nsoc))); CUDA_OK(h->d_socd.alloc(std::max<int64_t>(1, h->nsoc)));
        CUDA_OK(h->d_socu.alloc(std::max<int64_t>(1, socrow))); CUDA_OK(h->d_socv.alloc(std::max<int64_t>(1, socrow)));
        CUDA_OK(h->d_rx.alloc(std::max<int64_t>(1, n))); CUDA_OK(h->d_rz.alloc(std::max<int64_t>(1, m)));
        h->h_ctype.assign(cone_type, cone_type + ncones); h->h_cdim.assign(cone_dim, cone_dim + ncones);
        h->scale_ready = false;
        CUDA_OK(cudaStreamSynchronize(s));
        h->maps_set = true;
        return 0;
    } catch (const std::exception& e) { set_error(e.what()); return -1; }
}

int32_t cb200_update_cones(cb200_handle* h, const double* w, const double* soc_eta,
                           const double* soc_d, const double* soc_u, const double* soc_v,
                           const double* psd_R) {
    if (!h->maps_set) { set_error("cb200_update_cones: cb200_set_maps not called"); return -2; }
    CUDA_OK(cudaSetDevice(h->st.device));
    cudaStream_t st = h->stream;
    h->tm.begin(Timers::CONE, st);
    // host pointers normally; in resident mode (cb200_set_resident) non-NULL arguments are DEVICE pointers
    // (inputs staged in HBM by the caller, copied device-to-device).  In both modes NULL keeps the state on the
    // device: what the previous call uploaded, or what cb200_update_scaling computed.
    const cudaMemcpyKind kind = h->resident ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    auto put = [&](double* dst, const double* src, int64_t len) -> cudaError_t {
        if (len <= 0 || !src) return cudaSuccess;
        return cudaMemcpyAsync(dst, src, len * sizeof(double), kind, st);
    };
    CUDA_OK(put(h->d_w.p, w, h->m));
    CUDA_OK(put(h->d_eta.p, soc_eta, h->nsoc)); CUDA_OK(put(h->d_socd.p, soc_d, h->nsoc));
    CUDA_OK(put(h->d_socu.p, soc_u, h->nsocrows)); CUDA_OK(put(h->d_socv.p, soc_v, h->nsocrows));
    CUDA_OK(put(h->d_psd_R.p, psd_R, h->psd_rtotal));
    if (h->ndiag) {
        k_hs_diag<<<nblk(h->ndiag, 256), 256, 0, st>>>(h->ndiag, h->d_dg_kind.p, h->d_dg_midx.p, h->d_dg_cone.p,
                                                       h->d_dg_map.p, h->d_w.p, h->d_eta.p, h->d_socd.p, h->d_nz.p);
        LAUNCH(h);
    }
    if (h->nsocd) {
        k_hs_soc_dense<<<nblk(h->nsocd, 128), 128, 0, st>>>(h->nsocd, h->d_sd_moff.p, h->d_sd_dim.p, h->d_sd_socid.p,
                                                            h->d_sd_hoff.p, h->d_mapHs.p, h->d_w.p, h->d_eta.p, h->d_nz.p);
        LAUNCH(h);
    }
    if (h->nexp) {
        k_soc_expansion<<<nblk(h->nexp, 256), 256, 0, st>>>(h->nexp, h->d_ex_src.p, h->d_ex_cone.p, h->d_mapu.p,
                                                            h->d_mapv.p, h->d_socu.p, h->d_socv.p, h->d_eta.p, h->d_nz.p);
        k_soc_D<<<nblk(h->nsocs, 128), 128, 0, st>>>(h->nsocs, h->d_exD_cone.p, h->d_mapD.p, h->d_eta.p, h->d_nz.p);
        h->tm.nlaunch += 2;
    }
    if (h->npsd) {
        k_psd_rrt<<<h->npsd, 256, 0, st>>>(h->d_psd_side.p, h->d_psd_roff.p, h->d_psd_R.p, h->d_psd_A.p);
        const int ne = h->psd_maxn * (h->psd_maxn + 1) / 2;
        k_psd_skron<<<dim3(std::max(1, std::min(64, nblk(ne, 8))), h->npsd), 256, 0, st>>>(
            h->d_psd_side.p, h->d_psd_roff.p, h->d_psd_hoff.p, h->d_psd_A.p, h->d_mapHs.p, h->d_nz.p);
        h->tm.nlaunch += 2;
    }
    h->tm.end(st);
    CUDA_OK(cudaGetLastError());
    int rc = factor(h, /*static_reg=*/true);
    if (rc) return rc;
    return finish_factor(h);
}

// G10 tables and output buffers, built by the first cb200_update_scaling / cb200_get_scaling from the cone table of
// cb200_set_maps, so that a caller that keeps the host scaling pays no memory for them.
static int prepare_scaling(cb200_handle* h) {
    if (h->scale_ready) return 0;
    int optin = 0;
    CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->st.device));
    cudaFuncAttributes fa;
    CUDA_OK(cudaFuncGetAttributes(&fa, k_scale_psd<true>));
    const int64_t dyn_cap = (int64_t)optin - (int64_t)fa.sharedSizeBytes;      // side <= 83 on an H100 (227 KB)
    std::vector<int32_t> nn_rows, soc_warp, soc_cta, soc_dim, psd_smem, psd_glob;
    std::vector<int64_t> soc_moff, soc_srow, psd_moff, psd_loff, psd_woff;
    int64_t moff = 0, srow = 0, loff = 0, wtot = 0, max_smem_side = 0;
    int32_t socid = 0, psdid = 0;
    for (size_t i = 0; i < h->h_ctype.size(); ++i) {
        const int t = h->h_ctype[i];
        const int64_t d = h->h_cdim[i];
        if (t == 1) {
            for (int64_t k = 0; k < d; ++k) nn_rows.push_back((int32_t)(moff + k));
        } else if (t == 2) {
            (d >= SOC_CTA_MIN_DIM ? soc_cta : soc_warp).push_back(socid++);
            soc_dim.push_back((int32_t)d); soc_moff.push_back(moff); soc_srow.push_back(srow);
            srow += d;
        } else if (t == 3) {
            if (32 * d * d <= dyn_cap) { psd_smem.push_back(psdid); max_smem_side = std::max(max_smem_side, d); }
            else { psd_glob.push_back(psdid); psd_woff.push_back(wtot); wtot += 4 * d * d; }
            psd_moff.push_back(moff); psd_loff.push_back(loff);
            loff += d; psdid++;
        }
        moff += t == 3 ? d * (d + 1) / 2 : d;
    }
    cudaStream_t s = h->stream;
    h->nnn = (int64_t)nn_rows.size();
    h->nsoc_warp = (int32_t)soc_warp.size(); h->nsoc_cta = (int32_t)soc_cta.size();
    h->npsd_smem = (int32_t)psd_smem.size(); h->npsd_glob = (int32_t)psd_glob.size();
    h->psd_ltotal = loff;
    soc_warp.insert(soc_warp.end(), soc_cta.begin(), soc_cta.end());
    psd_smem.insert(psd_smem.end(), psd_glob.begin(), psd_glob.end());
    CUDA_OK(h->d_nn_rows.upload(nn_rows, s));
    CUDA_OK(h->d_soc_list.upload(soc_warp, s)); CUDA_OK(h->d_soc_dim.upload(soc_dim, s));
    CUDA_OK(h->d_soc_moff.upload(soc_moff, s)); CUDA_OK(h->d_soc_srow.upload(soc_srow, s));
    CUDA_OK(h->d_psd_list.upload(psd_smem, s)); CUDA_OK(h->d_psd_moff.upload(psd_moff, s));
    CUDA_OK(h->d_psd_loff.upload(psd_loff, s)); CUDA_OK(h->d_psd_woff.upload(psd_woff, s));
    const int64_t m1 = std::max<int64_t>(1, h->m);
    CUDA_OK(h->d_lam.alloc(m1)); CUDA_OK(h->d_ss.alloc(m1)); CUDA_OK(h->d_sz.alloc(m1));
    CUDA_OK(h->d_psd_Rinv.alloc(std::max<int64_t>(1, h->psd_rtotal)));
    CUDA_OK(h->d_psd_lam.alloc(std::max<int64_t>(1, loff)));
    CUDA_OK(h->d_psd_ws.alloc(std::max<int64_t>(1, wtot), /*fill=*/false));
    CUDA_OK(h->d_scale_flags.alloc(2));
    h->psd_smem_bytes = (size_t)(32 * max_smem_side * max_smem_side);     // four n x n FP64 matrices
    if (max_smem_side)
        CUDA_OK(cudaFuncSetAttribute(k_scale_psd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)h->psd_smem_bytes));
    for (cudaEvent_t& e : h->ev_scale) if (!e) CUDA_OK(cudaEventCreate(&e));
    CUDA_OK(cudaStreamSynchronize(s));
    h->scale_ready = true;
    return 0;
}

int32_t cb200_update_scaling(cb200_handle* h, const double* s, const double* z, int32_t* ok_scale) {
    if (!h->maps_set) { set_error("cb200_update_scaling: cb200_set_maps not called"); return -2; }
    for (int32_t t : h->h_ctype)
        if (t >= 4) {
            set_error("cb200_update_scaling: exponential, power and generalised power cones keep their host scaling");
            return -2;
        }
    if ((!s || !z) && h->m) { set_error("cb200_update_scaling: s and z are required"); return -2; }
    try {
        CUDA_OK(cudaSetDevice(h->st.device));
        int rc = prepare_scaling(h);
        if (rc) return rc;
        cudaStream_t st = h->stream;
        const int64_t m = h->m;
        // host pointers normally, device pointers in resident mode (read in place)
        const double* ds = s;
        const double* dz = z;
        if (!h->resident && m) {
            CUDA_OK(cudaMemcpyAsync(h->d_ss.p, s, m * sizeof(double), cudaMemcpyHostToDevice, st));
            CUDA_OK(cudaMemcpyAsync(h->d_sz.p, z, m * sizeof(double), cudaMemcpyHostToDevice, st));
            ds = h->d_ss.p; dz = h->d_sz.p;
        }
        CUDA_OK(cudaEventRecord(h->ev_scale[0], st));
        CUDA_OK(cudaMemsetAsync(h->d_scale_flags.p, 0, 2 * sizeof(int), st));
        int* fl = h->d_scale_flags.p;
        if (h->nnn) {
            k_scale_nn<<<nblk(h->nnn, SCALE_THREADS), SCALE_THREADS, 0, st>>>(h->nnn, h->d_nn_rows.p, ds, dz, h->d_w.p,
                                                                             h->d_lam.p);
            LAUNCH(h);
        }
        if (h->nsoc_warp) {
            k_scale_soc<32><<<nblk(h->nsoc_warp, SCALE_THREADS / 32), SCALE_THREADS, 0, st>>>(
                h->nsoc_warp, h->d_soc_list.p, h->d_soc_moff.p, h->d_soc_dim.p, h->d_soc_srow.p, ds, dz, h->d_w.p,
                h->d_lam.p, h->d_eta.p, h->d_socd.p, h->d_socu.p, h->d_socv.p, fl);
            LAUNCH(h);
        }
        if (h->nsoc_cta) {
            k_scale_soc<SCALE_THREADS><<<h->nsoc_cta, SCALE_THREADS, 0, st>>>(
                h->nsoc_cta, h->d_soc_list.p + h->nsoc_warp, h->d_soc_moff.p, h->d_soc_dim.p, h->d_soc_srow.p, ds, dz,
                h->d_w.p, h->d_lam.p, h->d_eta.p, h->d_socd.p, h->d_socu.p, h->d_socv.p, fl);
            LAUNCH(h);
        }
        constexpr int kMaxSweeps = 30;
        if (h->npsd_smem) {
            k_scale_psd<true><<<h->npsd_smem, SCALE_THREADS, h->psd_smem_bytes, st>>>(
                h->d_psd_list.p, h->d_psd_side.p, h->d_psd_moff.p, h->d_psd_roff.p, h->d_psd_loff.p, nullptr, ds, dz,
                nullptr, h->d_psd_R.p, h->d_psd_Rinv.p, h->d_psd_lam.p, fl, kMaxSweeps);
            LAUNCH(h);
        }
        if (h->npsd_glob) {
            k_scale_psd<false><<<h->npsd_glob, SCALE_THREADS, 0, st>>>(
                h->d_psd_list.p + h->npsd_smem, h->d_psd_side.p, h->d_psd_moff.p, h->d_psd_roff.p, h->d_psd_loff.p,
                h->d_psd_woff.p, ds, dz, h->d_psd_ws.p, h->d_psd_R.p, h->d_psd_Rinv.p, h->d_psd_lam.p, fl, kMaxSweeps);
            LAUNCH(h);
        }
        CUDA_OK(cudaEventRecord(h->ev_scale[1], st));
        CUDA_OK(cudaGetLastError());
        int flags[2] = {0, 0};
        CUDA_OK(cudaMemcpyAsync(flags, fl, sizeof(flags), cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        float ms = 0.f;
        CUDA_OK(cudaEventElapsedTime(&ms, h->ev_scale[0], h->ev_scale[1]));
        h->scale_ms += ms;
        h->last_sweeps = flags[1];
        if (ok_scale) *ok_scale = flags[0] ? 0 : 1;
        return 0;
    } catch (const std::exception& e) { set_error(e.what()); return -1; }
}

int32_t cb200_get_scaling(cb200_handle* h, double* w, double* lam, double* eta, double* d, double* u, double* v,
                          double* R, double* Rinv, double* psd_lam) {
    if (!h->maps_set) { set_error("cb200_get_scaling: cb200_set_maps not called"); return -2; }
    try {
        CUDA_OK(cudaSetDevice(h->st.device));
        int rc = prepare_scaling(h);
        if (rc) return rc;
        cudaStream_t st = h->stream;
        auto get = [&](double* dst, const double* src, int64_t len) -> cudaError_t {
            if (!dst || len <= 0) return cudaSuccess;
            return cudaMemcpyAsync(dst, src, len * sizeof(double), cudaMemcpyDeviceToHost, st);
        };
        CUDA_OK(get(w, h->d_w.p, h->m)); CUDA_OK(get(lam, h->d_lam.p, h->m));
        CUDA_OK(get(eta, h->d_eta.p, h->nsoc)); CUDA_OK(get(d, h->d_socd.p, h->nsoc));
        CUDA_OK(get(u, h->d_socu.p, h->nsocrows)); CUDA_OK(get(v, h->d_socv.p, h->nsocrows));
        CUDA_OK(get(R, h->d_psd_R.p, h->psd_rtotal)); CUDA_OK(get(Rinv, h->d_psd_Rinv.p, h->psd_rtotal));
        CUDA_OK(get(psd_lam, h->d_psd_lam.p, h->psd_ltotal));
        CUDA_OK(cudaStreamSynchronize(st));
        return 0;
    } catch (const std::exception& e) { set_error(e.what()); return -1; }
}

int32_t cb200_setrhs(cb200_handle* h, const double* rhsx, const double* rhsz) {
    if (!h->maps_set) { set_error("cb200_setrhs: cb200_set_maps not called"); return -2; }
    CUDA_OK(cudaSetDevice(h->st.device));
    cudaStream_t st = h->stream;
    // resident mode: non-NULL arguments are device pointers (see cb200_update_cones), stream-ordered copy
    const cudaMemcpyKind kind = h->resident ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (h->n && rhsx) CUDA_OK(cudaMemcpyAsync(h->d_rx.p, rhsx, h->n * sizeof(double), kind, st));
    if (h->m && rhsz) CUDA_OK(cudaMemcpyAsync(h->d_rz.p, rhsz, h->m * sizeof(double), kind, st));
    if (!h->resident) CUDA_OK(cudaStreamSynchronize(st));        // the caller may overwrite its buffers on return
    return 0;
}

int32_t cb200_solve_ir(cb200_handle* h, const double* rhsx, const double* rhsz,
                       double* lhsx, double* lhsz, int32_t* ir_rounds) {
    if (!h->maps_set) { set_error("cb200_solve_ir: cb200_set_maps not called"); return -2; }
    CUDA_OK(cudaSetDevice(h->st.device));
    cudaStream_t st = h->stream;
    const int64_t N = h->N, n = h->n, m = h->m;
    if (ir_rounds) *ir_rounds = 0;
    if (N == 0) return 0;
    if (!h->resident) {      // each part is optional on its own (a NULL part keeps what cb200_setrhs stored)
        if (n && rhsx) CUDA_OK(cudaMemcpyAsync(h->d_rx.p, rhsx, n * sizeof(double), cudaMemcpyHostToDevice, st));
        if (m && rhsz) CUDA_OK(cudaMemcpyAsync(h->d_rz.p, rhsz, m * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    k_build_rhs<<<nblk(N, 256), 256, 0, st>>>(h->d_rx.p, h->d_rz.p, n, m, N, h->d_b.p);
    CUDA_OK(cudaMemsetAsync(h->d_scal.p + 1, 0, sizeof(unsigned long long), st));
    k_absmax<<<std::min(nblk(N, 256), h->reduce_blocks), 256, 0, st>>>(h->d_b.p, N, h->d_scal.p + 1);
    h->tm.nlaunch += 2;
    double* x = h->d_x.p; double* dx = h->d_dx.p; double* e = h->d_e.p;
    int rc = reset_chain_error(h); if (rc) return rc;
    rc = tri_solve(h, h->d_b.p, x);
    if (rc) return rc;
    int ok = 1;
    if (h->st.iterative_refinement_enable) {
        // _iterative_refinement (kktsolver_directldl.jl:389-449)
        rc = residual(h, x, e, 2); if (rc) return rc;
        double sc[2];
        rc = read_scalars(h, sc, 1, 2); if (rc) return rc;
        const double normb = sc[0];
        double norme = sc[1];
        if (!std::isfinite(norme)) ok = 0;
        for (int i = 0; ok && i < h->st.iterative_refinement_max_iter; ++i) {
            if (norme <= h->st.iterative_refinement_abstol + h->st.iterative_refinement_reltol * normb) break;
            const double lastnorme = norme;
            rc = tri_solve(h, e, dx); if (rc) return rc;
            k_axpy1<<<nblk(N, 256), 256, 0, st>>>(dx, x, N); LAUNCH(h);
            rc = residual(h, dx, e, 2); if (rc) return rc;
            rc = read_scalars(h, sc, 2, 1); if (rc) return rc;
            norme = sc[0];
            if (ir_rounds) (*ir_rounds)++;
            if (!std::isfinite(norme)) { ok = 0; break; }
            const double ratio = lastnorme / norme;
            if (ratio < h->st.iterative_refinement_stop_ratio) {
                if (ratio > 1.0) std::swap(x, dx);
                break;
            }
            std::swap(x, dx);
        }
    } else {
        CUDA_OK(cudaMemsetAsync(h->d_scal.p + 2, 0, sizeof(unsigned long long), st));
        k_absmax<<<std::min(nblk(N, 256), h->reduce_blocks), 256, 0, st>>>(x, N, h->d_scal.p + 2); LAUNCH(h);
        double sc[1];
        rc = read_scalars(h, sc, 2, 1); if (rc) return rc;
        ok = std::isfinite(sc[0]);
    }
    // keep handle buffers consistent with the pointer swaps (kktsolver_directldl.jl:445)
    if (x != h->d_x.p) std::swap(h->d_x.p, h->d_dx.p);
    if (ok && !h->resident) {
        if (lhsx && n) CUDA_OK(cudaMemcpyAsync(lhsx, h->d_x.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (lhsz && m) CUDA_OK(cudaMemcpyAsync(lhsz, h->d_x.p + n, m * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    unsigned chain_err = 0;
    rc = read_chain_error(h, &chain_err); if (rc) return rc;
    CUDA_OK(cudaStreamSynchronize(st));
    h->tm.collect();
    if (chain_err) { set_error("cb200_solve_ir: a big-front solve chain timed out waiting for a block"); ok = 0; }
    if (!ok && !h->resident) {
        // a failed solve must not leave stale finite values in the caller's vectors: the reference
        // checks all(isfinite, x) on them when refinement is disabled (kktsolver_directldl.jl:356-370)
        const double qnan = std::numeric_limits<double>::quiet_NaN();
        if (lhsx) std::fill(lhsx, lhsx + n, qnan);
        if (lhsz) std::fill(lhsz, lhsz + m, qnan);
    }
    return ok ? 0 : 1;
}

int32_t cb200_solve_multi(cb200_handle* h, int32_t nrhs, double* X, int64_t ldx, const double* B, int64_t ldb) {
    const int64_t N = h->N;
    if (nrhs < 0) { set_error("cb200_solve_multi: nrhs < 0"); return -2; }
    if (nrhs == 0) return 0;
    if (!X || !B) { set_error("cb200_solve_multi: X or B is NULL"); return -2; }
    if (ldx < N || ldb < N) { set_error("cb200_solve_multi: leading dimension < N"); return -2; }
    if (N == 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    int rc = ensure_multi(h); if (rc) return rc;
    cudaStream_t st = h->stream;
    if (h->dist || h->use_subtree) {
        // column by column through cb200_solve (multi-GPU sweeps and the subtree kernels have no R-wide
        // form); the last single solve (download selector 6) is kept
        CUDA_OK(cudaMemcpyAsync(h->d_me.p, h->d_x.p, N * sizeof(double), cudaMemcpyDeviceToDevice, st));
        for (int32_t j = 0; j < nrhs && rc == 0; ++j) {
            rc = cb200_solve(h, X + j * ldx, B + j * ldb);
            h->n_percol += 1;
        }
        // put the last single solution back on every path, failed calls included
        const cudaError_t e = cudaMemcpyAsync(h->d_x.p, h->d_me.p, N * sizeof(double), cudaMemcpyDeviceToDevice, st);
        if (rc) return rc;
        CUDA_OK(e);
        CUDA_OK(cudaStreamSynchronize(st));
        return 0;
    }
    rc = reset_chain_error(h); if (rc) return rc;
    for (int32_t c0 = 0; c0 < nrhs;) {
        const int R = chunk_width(h->multi_w, nrhs - c0), k = std::min(R, nrhs - c0);
        CUDA_OK(cudaMemcpy2DAsync(h->d_mstage.p, N * sizeof(double), B + c0 * ldb, ldb * sizeof(double),
                                  N * sizeof(double), k, cudaMemcpyHostToDevice, st));
        rc = tri_solve_multi(h, R, k, h->d_mstage.p, 1, N, h->d_mstage.p, 1, N); if (rc) return rc;
        CUDA_OK(cudaMemcpy2DAsync(X + c0 * ldx, ldx * sizeof(double), h->d_mstage.p, N * sizeof(double),
                                  N * sizeof(double), k, cudaMemcpyDeviceToHost, st));
        c0 += k;
    }
    unsigned chain_err = 0;
    rc = read_chain_error(h, &chain_err); if (rc) return rc;
    CUDA_OK(cudaStreamSynchronize(st));
    h->tm.collect();
    if (chain_err) { set_error("cb200_solve_multi: a big-front solve chain timed out waiting for a block"); return -4; }
    return 0;
}

int32_t cb200_solve_ir_multi(cb200_handle* h, int32_t nrhs, const double* rhsx, const double* rhsz,
                             double* lhsx, double* lhsz, int32_t* ir_rounds, int32_t* status) {
    if (!h->maps_set) { set_error("cb200_solve_ir_multi: cb200_set_maps not called"); return -2; }
    if (nrhs < 0) { set_error("cb200_solve_ir_multi: nrhs < 0"); return -2; }
    if (nrhs == 0) return 0;
    const int64_t N = h->N, n = h->n, m = h->m;
    if ((n && !rhsx) || (m && !rhsz)) { set_error("cb200_solve_ir_multi: rhsx or rhsz is NULL"); return -2; }
    for (int32_t j = 0; j < nrhs; ++j) { if (ir_rounds) ir_rounds[j] = 0; if (status) status[j] = 0; }
    if (N == 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    int rc = ensure_multi(h); if (rc) return rc;
    cudaStream_t st = h->stream;
    if ((int64_t)h->d_msol.n < N * nrhs) CUDA_OK(h->d_msol.alloc((size_t)(N * nrhs)));
    h->msol_cols = nrhs;
    std::vector<int32_t> rounds(nrhs, 0), okv(nrhs, 1);
    if (h->dist || h->use_subtree) {
        // column by column through cb200_solve_ir; what cb200_setrhs stored and the last single solution
        // (download selector 6) are put back afterwards
        CUDA_OK(cudaMemcpyAsync(h->d_me.p, h->d_x.p, N * sizeof(double), cudaMemcpyDeviceToDevice, st));
        if (n) CUDA_OK(cudaMemcpyAsync(h->d_mdx.p, h->d_rx.p, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
        if (m) CUDA_OK(cudaMemcpyAsync(h->d_mdx.p + n, h->d_rz.p, m * sizeof(double), cudaMemcpyDeviceToDevice, st));
        for (int32_t j = 0; j < nrhs && rc >= 0; ++j) {
            if (h->resident) {
                if (n) CUDA_OK(cudaMemcpyAsync(h->d_rx.p, rhsx + j * n, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
                if (m) CUDA_OK(cudaMemcpyAsync(h->d_rz.p, rhsz + j * m, m * sizeof(double), cudaMemcpyDeviceToDevice, st));
                rc = cb200_solve_ir(h, nullptr, nullptr, nullptr, nullptr, &rounds[j]);
            } else {
                rc = cb200_solve_ir(h, n ? rhsx + j * n : nullptr, m ? rhsz + j * m : nullptr,
                                    lhsx ? lhsx + j * n : nullptr, lhsz ? lhsz + j * m : nullptr, &rounds[j]);
            }
            if (rc < 0) break;
            okv[j] = rc == 0;
            CUDA_OK(cudaMemcpyAsync(h->d_msol.p + j * N, h->d_x.p, N * sizeof(double), cudaMemcpyDeviceToDevice, st));
            h->n_percol += 1;
        }
        // restore the single-RHS state on every path, failed calls included
        cudaError_t e = cudaMemcpyAsync(h->d_x.p, h->d_me.p, N * sizeof(double), cudaMemcpyDeviceToDevice, st);
        if (n && e == cudaSuccess) e = cudaMemcpyAsync(h->d_rx.p, h->d_mdx.p, n * sizeof(double), cudaMemcpyDeviceToDevice, st);
        if (m && e == cudaSuccess) e = cudaMemcpyAsync(h->d_rz.p, h->d_mdx.p + n, m * sizeof(double), cudaMemcpyDeviceToDevice, st);
        if (rc < 0) return rc;
        CUDA_OK(e);
        CUDA_OK(cudaStreamSynchronize(st));
    } else {
        const int w = h->multi_w;
        if (!h->resident) {
            if ((int64_t)h->d_mrx.n < std::max<int64_t>(1, n) * w) CUDA_OK(h->d_mrx.alloc((size_t)std::max<int64_t>(1, n) * w));
            if ((int64_t)h->d_mrz.n < std::max<int64_t>(1, m) * w) CUDA_OK(h->d_mrz.alloc((size_t)std::max<int64_t>(1, m) * w));
        }
        rc = reset_chain_error(h); if (rc) return rc;
        for (int32_t c0 = 0; c0 < nrhs;) {
            const int R = chunk_width(w, nrhs - c0), k = std::min(R, nrhs - c0);
            const double* rx = rhsx ? rhsx + c0 * n : nullptr;
            const double* rz = rhsz ? rhsz + c0 * m : nullptr;
            if (!h->resident) {         // host columns -> device staging (the caller may reuse them on return)
                if (n) CUDA_OK(cudaMemcpyAsync(h->d_mrx.p, rx, k * n * sizeof(double), cudaMemcpyHostToDevice, st));
                if (m) CUDA_OK(cudaMemcpyAsync(h->d_mrz.p, rz, k * m * sizeof(double), cudaMemcpyHostToDevice, st));
                rx = h->d_mrx.p; rz = h->d_mrz.p;
            }
            k_build_rhs_multi<<<nblk(N * R, 256), 256, 0, st>>>(rx, rz, n, m, N, k, R, h->d_mb.p); LAUNCH(h);
            rc = solve_ir_chunk(h, R, k, rounds.data() + c0, okv.data() + c0); if (rc) return rc;
            k_deinterleave<<<nblk(N * R, 256), 256, 0, st>>>(h->d_mx.p, k, R, N, h->d_msol.p + c0 * N, N); LAUNCH(h);
            c0 += k;
        }
        if (!h->resident) {
            if (lhsx && n) CUDA_OK(cudaMemcpy2DAsync(lhsx, n * sizeof(double), h->d_msol.p, N * sizeof(double),
                                                     n * sizeof(double), nrhs, cudaMemcpyDeviceToHost, st));
            if (lhsz && m) CUDA_OK(cudaMemcpy2DAsync(lhsz, m * sizeof(double), h->d_msol.p + n, N * sizeof(double),
                                                     m * sizeof(double), nrhs, cudaMemcpyDeviceToHost, st));
        }
        unsigned chain_err = 0;
        rc = read_chain_error(h, &chain_err); if (rc) return rc;
        CUDA_OK(cudaStreamSynchronize(st));
        h->tm.collect();
        if (chain_err) {
            set_error("cb200_solve_ir_multi: a big-front solve chain timed out waiting for a block");
            std::fill(okv.begin(), okv.end(), 0);
        }
        if (!h->resident) {            // failed columns are NaN-filled, as cb200_solve_ir does
            const double qnan = std::numeric_limits<double>::quiet_NaN();
            for (int32_t j = 0; j < nrhs; ++j) {
                if (okv[j]) continue;
                if (lhsx) std::fill(lhsx + j * n, lhsx + (j + 1) * n, qnan);
                if (lhsz) std::fill(lhsz + j * m, lhsz + (j + 1) * m, qnan);
            }
        }
    }
    bool all_ok = true;
    for (int32_t j = 0; j < nrhs; ++j) {
        if (ir_rounds) ir_rounds[j] = rounds[j];
        if (status) status[j] = okv[j] ? 0 : 1;
        all_ok &= okv[j] != 0;
    }
    return all_ok ? 0 : 1;
}

static int32_t update_block(cb200_handle* h, const DevBuf<int64_t>& map, const double* values, int64_t len) {
    if (!h->maps_set) { set_error("cb200_update_P/A: cb200_set_maps not called"); return -2; }
    if ((int64_t)map.n != len) { set_error("cb200_update_P/A: length mismatch"); return -2; }
    if (len == 0) return 0;
    CUDA_OK(cudaSetDevice(h->st.device));
    { int rc = stage_reserve(h, 0, (size_t)len); if (rc) return rc; }
    CUDA_OK(cudaMemcpyAsync(h->d_stage_val.p, values, len * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    k_update_values<<<nblk(len, 256), 256, 0, h->stream>>>(h->d_nz.p, map.p, h->d_stage_val.p, len, 0);
    LAUNCH(h);
    CUDA_OK(cudaGetLastError());
    if (host_is_pinned(values)) CUDA_OK(cudaStreamSynchronize(h->stream));
    return 0;
}
int32_t cb200_update_P(cb200_handle* h, const double* values, int64_t len) { return update_block(h, h->d_mapP, values, len); }
int32_t cb200_update_A(cb200_handle* h, const double* values, int64_t len) { return update_block(h, h->d_mapA, values, len); }

int32_t cb200_download(cb200_handle* h, int32_t what, double* out, int64_t len) {
    CUDA_OK(cudaSetDevice(h->st.device));
    cudaStream_t st = h->stream;
    const double* src = nullptr; int64_t n = 0;
    switch (what) {
        case 0: src = h->d_nz.p; n = h->nnzK; break;
        case 1: src = h->d_D.p; n = h->N; break;
        case 2: src = h->d_L.p; n = (int64_t)h->d_L.n; break;
        case 3: { if (len != h->N) { set_error("download: length"); return -2; }
                  for (int64_t i = 0; i < len; ++i) out[i] = (double)h->S.perm[i]; return 0; }
        case 4: src = h->d_eps.p; n = 1; break;
        case 5: { if (len != 1) { set_error("download: length"); return -2; }
                  unsigned int v = 0;
                  CUDA_OK(cudaMemcpyAsync(&v, h->d_nreg.p, sizeof(v), cudaMemcpyDeviceToHost, st));
                  CUDA_OK(cudaStreamSynchronize(st)); out[0] = (double)v; return 0; }
        case 6: src = h->d_x.p; n = h->N; break;       // full solution [x; z; expansion variables] of the last solve
        case 8: src = h->d_msol.p; n = h->N * h->msol_cols; break;   // the same, N x nrhs, of the last cb200_solve_ir_multi
        case 9: src = h->d_e.p; n = h->N; break;       // residual b - K x last computed by cb200_solve_ir
        case 7: { if (len != 64) { set_error("download: length"); return -2; }     // ORIGINAL indices of the first 64 regularised pivots
                  int32_t v[64]; unsigned int cnt = 0;
                  CUDA_OK(cudaMemcpyAsync(v, h->d_reglog.p, sizeof(v), cudaMemcpyDeviceToHost, st));
                  CUDA_OK(cudaMemcpyAsync(&cnt, h->d_nreg.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
                  CUDA_OK(cudaStreamSynchronize(st));
                  for (int i = 0; i < 64; ++i) out[i] = i < (int)cnt ? (double)h->S.perm[v[i]] : -1.0;
                  return 0; }
        default: set_error("download: bad selector"); return -2;
    }
    if (len != n) { set_error("download: length mismatch"); return -2; }
    if (n) CUDA_OK(cudaMemcpyAsync(out, src, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

int32_t cb200_get_timers(cb200_handle* h, double* out, int32_t len) {
    double v[12] = {h->tm.ms[0], h->tm.ms[1], h->tm.ms[2], h->tm.ms[3], h->tm.nfactor, h->tm.nsolve, h->tm.nlaunch,
                    h->tm.ms[4], h->tm.ms[5], h->tm.ms[6], h->tm.ms[7], h->scale_ms};
    for (int i = 0; i < len && i < 12; ++i) out[i] = v[i];
    return 0;
}
int32_t cb200_nccl_unique_id(char out[128]) {
    if (!g_nccl.load()) { set_error("NCCL library not found (dlopen libnccl.so.2)"); return -5; }
    ncclUniqueId id;
    NCCL_OK(g_nccl.GetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId size");
    std::memcpy(out, &id, 128);
    return 0;
}

int32_t cb200_dist_init(cb200_handle* h, int32_t rank, int32_t nranks, const char uid[128]) {
    try {
        if (nranks <= 1) return 0;
        if (!g_nccl.load()) { set_error("NCCL library not found (dlopen libnccl.so.2)"); return -5; }
        CUDA_OK(cudaSetDevice(h->st.device));
        ncclUniqueId id; std::memcpy(&id, uid, 128);
        NCCL_OK(g_nccl.CommInitRank(&h->comm, nranks, id, rank));
        h->rank = rank; h->nranks = nranks; h->dist = true;
        const Symbolic& S = h->S;
        partition_subtrees(S, nranks, h->owner, h->is_top);
        h->h_top_list.clear(); h->h_top_by_level.assign(S.nlevels, {});
        for (int lv = 0; lv < S.nlevels; ++lv)
            for (int32_t q = S.level_ptr[lv]; q < S.level_ptr[lv + 1]; ++q) {
                const int32_t sn = S.level_list[q];
                if (h->is_top[sn]) { h->h_top_list.push_back(sn); h->h_top_by_level[lv].push_back(sn); }
            }
        std::vector<int8_t> active(S.nsuper), keep(S.N), topkeep(S.N);
        for (int32_t sn = 0; sn < S.nsuper; ++sn) {
            const bool top = h->is_top[sn];
            active[sn] = top ? (rank == 0) : (h->owner[sn] == rank);
            const int8_t kc = top ? (rank == 0) : (h->owner[sn] == rank);
            for (int32_t j = S.sn_first[sn]; j < S.sn_first[sn + 1]; ++j) {
                keep[j] = kc;
                topkeep[j] = top ? (rank == 0) : 1;
            }
        }
        cudaStream_t s = h->stream;
        CUDA_OK(h->d_active.upload(active, s)); CUDA_OK(h->d_keepcol.upload(keep, s));
        h->h_active = active;
        CUDA_OK(h->d_topcolkeep.upload(topkeep, s)); CUDA_OK(h->d_top_list.upload(h->h_top_list, s));
        // update blocks of supernodes other ranks own are never written here: keep them zero
        CUDA_OK(cudaMemsetAsync(h->d_U.p, 0, h->d_U.n * sizeof(double), s));
        int rc = build_plans(h);
        if (!rc) rc = upload_tile_lists(h);
        if (rc) return rc;
        // the captured launch sequences (if any) belong to the single-GPU plans
        for (GraphExec* g : {&h->g_factor[0], &h->g_factor[1], &h->g_solve, &h->g_msolve[0], &h->g_msolve[1]}) {
            if (g->exec) { cudaGraphExecDestroy(g->exec); g->exec = nullptr; }
            g->failed = false;
        }
        const char* env = getenv("CB200_DIST_GRAPH");
        if (!(env && env[0] == '1')) h->st.use_cuda_graph = 0;   // NCCL inside stream capture: opt-in
        CUDA_OK(cudaStreamSynchronize(s));
        return 0;
    } catch (const std::exception& e) { set_error(e.what()); return -1; }
}

int32_t cb200_set_detail(cb200_handle* h, int32_t level) { h->detail = level < 0 ? 0 : (level > 2 ? 2 : level); return 0; }

static const char* const kFineNames[Timers::NFINE] = {
    "factor_small_nf16", "factor_small_nf32", "factor_small_nf64", "factor_small_nf96", "factor_small_nf128",
    "factor_small_nf152", "factor_panel_c0", "factor_panel_c1", "factor_panel_c2", "factor_panel_c3",
    "zero_update_blocks", "assemble_large", "piv_diag", "piv_rows", "schur_gemm", "finish_large", "factor_prologue",
    "fwd_leaf", "fwd_sub", "fwd_warp", "fwd_cta", "fwd_big_assemble", "fwd_big_tri", "fwd_big_gemv",
    "bwd_leaf", "bwd_sub", "bwd_warp", "bwd_cta", "bwd_big_gemvT", "bwd_big_tri", "permute_vectors", "nccl",
    "panel_update"};

int32_t cb200_get_fine_timers(cb200_handle* h, double* out_ms, int32_t len) {
    for (int i = 0; i < len && i < Timers::NFINE; ++i) out_ms[i] = h->tm.ms[Timers::NCOARSE + i];
    return Timers::NFINE;
}
const char* cb200_fine_timer_name(int32_t i) { return (i >= 0 && i < Timers::NFINE) ? kFineNames[i] : ""; }

int32_t cb200_get_stats(const cb200_handle* h, double* out, int32_t len) {
    const Symbolic& S = h->S;
    double schur = 0, panel_large = 0, big_bytes = 0, nlarge = 0;
    double my_flops = 0;
    for (int32_t sn = 0; sn < S.nsuper; ++sn) {
        const double ns = S.ns(sn), nr = S.nr(sn), nf = ns + nr;
        // multi-GPU: only the fronts THIS rank factors (its own subtrees + the replicated top)
        if (h->dist && !h->is_top[sn] && h->owner[sn] != h->rank) continue;
        for (double k = 0; k < ns; ++k) my_flops += (nf - k) * (nf - k);
        if (h->to_large((int)nf, (int)ns)) {
            nlarge += 1;
            schur += nr * (nr + 1.0) * ns;                 // flops of F22 -= L21 D L21' (lower part)
            for (double k = 0; k < ns; ++k) panel_large += (nf - k) * (nf - k);
        }
        if (nf * ns >= 65536 && ns > 32) big_bytes += 8.0 * nf * ns;
    }
    double v[26] = {S.flops, schur, panel_large - schur, (double)S.nnzL, (double)S.nlevels, (double)S.nsuper,
                    nlarge, big_bytes, (double)S.upd_total * 8.0, (double)S.panel_off.back() * 8.0,
                    (double)S.ordering_used, my_flops, h->use_tma ? 1.0 : 0.0, (double)h->tma_kmajor,
                    (double)((h->g_factor[0].exec != nullptr) + (h->g_factor[1].exec != nullptr)),
                    h->g_solve.exec ? 1.0 : 0.0, (double)h->nsub,
                    (double)h->n_schur_tiles, (double)h->n_schur_rects, (double)h->n_asm_tiles, (double)h->n_asm_rects,
                    h->n_multi_sweeps, h->n_percol,
                    (double)h->npsd_smem, (double)h->npsd_glob, h->last_sweeps};
    for (int i = 0; i < len && i < 26; ++i) out[i] = v[i];
    return 0;
}

void* cb200_get_stream(cb200_handle* h) { return (void*)h->stream; }
int32_t cb200_set_resident(cb200_handle* h, int32_t resident) { h->resident = resident != 0; return 0; }
int32_t cb200_reset_timers(cb200_handle* h) {
    for (double& x : h->tm.ms) x = 0;
    h->tm.nfactor = h->tm.nsolve = h->tm.nlaunch = 0;
    h->scale_ms = 0;
    return 0;
}

}  // extern "C"
