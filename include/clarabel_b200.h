/* clarabel_b200.h — C-ABI of the CUDA (H100, sm_90a) KKT linear-system backend for Clarabel.jl.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Two reference interfaces are covered:
 *
 *  (1) INNER = the reference's LDL plugin API `AbstractDirectLDLSolver`
 *      (Clarabel.jl/src/kktsolvers/direct-ldl/directldl_defaults.jl:1-72; the QDLDL
 *      implementation it replaces is directldl_qdldl.jl:1-96).  One C function per method.
 *  (2) OUTER = `AbstractKKTSolver` (Clarabel.jl/src/kktsolvers/kktsolver_defaults.jl:1-47,
 *      concrete reference implementation kktsolver_directldl.jl), fused so that cone state is
 *      uploaded once per iteration and the cone->K update, static regularisation,
 *      factorisation, solves and iterative refinement all run on the device.
 *
 * Conventions: every function returns int32 status: 0 = ok, >0 = numerical failure (the Julia
 * shim returns `false`, never throws — kktsolver_directldl.jl:281,356-370), <0 = usage/CUDA error
 * (the shim calls `error(...)`).  Host pointers in/out, synchronous on return (the reference
 * caller is single-threaded and synchronous).  Indices are 0- or 1-based according to
 * cb200_settings.index_base.  Float64 only (T == Float64, as for every external reference
 * engine: ext/directldl_hsl.jl:18).
 */
#ifndef CLARABEL_B200_H
#define CLARABEL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cb200_handle cb200_handle;

/* Mirrors the KKT-relevant fields of `Settings{Float64}` (src/settings.jl:110-132). */
typedef struct cb200_settings {
    int32_t index_base;                 /* 0 (C / Python harness) or 1 (Julia) */
    int32_t device;                     /* CUDA device ordinal */
    int32_t static_regularization_enable;         /* settings.jl:117 */
    double  static_regularization_constant;       /* :118  (1e-8) */
    double  static_regularization_proportional;   /* :119  (eps^2) */
    int32_t dynamic_regularization_enable;        /* :122 */
    double  dynamic_regularization_eps;           /* :123  (1e-13) */
    double  dynamic_regularization_delta;         /* :124  (2e-7) */
    int32_t iterative_refinement_enable;          /* :127 */
    double  iterative_refinement_reltol;          /* :128  (1e-13) */
    double  iterative_refinement_abstol;          /* :129  (1e-12) */
    int32_t iterative_refinement_max_iter;        /* :131  (10) */
    double  iterative_refinement_stop_ratio;      /* :132  (5) */
    int32_t ordering;                   /* 0 AMD, 1 auto (default): nested dissection unless > 3x AMD cost;
                                         * AMD when K holds a dense PSD cone block (detected from pattern + Dsigns), 2 natural */
    double  amd_dense_scale;            /* dense-row threshold multiplier (reference QDLDL path: 1.5, directldl_qdldl.jl:24; default here 0.3) */
    int32_t nd_leaf_size;
    int32_t use_cuda_graph;             /* bit mask: 1 replay the solve sweeps, 2 the factorisation, through CUDA graphs */
    int32_t reserved[8];
} cb200_settings;

void cb200_default_settings(cb200_settings* s);

/* ---------------------------------------------------------------- host-only symbolic analysis
 * (no CUDA call; used by tests and by the CPU-side tooling).  Replaces the symbolic half of
 * QDLDL.qdldl(KKT; logical=true) — directldl_qdldl.jl:18-25. */
typedef struct cb200_symbolic cb200_symbolic;
int32_t cb200_symbolic_create(int64_t N, const int64_t* colptr, const int64_t* rowval,
                              const cb200_settings* st, const int64_t* user_perm,
                              cb200_symbolic** out);
void    cb200_symbolic_destroy(cb200_symbolic* s);
/* what: 0 N, 1 nsuper, 2 nnzL, 3 nlevels, 4 max_front, 5 max_width, 6 upd_total, 7 panel_total,
 *       8 rows_total, 9 nnzK */
int64_t cb200_symbolic_stat(const cb200_symbolic* s, int32_t what);
double  cb200_symbolic_flops(const cb200_symbolic* s);
/* which: 0 perm[N], 1 sn_first[nsuper+1], 2 rows_ptr[nsuper+1], 3 rows[rows_total],
 *        4 rel[rows_total], 5 sn_parent[nsuper], 6 panel_off[nsuper+1], 7 upd_off[nsuper+1],
 *        8 a_map[nnzK], 9 sn_level[nsuper], 10 child_ptr[nsuper+1], 11 child_list[nsuper-#roots],
 *        12 panel_ld[nsuper], 13 per-front child lists [3 * (nsuper-#roots)]: (update-block offset,
 *        rel offset, nr) of child_list[q] at 3q (symbolic.h, kids), the destination-owner assembly maps
 *        14 front_ptr[nsuper+1], 15 asm_base[nsuper+1], 16 asm_colptr[front_ptr[nsuper]],
 *        17 asm_src[asm_base[nsuper]], 18 asm_child[asm_base[nsuper]]
 * All arrays are returned widened to int64 into caller storage of the stated length. */
int32_t cb200_symbolic_get(const cb200_symbolic* s, int32_t which, int64_t* out, int64_t len);
/* Per-tile source lists of the large-front extend-add (symbolic.h, build_tile_lists) for the batch
 * fronts[0..nfronts) and tile size T (64 or 128): schur = 1 the Schur GEMM's tiles, 0 the assembly
 * tiles; gather = 0 for pre-assembled (replicated top) fronts; active (NULL = all, else [nsuper], nonzero
 * = assembled here): multi-GPU mask of the children whose contributions a rank adds, the others get no
 * rectangles.  counts[0] = tiles, counts[1] =
 * rectangles.  If non-NULL, tiles receives (slot, ti, tj, first rectangle) per tile and rects
 * (child, ja, jb, ia, ib) per rectangle; call once with NULL to size them. */
int32_t cb200_symbolic_tile_lists(const cb200_symbolic* s, const int64_t* fronts, int32_t nfronts, int32_t T,
                                  int32_t schur, int32_t gather, const int64_t* active, int64_t* counts,
                                  int64_t* tiles, int64_t* rects);

/* Multi-GPU partition of the assembly tree (host-only): owner[s] in [0,nranks) or -1 for the
 * replicated top set, is_top[s] in {0,1}, rank_load[nranks] = factor-flop weight per rank. */
int32_t cb200_symbolic_partition(const cb200_symbolic* s, int32_t nranks, int64_t* owner,
                                 int64_t* is_top, double* rank_load);

/* Optional ordering hint, consumed by the NEXT cb200_symbolic_create / cb200_create on this thread:
 * block_id[i] >= 0 marks row/column i of K as part of a dense cone block (PSD triangle, dense SOC);
 * nested dissection then keeps each block in one piece (a separator cutting such a clique was
 * observed to destabilise the factorisation late in the IP iteration).  NULL clears the hint. */
int32_t cb200_hint_blocks(const int64_t* block_id, int64_t N);

/* Fill-reducing orderings (perm[k] = original index of the k-th pivot). */
int32_t cb200_order_amd(int64_t n, const int64_t* colptr, const int64_t* rowval,
                        double dense_scale, int64_t* perm);
int32_t cb200_order_nd(int64_t n, const int64_t* colptr, const int64_t* rowval,
                       double dense_scale, int64_t leaf_size, int64_t* perm);

/* ---------------------------------------------------------------- INNER boundary
 * Constructor `MyT{T}(KKT::SparseMatrixCSC, Dsigns::Vector{Int}, settings)` called at
 * kktsolver_directldl.jl:86: symbolic analysis + device upload.  `colptr/rowval/nzval` is the
 * upper-triangular (:triu) KKT matrix; Dsigns in {+1,-1}. */
int32_t cb200_create(int64_t N, const int64_t* colptr, const int64_t* rowval, const double* nzval,
                     const int64_t* Dsigns, const cb200_settings* st, cb200_handle** out);
void    cb200_destroy(cb200_handle* h);                       /* Julia finalizer (MOI_wrapper.jl:133) */
/* update_values!(s, index, values)   — directldl_qdldl.jl:46-56 */
int32_t cb200_update_values(cb200_handle* h, const int64_t* index, const double* values, int64_t len);
/* scale_values!(s, index, scale)     — directldl_qdldl.jl:60-68 */
int32_t cb200_scale_values(cb200_handle* h, const int64_t* index, int64_t len, double scale);
/* refactor!(s, KKT)::Bool            — directldl_qdldl.jl:72-81 ; >0 = non-finite pivot */
int32_t cb200_refactor(cb200_handle* h);
/* solve!(s, KKT, x, b)               — directldl_qdldl.jl:85-96 */
int32_t cb200_solve(cb200_handle* h, double* x, const double* b);
/* linear_solver_info(s)              — directldl_qdldl.jl:35-42 */
int32_t cb200_info(const cb200_handle* h, int64_t* nnzA, int64_t* nnzL, int32_t* ngpus);

/* ---------------------------------------------------------------- OUTER boundary (fused)
 * cb200_set_maps: once after create; uploads LDLDataMap (directldl_datamaps.jl:170-214) and the
 * cone table (CompositeCone.rng_cones / rng_blocks, compositecone_type.jl:96-141).
 *   cone_type[i]: 0 Zero, 1 Nonnegative, 2 SecondOrder, 3 PSDTriangle, 4 Exponential, 5 Power,
 *                 6 GenPower ; cone_dim[i]: dim (PSD: side n)
 *   map_soc_u / map_soc_v: concatenated over sparse SOCs (dim > 4) in cone order; map_soc_D: 2 each.
 *   Nonsymmetric cones (types 4-6): their Hs block (3x3 for exp/pow, coneops_expcone.jl:92-100;
 *   diagonal + expansion columns for genpow, directldl_datamaps.jl:146-166) is the output of the
 *   caller's update_scaling!; the caller sends those few values with cb200_update_values right
 *   before cb200_update_cones, which leaves the entries untouched. */
int32_t cb200_set_maps(cb200_handle* h, int64_t n, int64_t m, int64_t p,
                       const int64_t* map_P, int64_t nnzP, const int64_t* map_A, int64_t nnzA,
                       const int64_t* map_Hs, int64_t nHs, const int64_t* map_diag_full,
                       int64_t ncones, const int32_t* cone_type, const int64_t* cone_dim,
                       const int64_t* map_soc_u, const int64_t* map_soc_v, const int64_t* map_soc_D);
/* kktsolver_update!(ks, cones)::Bool — kktsolver_directldl.jl:197-294 (get_Hs!, sign flip,
 * sparse-cone scatter, static regularisation, refactor).  Cone scaling state as produced by
 * update_scaling! on the host: w over all m rows (NN: w, SOC: w), per-SOC eta and d, SOC u/v
 * over all SOC rows, PSD R matrices (column-major n*n each, cone order).  A NULL argument keeps
 * that part of the state on the device (the previous upload, or what cb200_update_scaling
 * computed), in both modes. */
int32_t cb200_update_cones(cb200_handle* h, const double* w, const double* soc_eta,
                           const double* soc_d, const double* soc_u, const double* soc_v,
                           const double* psd_R);
/* update_scaling!(cones, s, z, μ, strategy) for symmetric cones — coneops_nncone.jl:77-89,
 * coneops_socone.jl:75-154, coneops_psdtrianglecone.jl:78-143 — on the device.  s and z have length m (host
 * pointers; device pointers under cb200_set_resident).  Writes the state cb200_update_cones reads (w, eta, d, u, v,
 * PSD R), so that cb200_update_cones(h, NULL, ..., NULL) refactors from it, plus λ (NN/SOC rows), PSD Rinv and PSD
 * λ for the host cone operations (cb200_get_scaling).  *ok_scale = 0 where the host returns false: a SOC residual
 * of z, s or w not > 0 (NaN included), a Cholesky pivot of S or Z not > 0, or a Jacobi SVD of L2'L1 that has not
 * converged in 30 sweeps; NN cones are not checked.  PSD λ is not sorted (R, Rinv and λ agree with each other).
 * Returns -2 if the cone table has exponential, power or generalised power cones (types 4-6): they keep their host
 * scaling.  In multi-GPU mode every rank computes the whole state from its own (replicated) s and z. */
int32_t cb200_update_scaling(cb200_handle* h, const double* s, const double* z, int32_t* ok_scale);
/* Download the scaling state into host arrays; NULL skips an array.  Lengths: w, lam m; eta, d #SOC; u, v the SOC
 * rows; R, Rinv the sum of n*n over the PSD cones (column-major each, cone order); psd_lam the sum of n. */
int32_t cb200_get_scaling(cb200_handle* h, double* w, double* lam, double* eta, double* d, double* u, double* v,
                          double* R, double* Rinv, double* psd_lam);
/* kktsolver_setrhs!(ks, rhsx, rhsz) — kktsolver_directldl.jl:313-327: b = [rhsx; rhsz; 0_p].  The
 * right-hand side is copied to the device here (the caller may reuse its buffers on return);
 * a following cb200_solve_ir with rhsx == rhsz == NULL solves for it. */
int32_t cb200_setrhs(cb200_handle* h, const double* rhsx, const double* rhsz);
/* kktsolver_setrhs! + kktsolver_solve! (+ getlhs) — kktsolver_directldl.jl:313-371, with
 * _iterative_refinement :389-449 on the device.  lhsx / lhsz may be NULL (Julia `nothing`);
 * rhsx == rhsz == NULL: use the right-hand side set by cb200_setrhs. */
int32_t cb200_solve_ir(cb200_handle* h, const double* rhsx, const double* rhsz,
                       double* lhsx, double* lhsz, int32_t* ir_rounds);
/* Several right-hand sides against the current factorisation, one pass over L per sweep: a sweep carries up
 * to 4 columns (more columns run in ceil(nrhs / 4) sweeps), interleaved so that every L entry is loaded once
 * for all of them.  These calls leave the single-RHS state alone: what cb200_setrhs stored and the last
 * single solution (download selector 6) are unchanged.  nrhs == 0 is a no-op; nrhs < 0, a leading
 * dimension < N or a NULL required pointer return -2.
 * cb200_solve_multi: B, X column-major N x nrhs with leading dimensions ldb, ldx >= N (host pointers, like
 * cb200_solve).  Column j of X is bit-for-bit what cb200_solve(h, x, B[:, j]) returns. */
int32_t cb200_solve_multi(cb200_handle* h, int32_t nrhs, double* X, int64_t ldx,
                          const double* B, int64_t ldb);
/* kktsolver_setrhs! + kktsolver_solve! for nrhs systems: rhsx n x nrhs, rhsz m x nrhs (column-major, packed),
 * lhsx / lhsz the same shapes or NULL.  Iterative refinement runs per column with the single-RHS rules
 * (kktsolver_directldl.jl:389-449).  ir_rounds[nrhs] and status[nrhs] (0 ok, 1 numerical failure) are
 * optional outputs.  Returns 0 if every column succeeded, 1 otherwise; failed columns of lhsx / lhsz are
 * NaN-filled as in cb200_solve_ir.  Column j is bit-for-bit what cb200_solve_ir(h, rhsx[:, j], rhsz[:, j], ...)
 * returns, with the same ir_rounds.  Needs cb200_set_maps.  Resident mode: rhsx / rhsz are device pointers
 * and the results stay on the device (cb200_download selector 8).  In multi-GPU mode and with
 * CB200_SUBTREE=1 both calls solve column by column through the single-RHS path (cb200_get_stats 22). */
int32_t cb200_solve_ir_multi(cb200_handle* h, int32_t nrhs, const double* rhsx, const double* rhsz,
                             double* lhsx, double* lhsz, int32_t* ir_rounds, int32_t* status);
/* kktsolver_update_P!/A! — kktsolver_directldl.jl:374-386 */
int32_t cb200_update_P(cb200_handle* h, const double* values, int64_t len);
int32_t cb200_update_A(cb200_handle* h, const double* values, int64_t len);

/* ---------------------------------------------------------------- introspection (tests / bench)
 * what: 0 device KKT nzval (unregularised, len nnzK), 1 D (permuted, len N), 2 panel storage,
 *       3 perm (as doubles), 4 last static regulariser (len 1), 5 regularised-pivot count (len 1),
 *       6 full solution [x; z; expansion variables] of the last solve (len N),
 *       7 original indices of the first 64 dynamically regularised pivots of the last factorisation (len 64, -1 = none),
 *       8 full solutions of the last cb200_solve_ir_multi, N x nrhs column-major (len N * nrhs),
 *       9 residual e = b - K x (unregularised K) last computed by cb200_solve_ir (len N): x is the last
 *         iterate refinement tried, which is the returned solution unless the final round was rejected
 *         (with iterative_refinement_max_iter = 0 it is the unrefined solve); not written when
 *         refinement is disabled */
int32_t cb200_download(cb200_handle* h, int32_t what, double* out, int64_t len);
/* timers (ms, accumulated CUDA-event times on the handle's stream): 0 cone update + scatter,
 * 1 factor, 2 triangular solves, 3 spmv/residual ; counters: 4 #factor, 5 #solve sweeps (a multi-RHS sweep of
 * up to 4 columns counts once), 6 #kernel launches ;
 * with cb200_set_detail(h,1) also per kernel class inside the factorisation: 7 k_schur_large,
 * 8 pivot-block phase (k_diag64 + k_rows64), 9 small fronts (k_factor_small), 10 assembly ;
 * 11 device time of cb200_update_scaling (its kernels, always recorded) */
int32_t cb200_get_timers(cb200_handle* h, double* out, int32_t len);
int32_t cb200_reset_timers(cb200_handle* h);
/* event timing inside the phases (disables CUDA-graph replay while on): level 0 off, 1 the four
 * factorisation groups of cb200_get_timers, 2 additionally every kernel class of the factorisation
 * and of the solve sweeps (cb200_get_fine_timers) */
int32_t cb200_set_detail(cb200_handle* h, int32_t level);
/* detail level 2: accumulated ms per kernel class; writes min(len, count) values, returns count;
 * cb200_fine_timer_name(i) names class i.  Reset by cb200_reset_timers. */
int32_t cb200_get_fine_timers(cb200_handle* h, double* out_ms, int32_t len);
const char* cb200_fine_timer_name(int32_t i);
/* symbolic statistics: 0 factor flops (sum of squared column lengths), 1 flops of the large-front
 * Schur GEMMs, 2 flops of the large-front panel phase, 3 nnzL, 4 levels, 5 supernodes, 6 large
 * fronts, 7 panel bytes of the multi-CTA solve class, 8 update-storage bytes, 9 panel-storage bytes,
 * 10 ordering used, 11 flops of this rank's fronts, 12 TMA tensor maps in use, 13 their k-major order,
 * 14 factorisation graphs instantiated (0-2), 15 solve-sweep graph instantiated, 16 bottom subtrees
 * solved by k_fwd_subtree / k_bwd_subtree, 17 Schur tiles and 18 their child rectangles, 19 assembly
 * tiles and 20 their child rectangles (all large batches, cb200_symbolic_tile_lists), 21 multi-RHS sweeps run
 * batched, 22 columns of the multi-RHS calls solved one by one through the single-RHS path, 23 PSD cones
 * scaled in shared memory and 24 in a global workspace by cb200_update_scaling, 25 Jacobi sweeps of its last call
 * (maximum over the PSD cones) */
int32_t cb200_get_stats(const cb200_handle* h, double* out, int32_t len);
/* ---------------------------------------------------------------- multi-GPU (one process per GPU)
 * Every rank creates the same handle on its own device (replicated symbolic analysis), then
 * calls cb200_dist_init with a NCCL unique id obtained on rank 0 (cb200_nccl_unique_id) and
 * distributed by the caller (torch.distributed / MPI).  Independent elimination-tree subtrees
 * are factored and solved on their owner rank; the replicated top (root separator) fronts are
 * assembled with an NCCL all-reduce over NVLink.  All ranks must then issue the same sequence
 * of refactor / update_cones / solve calls with the same inputs; results are replicated. */
int32_t cb200_nccl_unique_id(char out[128]);
int32_t cb200_dist_init(cb200_handle* h, int32_t rank, int32_t nranks, const char uid[128]);

/* The CUDA stream (cudaStream_t) all of this handle's work is enqueued on, so a caller can
 * bracket calls with its own events. */
void*   cb200_get_stream(cb200_handle* h);
/* resident != 0: the inputs live in HBM.  Non-NULL pointer arguments of cb200_update_cones and
 * cb200_setrhs are then DEVICE pointers (copied device-to-device on the handle's stream), NULL
 * keeps what the previous call left on the device; cb200_solve_ir ignores its host pointers and
 * leaves the solution on the device (cb200_download selector 6).  This is the mode bench.py's
 * device-resident `value` is measured in; the drop-in path (resident == 0) takes host pointers. */
int32_t cb200_set_resident(cb200_handle* h, int32_t resident);
const char* cb200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* CLARABEL_B200_H */
