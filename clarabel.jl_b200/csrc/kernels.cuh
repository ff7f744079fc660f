// Device kernels for the H100 KKT path (sm_90a).  FP64 throughout (the reference is Float64
// end-to-end and its IR tolerance is 1e-13 - src/settings.jl:127-132).
//
//   G1  cone -> K value update            k_hs_diag, k_hs_soc_dense, k_soc_expansion, k_soc_D
//   G2  PSD skron                         k_psd_rrt, k_psd_skron
//   G3  static regularisation             k_diag_absmax, k_compute_eps, k_shift_diag
//   G4  small-front LDL' (shared memory)  k_factor_small (nf <= 64), k_factor_panel (64 < nf <= 152)
//   G5  large-front blocked LDL'          k_piv_diag, k_piv_rows, k_ldl_update_tma (TMA-fed 128 x 128 DMMA GEMM),
//                                         k_ldl_update_ldg (fallback), k_finish_large
//   G6  extend-add                        fused in G4 ; k_assemble_tiles ; add_tile_rects (also in the Schur
//                                         epilogue) ; k_assemble_atomic
//   G7  multifrontal triangular solves    k_fwd_{leaf,warp<16|32>,cta}, k_bwd_*, k_big_{asm,tri,gemv}_*, k_*_subtree,
//                                         k_pack_perm, k_unpack_perm ; R-wide forms for several right-hand sides:
//                                         kernels_multi.cuh
//   G8  symmetric SpMV residual + norm    k_residual, k_residual_long
//   G9  multi-GPU helpers                 k_zero_panels, k_mask_vec  (collectives: api_cuda.cu)
//   G10 NT scaling of the symmetric cones k_scale_nn, k_scale_soc, k_scale_psd: kernels_scaling.cuh
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include <cuda.h>          // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)
#include "symbolic.h"      // MANY_CHILDREN, TileEntry, TileRect

namespace cb200 {

struct DevSym {                 // device copies of the Symbolic arrays
    const int32_t* sn_first;    // [nsuper+1]
    const int64_t* rows_ptr;    // [nsuper+1]
    const int32_t* rows;
    const int32_t* rel;
    const int32_t* child_ptr;
    const int32_t* child_list;
    const int64_t* panel_off;
    const int32_t* ld;          // [nsuper] leading dimension of each panel (>= nf; padded for large fronts)
    const int64_t* upd_off;
    const int8_t*  dsign;       // [N] permuted pivot signs
    const int64_t* front_ptr;   // destination-owner assembly maps (symbolic.h)
    const int64_t* asm_base;
    const int32_t* asm_colptr;
    const int32_t* asm_src;
    const int32_t* asm_child;
    const Symbolic::KidEntry* kids;   // per-front child lists of k_factor_small (symbolic.h)
    const int8_t*  active;      // multi-GPU: per-supernode mask of children whose contributions this rank
                                // assembles into the replicated top fronts (nullptr = all)
};

struct RegParams { double eps, delta; int enable; int32_t* log; };   // log: first 64 regularised pivots (permuted column, unregularised value bits elsewhere)
__device__ __forceinline__ void note_reg(const RegParams& rp, unsigned int* nreg, int col, unsigned int count = 1u) {
    const unsigned int slot = atomicAdd(nreg, count);
    if (rp.log && slot < 64u) rp.log[slot] = col;
}

// ------------------------------------------------------------------ inverted diagonal blocks
// The triangular solves never substitute column by column: every SBxSB diagonal block of the
// unit-lower L11 of a supernode is replaced, in place, by its inverse at factorisation time, so
// a solve is a sequence of block GEMVs  x_kb = inv(L_kb,kb) w_kb ;  w_rest -= L[rest,kb] x_kb
// with no per-column dependency chain (chain length ns/SB instead of ns).
constexpr int SB = 64;

// ------------------------------------------------------------------ G4 small fronts
// One group of G threads per front (a warp for nf <= 32, several fronts per CTA; the whole CTA
// above); the whole front lives in shared memory.  Fuses: extend-add of the children's update
// blocks (G6), right-looking LDL' of the ns pivot columns with the reference's sign-based dynamic
// regularisation (QDLDL semantics: if D[k]*sign < eps then D[k] = delta*sign), the inversion of the
// diagonal blocks of L11 and the write-back of the L panel and of this front's update block.
// Every entry sees the same floating-point operations in the same order as in the column-serial
// schedule (per-entry order noted at each step), so the factor does not depend on G.
// a warp group waits on its own named barrier (1 + its index in the CTA): __syncwarp() would bring
// WARPSYNC.COLLECTIVE landing pads into the pivot loop
template <int G>
__device__ __forceinline__ void group_sync() {
    if constexpr (G == 32) asm volatile("bar.sync %0, 32;" :: "r"(1 + (int)(threadIdx.x >> 5)) : "memory");
    else __syncthreads();
}

template <int G, int FPC>
__global__ void __launch_bounds__(G * FPC)
k_factor_small(DevSym S, const int32_t* __restrict__ batch, int cnt, int fstride, double* __restrict__ Lst,
               double* __restrict__ Ust, double* __restrict__ D, double* __restrict__ Dinv,
               RegParams rp, unsigned int* __restrict__ nreg) {
    static_assert(FPC == 1 || (G == 32 && FPC <= 15), "several fronts per CTA only with one warp per front");
    extern __shared__ double smem_small[];
    const int slot = blockIdx.x * FPC + (int)threadIdx.x / G;
    if (slot >= cnt) return;                            // a whole group (FPC > 1: a whole warp)
    double* F = smem_small + (size_t)((int)threadIdx.x / G) * fstride;
    const int s = batch[slot];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    const int tid = (int)threadIdx.x % G, lane = tid & 31, wid = tid >> 5;
    constexpr int NW = G / 32;
    double* Lp = Lst + S.panel_off[s];
    // 1. panel -> first ns columns (identical layout), zero the trailing block
    for (int i = tid; i < nf * ns; i += G) F[i] = Lp[i];
    for (int i = nf * ns + tid; i < nf * nf; i += G) F[i] = 0.0;
    group_sync<G>();
    // 2. extend-add from the per-front child list, one child after the other with all threads: a child
    // adds the lower triangle of its update block through rel (injective, so no two threads meet), and
    // every entry is summed start + c1 + c2 ... in child_list order, the order of the destination-owner maps
    {
        const int q0 = S.child_ptr[s], nch = S.child_ptr[s + 1] - q0;
        Symbolic::KidEntry nxt{};
        if (nch > 0) nxt = S.kids[q0];
        for (int q = 0; q < nch; ++q) {
            const Symbolic::KidEntry kd = nxt;
            if (q + 1 < nch) nxt = S.kids[q0 + q + 1];
            const int m = kd.nrc;
            const int32_t* relc = S.rel + kd.roff;
            const double* U = Ust + kd.uoff;
            // thread tid takes entries tid, tid + G, ... of the lower triangle, column by column: column j
            // holds rows j..m-1, so stepping past its end continues at row j+1 of column j+1
            int i = tid, j = 0;
            while (j < m && i >= m) { i -= m - j - 1; ++j; }
            while (j < m) {
                F[relc[i] + relc[j] * nf] += U[i + (int64_t)j * m];
                i += G;
                while (j < m && i >= m) { i -= m - j - 1; ++j; }
            }
            group_sync<G>();
        }
    }
    // 3. right-looking LDL' on the pivot columns, one barrier per pivot: step k applies pivot k to the
    // columns right of it (entry (i,j) -= F_ik * (F_jk * dinv_k), ascending k) and scales column k-1,
    // which step k no longer reads
    {
        double dp = 0.0, dinvp = 0.0;
        bool regp = false;
        for (int k = 0; k <= ns; ++k) {
            if (k > 0) {
                const int c = k - 1;
                for (int i = k + tid; i < nf; i += G) F[i + c * nf] *= dinvp;
                if (tid == 0) {
                    F[c + c * nf] = dp; D[f + c] = dp; Dinv[f + c] = dinvp;
                    if (regp) note_reg(rp, nreg, f + c);
                }
            }
            if (k == ns) break;
            double d = F[k + k * nf];
            const double sg = (double)S.dsign[f + k];
            bool reg = false;
            if (rp.enable && d * sg < rp.eps) { d = rp.delta * sg; reg = true; }
            const double dinv = 1.0 / d;
            const double* ck = F + k * nf;
            for (int j = k + 1 + wid; j < nf; j += NW) {
                const double wj = ck[j] * dinv;
                double* cj = F + j * nf;
                for (int i = j + lane; i < nf; i += 32) cj[i] -= ck[i] * wj;
            }
            dp = d; dinvp = dinv; regp = reg;
            group_sync<G>();
        }
        group_sync<G>();
    }
    // 3b. replace the diagonal blocks of L11 by their inverses in place (X = T^-1 for the solves' block
    // GEMVs, see "inverted diagonal blocks" above).  T_ij is parked at the unused mirror position (j, i) and X_ij starts at
    // -T_ij; step k subtracts T_ik X_kj from every X_ij with j < k < i, so each entry is
    // -T_ij - sum_{k=j+1}^{i-1} T_ik X_kj accumulated in ascending k, with all threads on each step.
    for (int kb = 0; kb < ns; kb += SB) {
        const int sb = min(SB, ns - kb);
        if (sb < 2) continue;
        double* T = F + kb + kb * nf;
        for (int e = tid; e < sb * sb; e += G) {
            const int i = e % sb, j = e / sb;
            if (i > j) { const double t = T[i + j * nf]; T[j + i * nf] = t; T[i + j * nf] = -t; }
        }
        group_sync<G>();
        for (int k = 1; k < sb - 1; ++k) {
            const int mi = sb - 1 - k;                  // rows k+1 .. sb-1
            for (int e = tid; e < k * mi; e += G) {
                const int i = k + 1 + e % mi, j = e / mi;
                T[i + j * nf] -= T[k + i * nf] * T[k + j * nf];
            }
            group_sync<G>();
        }
    }
    // 4. write back (the upper triangle of L11 is zero in the panel storage; the mirrors are dropped)
    for (int e = tid; e < nf * ns; e += G) {
        const int i = e % nf, j = e / nf;
        Lp[e] = i < j ? 0.0 : F[e];
    }
    if (nr > 0) {
        double* Us = Ust + S.upd_off[s];
        for (int j = wid; j < nr; j += NW) {
            const double* cj = F + (ns + j) * nf + ns;
            for (int i = j + lane; i < nr; i += 32) Us[i + (int64_t)j * nr] = cj[i];
        }
    }
}

// ------------------------------------------------------------------ G4b mid-size fronts (64 < nf <= 152)
// Only the nf x ns panel lives in shared memory (a front of 128 x 30 needs 31 KB instead of
// 128 KB => several CTAs per SM); the update block stays in global memory:
//   1. panel <- scattered K entries ; extend-add: destination columns < ns accumulate into the smem
//      panel, columns >= ns are summed in a per-warp smem column buffer and written to the update
//      block (destination-owner lists => fixed summation order);
//   2. blocked LDL' of the panel in 16-column steps: 16x16 diagonal sub-block in registers of one
//      warp (shuffles), thread-per-row solve of the rows below, rank-16 update of the remaining
//      panel columns; sign-based dynamic regularisation per pivot as in QDLDL;
//   3. Schur complement U -= L21 D L21' with 4x4 register tiles read from the smem panel;
//   4. inverse of the 64x64 diagonal blocks of L11 (4 threads per column) and write-back.
// dynamic smem: panel (maxpanel) + Xs (nf x 17) + colbuf (8 x nf) doubles.
__global__ void __launch_bounds__(256)
k_factor_panel(DevSym S, const int32_t* __restrict__ batch, int maxpanel, int maxnf,
               double* __restrict__ Lst, double* __restrict__ Ust, double* __restrict__ D,
               double* __restrict__ Dinv, RegParams rp, unsigned int* __restrict__ nreg) {
    extern __shared__ double smem[];
    __shared__ double dvs[160], dis[160];
    __shared__ double ps4[256];
    const int s = batch[blockIdx.x];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    double* P = smem;                                   // nf x ns, column-major, ld = nf
    double* Xs = smem + (size_t)nf * ns;                // (rows below) x 17
    double* colbuf = Xs + (size_t)nf * 17;              // 8 warps x nf   (total nf*ns + 25*nf doubles)
    (void)maxpanel; (void)maxnf;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    double* Lp = Lst + S.panel_off[s];
    double* Us = Ust + S.upd_off[s];
    for (int i = tid; i < nf * ns; i += 256) P[i] = Lp[i];
    __syncthreads();
    // ---- 1. extend-add
    {
        const int32_t* cp = S.asm_colptr + S.front_ptr[s];
        const int64_t base = S.asm_base[s];
        double* cb = colbuf + (size_t)wid * nf;
        for (int d = wid; d < nf; d += 8) {
            const bool in_panel = d < ns;
            double* dst = in_panel ? P + d * nf : cb;
            if (!in_panel) { for (int r = d + lane; r < nf; r += 32) cb[r] = 0.0; __syncwarp(); }
            for (int e = cp[d]; e < cp[d + 1]; ++e) {
                const int q = S.asm_src[base + e];
                const int c = S.asm_child[base + e];
                const int64_t rp0 = S.rows_ptr[c];
                const int nrc = (int)(S.rows_ptr[c + 1] - rp0);
                const int j = (int)(q - rp0);
                const int32_t* relc = S.rel + rp0;
                const double* src = Ust + S.upd_off[c] + (int64_t)j * nrc;
                for (int i = j + lane; i < nrc; i += 32) dst[relc[i]] += src[i];
                __syncwarp();
            }
            if (!in_panel) {
                double* ucol = Us + (int64_t)(d - ns) * nr - ns;
                for (int r = d + lane; r < nf; r += 32) ucol[r] = cb[r];
                __syncwarp();
            }
        }
    }
    __syncthreads();
    // ---- 2. blocked LDL' of the panel
    for (int kb = 0; kb < ns; kb += 16) {
        const int cbk = min(16, ns - kb);
        if (wid == 0) {
            // right-looking LDL' of the cbk x cbk diagonal sub-block in shared memory, lane j owns column
            // kb + j.  (The former register/shuffle version sat inside a loop whose bounds the compiler cannot
            // prove warp-uniform: every shuffle became a WARPSYNC.COLLECTIVE, tens of cycles each.)
            for (int k = 0; k < cbk; ++k) {
                double d = P[(kb + k) + (kb + k) * nf];
                const double sg = (double)S.dsign[f + kb + k];
                bool reg = false;
                if (rp.enable && d * sg < rp.eps) { d = rp.delta * sg; reg = true; }
                const double dinv = 1.0 / d;
                if (lane > k && lane < cbk) {
                    const double wj = P[(kb + lane) + (kb + k) * nf] * dinv;
                    for (int i = lane; i < cbk; ++i) P[(kb + i) + (kb + lane) * nf] -= P[(kb + i) + (kb + k) * nf] * wj;
                }
                __syncwarp();
                if (lane > k && lane < cbk) P[(kb + lane) + (kb + k) * nf] *= dinv;
                if (lane == 0) { P[(kb + k) + (kb + k) * nf] = d; dvs[kb + k] = d; dis[kb + k] = dinv; if (reg) note_reg(rp, nreg, f + kb + k); }
                __syncwarp();
            }
        }
        __syncthreads();
        const int r0 = kb + cbk;                        // first row below the diagonal sub-block
        const int nbelow = nf - r0;
        for (int t = tid; t < nbelow; t += 256) {
            const int r = r0 + t;
            double x[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) x[j] = (j < cbk) ? P[r + (kb + j) * nf] : 0.0;
#pragma unroll
            for (int j = 1; j < 16; ++j) {
                if (j < cbk) {
                    double v = x[j];
#pragma unroll
                    for (int l = 0; l < 16; ++l) if (l < j) v -= x[l] * P[(kb + j) + (kb + l) * nf];
                    x[j] = v;
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                Xs[t * 17 + j] = x[j];
                if (j < cbk) P[r + (kb + j) * nf] = x[j] * dis[kb + j];
            }
        }
        __syncthreads();
        // remaining panel columns jc in [r0, ns): P[i][jc] -= sum_k X[i][k] L[jc][k], i >= jc
        const int ncols = ns - r0;
        if (ncols > 0) {
            for (int jc = wid; jc < ncols; jc += 8) {
                const int gj = r0 + jc;
                double lj[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) lj[k] = (k < cbk) ? P[gj + (kb + k) * nf] : 0.0;
                for (int i = gj + lane; i < nf; i += 32) {
                    const double* xr = Xs + (i - r0) * 17;
                    double acc = 0.0;
#pragma unroll
                    for (int k = 0; k < 16; ++k) acc += xr[k] * lj[k];
                    P[i + gj * nf] -= acc;
                }
            }
        }
        __syncthreads();
    }
    for (int k = tid; k < ns; k += 256) { D[f + k] = dvs[k]; Dinv[f + k] = dis[k]; }
    // ---- 3. Schur complement into the (already assembled) update block: 4 x 4 register tiles
    if (nr > 0) {
        const int T4 = (nr + 3) >> 2;
        for (int t = tid; t < T4 * T4; t += 256) {
            const int ti = t % T4, tj = t / T4;
            if (ti < tj) continue;
            const int i0 = ns + ti * 4, j0 = ns + tj * 4;
            double acc[4][4];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
            for (int k = 0; k < ns; ++k) {
                const double dk = dvs[k];
                double li[4], lj[4];
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    li[a] = (i0 + a < nf) ? P[(i0 + a) + k * nf] : 0.0;
                    lj[a] = (j0 + a < nf) ? P[(j0 + a) + k * nf] * dk : 0.0;
                }
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[a][c] += li[a] * lj[c];
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int gj = j0 + c;
                if (gj >= nf) continue;
                double* ucol = Us + (int64_t)(gj - ns) * nr - ns;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    const int gi = i0 + a;
                    if (gi < nf && gi >= gj) ucol[gi] -= acc[a][c];
                }
            }
        }
    }
    // ---- 4. inverse of every 64 x 64 diagonal block of L11, 4 threads per column; X[i][j] (i > j)
    // goes to the unused mirror position P[j + i*nf] and is swapped into place at write-back
    for (int b0 = 0; b0 < ns; b0 += SB) {
        const int sb = min(SB, ns - b0);
        const int j = tid >> 2, part = tid & 3;
        for (int i = 1; i < SB; ++i) {
            double acc2 = 0.0;
            if (i > j && i < sb)
                for (int k = j + 1 + part; k < i; k += 4) acc2 += P[(b0 + i) + (b0 + k) * nf] * P[(b0 + j) + (b0 + k) * nf];
            ps4[tid] = acc2;                         // 4 partial sums per column, summed through shared memory
            __syncwarp();                            // (no shuffles inside this loop: see the note above)
            if (part == 0) acc2 = (ps4[tid] + ps4[tid + 1]) + (ps4[tid + 2] + ps4[tid + 3]);
            if (part == 0 && i > j && i < sb) P[(b0 + j) + (b0 + i) * nf] = -(P[(b0 + i) + (b0 + j) * nf] + acc2);
            __syncwarp();
        }
    }
    __syncthreads();
    for (int e = tid; e < nf * ns; e += 256) {
        const int i = e % nf, j = e / nf;
        double v = P[e];
        if (i < ns && i > j && (i / SB) == (j / SB)) v = P[j + i * nf];     // inverted diagonal block
        Lp[e] = v;
    }
}

// ------------------------------------------------------------------ G6 assembly for large fronts
// Large fronts come in two kinds.  A gather front (the default: at most MANY_CHILDREN children, not a
// replicated top front) has only its panel columns assembled by k_assemble_tiles; its update block U
// is never zeroed or pre-assembled: the Schur epilogue builds each tile of U from the children
// (add_tile_rects) and writes U = sum - L21 D L21' once.  A pre-assembled front (more than
// MANY_CHILDREN children: k_assemble_atomic; multi-GPU top fronts: summed by NCCL before the Schur
// GEMM) is zeroed (k_zero_upd), fully assembled and then updated in place by the epilogue.
// Both walk host-built per-tile rectangle lists (symbolic.h, build_tile_lists).
__device__ __forceinline__ bool gathers_update(const DevSym& S, int s, int gather) {
    return gather && S.child_ptr[s + 1] - S.child_ptr[s] <= MANY_CHILDREN;
}

// Fronts with thousands of (tiny) children — e.g. the factor-row front of a portfolio KKT system
// with one child per asset: the destination-owner loop would serialise ~1e3 sources per column.
// Here every child is scattered by its own warp with FP64 atomics into the (zeroed / scattered)
// front.  This is the one place where the summation order is not fixed (documented in DESIGN.md);
// it is used only above MANY_CHILDREN children.  grid (children), 64 threads.
__global__ void __launch_bounds__(64)
k_assemble_atomic(DevSym S, int s, double* __restrict__ Lst, double* __restrict__ Ust) {
    const int c = S.child_list[S.child_ptr[s] + blockIdx.x];
    if (S.active && !S.active[c]) return;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    double* Lp = Lst + S.panel_off[s];
    double* Us = Ust + S.upd_off[s];
    const int64_t rp0 = S.rows_ptr[c];
    const int nrc = (int)(S.rows_ptr[c + 1] - rp0);
    const int32_t* relc = S.rel + rp0;
    const double* Uc = Ust + S.upd_off[c];
    for (int e = threadIdx.x; e < nrc * nrc; e += 64) {
        const int i = e % nrc, j = e / nrc;
        if (i < j) continue;
        const int dj = relc[j], di = relc[i];
        double* dst = dj < ns ? Lp + (int64_t)dj * ld + di : Us + (int64_t)(dj - ns) * nr + (di - ns);
        atomicAdd(dst, Uc[e]);
    }
}

// ------------------------------------------------------------------ G5 large fronts, blocked
// Right-looking blocked LDL' in global memory, batched over the large fronts of a level.  Panels
// of large fronts have a padded leading dimension ld (multiple of 8 doubles) so that TMA can
// address them.  Per pivot block J (PB = 64 columns) three launches:
//   k_piv_diag            one CTA per front: LDL' of the (already updated) 64 x 64 diagonal block with
//                         the sign-based dynamic regularisation, inverse of its unit-lower factor
//   k_piv_rows            CTA per 64-row tile below: L[rows,J] = F[rows,J] inv(L_JJ)' D_J^-1
//   k_ldl_update (mode 0) F[r,c] -= L[r,J] D_J L[c,J]'  for the remaining PANEL columns c, r >= c (K = 64)
// and once per front
//   k_ldl_update (mode 1) F22 -= L21 D L21'   (K = ns: the Schur complement into the update block)
//   k_finish_large        move the parked inverted diagonal blocks into the panel
// No CTA ever runs a deep GEMM on its own (the old left-looking k_diag64 did: K = J0 for a 64 x 64
// tile); the trailing update block is read and written once (big-K GEMM).
// k_ldl_update exists in two versions:
//   k_ldl_update_tma   128 x 128 CTA tile, operands brought in by TMA (cp.async.bulk.tensor.3d) through a
//                      4-stage mbarrier ring by one producer warp, 8 consumer warps on the FP64
//                      tensor-core path (DMMA; wgmma has no f64 type)
//   k_ldl_update_ldg   64 x 64 tile, LDG -> registers -> STS double buffering (fallback when the
//                      driver cannot encode tensor maps, and the reference for A/B comparisons)
constexpr int GBM = 64, GBK = 16;
constexpr int PB = 64;

constexpr int GLD = 72;                        // smem row stride (doubles)
constexpr int GSM = 2 * 2 * GBK * GLD;         // doubles of shared memory used by the tile routine

__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
// The wide FP64 tensor-core shape (sm_90+): D(16x8) += A(16x16) B(16x8).  Fragment layout (lane = 4 g + t):
//   a[2 v + h] = A[g + 8 h][t + 4 v]   b[v] = B[t + 4 v][g]   c[2 h + e] = C[g + 8 h][2 t + e]
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                 "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// Tile decode shared by both GEMM versions.  Updated elements: c_lo <= col < c_hi, col <= row < nf
// with k in [k0, k1).  Tiles of size T are anchored at front-local index 0.
//   mode 0 (panel step at pivot block J0): k = [J0, min(J0+PB, ns)), cols (k1, ns);  grid.x = nb * na,
//          tile (tj0 + b, tj0 + b + a) for b = x / na, a = x % na
//   mode 1 (Schur): k = [0, ns), cols [ns, nf);  grid.x = the batch's Schur tile list (build_tile_lists)
struct UpdTile { int k0, k1, c_lo, c_hi, ti, tj; bool valid; };
template <int T>
__device__ __forceinline__ UpdTile decode_update_tile(int mode, int J0, int na, int ns, int nf, const TileEntry& te) {
    UpdTile u; u.valid = false;
    if (mode == 0) {
        if (J0 >= ns) return u;
        u.k0 = J0; u.k1 = min(J0 + PB, ns); u.c_lo = u.k1; u.c_hi = ns;
        if (u.c_lo >= u.c_hi) return u;
        const int tj0 = u.c_lo / T;
        u.tj = tj0 + (int)blockIdx.x / na; u.ti = u.tj + (int)blockIdx.x % na;
        u.valid = (u.tj * T < u.c_hi) && (u.ti * T < nf);
    } else {                                    // every listed tile is a valid one
        u.k0 = 0; u.k1 = ns; u.c_lo = ns; u.c_hi = nf;
        u.ti = te.ti; u.tj = te.tj; u.valid = true;
    }
    return u;
}

// Entry (row r, column c) of a T x T column-major tile in shared memory.  The XOR moves the four
// column pairs of one accumulator fragment onto different banks.
template <int T>
__device__ __forceinline__ int tile_idx(int r, int c) { return c * T + (r ^ (((c >> 1) & 3) << 3)); }

// Adds the rectangles rect[0..nrect) of a tile (rows r0.., columns c0..) into the T x T tile in
// shared memory, one after the other: every entry becomes start + c1 + c2 + ... in child_list order,
// the order of the destination-owner maps.  The entries of one rectangle are distinct, so its
// threads need no ordering among themselves; a barrier separates consecutive rectangles.  Each
// rectangle's rel windows are staged in relw (2 x 2T ints, double-buffered so that one barrier per
// rectangle suffices): child rows [ia, ib) -> tile rows, child columns [ja, jb) -> tile columns.
// Every rectangle is processed, so that buffer k & 1 is never restaged before the barrier that
// ends its last use: the multi-GPU mask of inactive children is applied when the lists are built.
// Warp w adds child columns ja + w, ja + w + nthr / 32, ...; their rows are contiguous and ascending
// in the child's update block.  sync() synchronises the nthr threads; the last one publishes the tile.
template <int T, class Sync>
__device__ __forceinline__ void add_tile_rects(const DevSym& S, const double* __restrict__ Ust,
                                               const TileRect* __restrict__ rect, int nrect, int r0, int c0,
                                               double* tile, int* relw, int tid, int nthr, Sync sync) {
    const int lane = tid & 31;
    for (int k = 0; k < nrect; ++k) {
        const int4 a = __ldg(reinterpret_cast<const int4*>(rect + k));          // child, ja, jb, ia
        const int c = a.x, ja = a.y, jb = a.z, ia = a.w, ib = __ldg(&rect[k].ib);
        const int64_t rp0 = S.rows_ptr[c];
        const int nrc = (int)(S.rows_ptr[c + 1] - rp0);
        const int32_t* relc = S.rel + rp0;
        const double* src = Ust + S.upd_off[c];
        int* rw = relw + (k & 1) * 2 * T;
        for (int e = tid; e < ib - ia; e += nthr) rw[e] = relc[ia + e] - r0;
        for (int e = tid; e < jb - ja; e += nthr) rw[T + e] = relc[ja + e] - c0;
        sync();
        for (int j = ja + (tid >> 5); j < jb; j += nthr >> 5) {
            const int dl = rw[T + j - ja];
            const double* sc = src + (int64_t)j * nrc;
            const int i0 = max(ia, j) + lane;
            double v[T / 32];
#pragma unroll
            for (int u = 0; u < T / 32; ++u) v[u] = i0 + 32 * u < ib ? sc[i0 + 32 * u] : 0.0;
#pragma unroll
            for (int u = 0; u < T / 32; ++u)
                if (i0 + 32 * u < ib) tile[tile_idx<T>(rw[i0 + 32 * u - ia], dl)] += v[u];
        }
    }
    sync();
}

// One 64 x 64 tile of the panel columns of a gather front, or of any column of a pre-assembled front,
// per CTA (the batch's assembly tile list): the tile is read as k_scatter / k_zero_upd left it, the
// children's rectangles are added, and each entry is stored once.  256 threads.
constexpr int ASM_T = 64;
__global__ void __launch_bounds__(256)
k_assemble_tiles(DevSym S, const int32_t* __restrict__ batch, const TileEntry* __restrict__ tiles,
                 const TileRect* __restrict__ rects, int gather, double* __restrict__ Lst, double* __restrict__ Ust) {
    __shared__ double tile[ASM_T * ASM_T];
    __shared__ int relw[4 * ASM_T];
    const TileEntry te = tiles[blockIdx.x];
    const int rend = tiles[blockIdx.x + 1].rect;
    const int s = batch[te.slot];
    const int ns = S.sn_first[s + 1] - S.sn_first[s];
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    const int chi = gathers_update(S, s, gather) ? ns : nf;        // a gather front's U is built by the Schur epilogue
    double* Lp = Lst + S.panel_off[s];
    double* Us = Ust + S.upd_off[s];
    const int r0 = te.ti * ASM_T, c0 = te.tj * ASM_T;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    auto column = [&](int d) { return d < ns ? Lp + (int64_t)d * ld : Us + (int64_t)(d - ns) * nr - ns; };
    for (int dl = wid; dl < ASM_T && c0 + dl < chi; dl += 8) {
        const double* col = column(c0 + dl);
#pragma unroll
        for (int u = 0; u < ASM_T / 32; ++u) {
            const int r = r0 + lane + 32 * u;
            if (r >= c0 + dl && r < nf) tile[tile_idx<ASM_T>(lane + 32 * u, dl)] = col[r];
        }
    }
    add_tile_rects<ASM_T>(S, Ust, rects + te.rect, rend - te.rect, r0, c0, tile, relw, tid, 256,
                          [] { __syncthreads(); });
    for (int dl = wid; dl < ASM_T && c0 + dl < chi; dl += 8) {
        double* col = column(c0 + dl);
#pragma unroll
        for (int u = 0; u < ASM_T / 32; ++u) {
            const int r = r0 + lane + 32 * u;
            if (r >= c0 + dl && r < nf) col[r] = tile[tile_idx<ASM_T>(lane + 32 * u, dl)];
        }
    }
}

// acc (4 x 4 per thread, rows tx*4+a, cols ty*4+c) = sum_{k in [k0,k1)} L[rowA0+i, k] D[k] L[rowB0+j, k]
// 64 x 64 tile, 256 threads = 8 warps (2 x 4), each warp 32 x 16 of the tile as 4 x 2 DMMA fragments.
// K-step 16, register prefetch of the next K-slab, double-buffered shared memory with a 72-double
// row stride (conflict-free fragment loads).
__device__ __forceinline__ void ldl_gemm_tile(const double* __restrict__ Lp, int ld, int nf,
                                              const double* __restrict__ Dv, int rowA0, int rowB0,
                                              int k0, int k1, double (&acc)[4][4], double* gsm) {
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
    if (k0 >= k1) return;
    double* As = gsm;                           // [2][GBK][GLD]
    double* Bs = gsm + 2 * GBK * GLD;           // [2][GBK][GLD]
    const int lane = tid & 31, wid = tid >> 5;
    const int wm = (wid & 1) * 32, wn = (wid >> 1) * 16;     // warp origin inside the tile
    const int g = lane >> 2, t = lane & 3;
    double cf[4][2][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) { cf[i][j][0] = 0.0; cf[i][j][1] = 0.0; }
    double ra[4], rb[4];
    auto gload = [&](int kk) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int e = tid + 256 * u, r = e & 63, k = kk + (e >> 6);
            const int ga = rowA0 + r, gb = rowB0 + r;
            ra[u] = (k < k1 && ga < nf) ? Lp[(int64_t)k * ld + ga] : 0.0;
            rb[u] = (k < k1 && gb < nf) ? Lp[(int64_t)k * ld + gb] * Dv[k] : 0.0;
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int e = tid + 256 * u;
            As[(buf * GBK + (e >> 6)) * GLD + (e & 63)] = ra[u];
            Bs[(buf * GBK + (e >> 6)) * GLD + (e & 63)] = rb[u];
        }
    };
    gload(k0);
    sstore(0);
    __syncthreads();
    int buf = 0;
    for (int kk = k0; kk < k1; kk += GBK) {
        const bool more = kk + GBK < k1;
        if (more) gload(kk + GBK);
        const double* Ab = As + buf * GBK * GLD;
        const double* Bb = Bs + buf * GBK * GLD;
#pragma unroll
        for (int k4 = 0; k4 < GBK; k4 += 4) {
            double af[4], bf[2];
#pragma unroll
            for (int i = 0; i < 4; ++i) af[i] = Ab[(k4 + t) * GLD + wm + 8 * i + g];
#pragma unroll
            for (int j = 0; j < 2; ++j) bf[j] = Bb[(k4 + t) * GLD + wn + 8 * j + g];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) dmma884(cf[i][j][0], cf[i][j][1], af[i], bf[j]);
        }
        if (more) sstore(buf ^ 1);
        __syncthreads();
        buf ^= 1;
    }
    double* Cs = gsm;                           // 64 x 65 doubles, aliases the operand buffers
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int r = wm + 8 * i + g, c = wn + 8 * j + 2 * t;
            Cs[r * 65 + c] = cf[i][j][0];
            Cs[r * 65 + c + 1] = cf[i][j][1];
        }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = Cs[(tx * 4 + a) * 65 + ty * 4 + c];
    __syncthreads();
}

__global__ void __launch_bounds__(256)
k_ldl_update_ldg(DevSym S, const int32_t* __restrict__ batch, const TileEntry* __restrict__ tiles,
                 const TileRect* __restrict__ rects, int mode, int J0, int na, int gather,
                 double* __restrict__ Lst, double* __restrict__ Ust, const double* __restrict__ D) {
    __shared__ double gsm[GSM];
    __shared__ int relw[4 * GBM];
    static_assert(GBM * GBM <= GSM, "the gathered tile aliases the operand buffers");
    const TileEntry te = mode == 1 ? tiles[blockIdx.x] : TileEntry{(int32_t)blockIdx.y, 0, 0, 0};
    const int s = batch[te.slot];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    const UpdTile u = decode_update_tile<GBM>(mode, J0, na, ns, nf, te);
    if (!u.valid) return;
    double* Lp = Lst + S.panel_off[s];
    double acc[4][4];
    ldl_gemm_tile(Lp, ld, nf, D + f, u.ti * GBM, u.tj * GBM, u.k0, u.k1, acc, gsm);
    const bool gat = mode == 1 && gathers_update(S, s, gather);
    if (gat) {                                  // the tile aliases the operand buffers (free after ldl_gemm_tile)
        for (int e = threadIdx.x; e < GBM * GBM; e += 256) gsm[e] = 0.0;
        add_tile_rects<GBM>(S, Ust, rects + te.rect, tiles[blockIdx.x + 1].rect - te.rect, u.ti * GBM, u.tj * GBM,
                            gsm, relw, threadIdx.x, 256, [] { __syncthreads(); });
    }
    double* Us = Ust + S.upd_off[s];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double cv[4][4];
    double* dc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int col = u.tj * GBM + ty * 4 + c;
        const bool okc = col >= u.c_lo && col < u.c_hi;
        dc[c] = col < ns ? Lp + (int64_t)col * ld : Us + (int64_t)(col - ns) * nr - ns;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int row = u.ti * GBM + tx * 4 + a;
            cv[a][c] = !(okc && row < nf && row >= col) ? 0.0
                     : gat ? gsm[tile_idx<GBM>(row - u.ti * GBM, col - u.tj * GBM)] : dc[c][row];
        }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int col = u.tj * GBM + ty * 4 + c;
        const bool okc = col >= u.c_lo && col < u.c_hi;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int row = u.ti * GBM + tx * 4 + a;
            if (okc && row < nf && row >= col) dc[c][row] = cv[a][c] - acc[a][c];
        }
    }
}

// ---- TMA-fed version -------------------------------------------------------------------------
constexpr int TB = 128;                         // large CTA tile (rows and columns); the small one is 64
constexpr int TK = 16;                          // k-slab per pipeline stage
constexpr int TSTAGES = 4;
// tile T x T: consumer warps (T/64 x T/32 for T = 128: warp tile 64 x 32; 2 x 2 for T = 64: warp tile 32 x 32)
// plus one producer warp
constexpr int tma_threads(int T) { return (T == 128 ? 8 : 4) * 32 + 32; }
// stage ring (the gathered tile aliases it), full / empty barriers, rel windows of add_tile_rects
constexpr size_t tma_gemm_smem(int T) {
    return (size_t)TSTAGES * 2 * T * TK * sizeof(double) + 2 * TSTAGES * sizeof(uint64_t) + 4 * T * sizeof(int);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n\t}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 3-D tiled TMA load: box -> shared memory, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n"
                 :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// The tensor map of a panel views it as (8 rows, k, row-groups of 8) with strides (8 B, ld*8 B, 64 B):
// a box (8, TK, TB/8) lands in shared memory as [row-group][k][8 rows], so the four k-lanes of a DMMA
// fragment load read 32 consecutive doubles (conflict-free).  If the driver rejects that dimension
// order the natural one (8 rows, row-groups, k) is used: layout [k][row-group][8], strides passed in
// (sk, srg) - same kernel, 4-way bank conflicts on the fragment loads.
template <int T>
__global__ void __launch_bounds__(tma_threads(T), T == 128 ? 1 : 3)
k_ldl_update_tma(DevSym S, const int32_t* __restrict__ batch, const TileEntry* __restrict__ tiles,
                 const TileRect* __restrict__ rects, const CUtensorMap* __restrict__ maps,
                 const int32_t* __restrict__ map_of, int mode, int J0, int na, int gather, int kmajor,
                 double* __restrict__ Lst, double* __restrict__ Ust, const double* __restrict__ D) {
    extern __shared__ __align__(128) unsigned char tma_smem[];
    static_assert(T * T <= 2 * TSTAGES * T * TK, "the gathered tile aliases the stage ring");
    const TileEntry te = mode == 1 ? tiles[blockIdx.x] : TileEntry{(int32_t)blockIdx.y, 0, 0, 0};
    const int s = batch[te.slot];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nr = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    const UpdTile u = decode_update_tile<T>(mode, J0, na, ns, nf, te);
    if (!u.valid) return;
    double* sA = reinterpret_cast<double*>(tma_smem);
    constexpr int TTILE = T * TK;                      // doubles per operand per stage
    constexpr int NCW = T == 128 ? 8 : 4;              // consumer warps
    constexpr int WM = T == 128 ? 64 : 32, WN = 32;    // warp tile
    constexpr int MI = WM / 16, NJ = WN / 8;
    double* sB = sA + TSTAGES * TTILE;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + TSTAGES * TTILE);
    uint64_t* empty = full + TSTAGES;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int nk = (u.k1 - u.k0 + TK - 1) / TK;
    if (tid == 0) {
#pragma unroll
        for (int st = 0; st < TSTAGES; ++st) { mbar_init(full + st, 1); mbar_init(empty + st, NCW); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (wid == NCW) {
        // ===== TMA producer (one lane) =====
        if (lane == 0) {
            const CUtensorMap* tm = maps + map_of[s];
            for (int it = 0; it < nk; ++it) {
                const int st = it % TSTAGES;
                const uint32_t ph = (uint32_t)(it / TSTAGES) & 1u;
                mbar_wait(empty + st, ph ^ 1u);                      // slot free (passes at once on a fresh barrier)
                mbar_expect_tx(full + st, 2u * TTILE * (uint32_t)sizeof(double));
                const int kc = u.k0 + it * TK;
                if (kmajor & 1) {
                    tma_load_3d(sA + st * TTILE, tm, full + st, 0, kc, u.ti * (T / 8));
                    tma_load_3d(sB + st * TTILE, tm, full + st, 0, kc, u.tj * (T / 8));
                } else {
                    tma_load_3d(sA + st * TTILE, tm, full + st, 0, u.ti * (T / 8), kc);
                    tma_load_3d(sB + st * TTILE, tm, full + st, 0, u.tj * (T / 8), kc);
                }
            }
        }
        return;
    }
    // ===== 8 consumer warps (2 x 4), warp tile 64 x 32 = 4 x 4 DMMA m16n8k16 tiles per k-slab =====
    const int sk = (kmajor & 1) ? 8 : T, srg = (kmajor & 1) ? TK * 8 : 8;       // strides (doubles) of k and of a row-group
    const int wm = (wid & 1) * WM, wn = (wid >> 1) * WN;
    const int g = lane >> 2, t = lane & 3;
    const double* Dv = D + f;
    double acc[MI][NJ][4];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;
    for (int it = 0; it < nk; ++it) {
        const int st = it % TSTAGES;
        const uint32_t ph = (uint32_t)(it / TSTAGES) & 1u;
        double dv[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) { const int k = u.k0 + it * TK + 4 * v + t; dv[v] = (k < u.k1) ? Dv[k] : 0.0; }
        mbar_wait(full + st, ph);
        // Release of the PREVIOUS stage, one iteration late and after the wait above.  Releasing a stage at
        // the end of its own iteration is not safe: ptxas schedules the SYNCS.ARRIVE right behind the last
        // LDS *issue* (before the DMMAs that consume them - it did, DESIGN.md section 4),
        // the arrive does not wait for loads in flight, and with 3 CTAs per SM an LDS can be overtaken by
        // the TMA refill of its stage: rare corrupted tiles, seen on sm_100a.  Here
        // every DMMA of stage it-1 was issued before the spin-wait (they cannot sink below its loop), a DMMA
        // issues only when its LDS operands have arrived, and the arrive cannot rise above the acquire.
        if (it > 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + (it - 1) % TSTAGES);
        }
        const double* A = sA + st * TTILE + (wm / 8) * srg + g;
        const double* B = sB + st * TTILE + (wn / 8) * srg + g;
        // All A fragments stay live while the B fragments stream past them one n8 tile at a time
        // (MI x 8 + 4 doubles).  Holding all NJ B fragments instead made sm_90a spill the T = 64 loop
        // under its 3-CTA/SM budget of 128 registers.
        double af[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int v = 0; v < 4; ++v)
#pragma unroll
                for (int h = 0; h < 2; ++h) af[i][2 * v + h] = A[(2 * i + h) * srg + (4 * v + t) * sk];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            double bf[4];
#pragma unroll
            for (int v = 0; v < 4; ++v) bf[v] = B[j * srg + (4 * v + t) * sk] * dv[v];
#pragma unroll
            for (int i = 0; i < MI; ++i) dmma16816(acc[i][j], af[i], bf);
        }
    }
    // ===== epilogue: subtract into the panel (col < ns) or the update block.  All loads of a column
    // pair are issued before the first store (a plain  *p -= v  loop serialises 64 load->store chains).
    // A gather front's U tile is built in the stage ring instead: every stage has been waited on, so
    // no TMA write is in flight, and the producer warp has returned (named barrier 1, consumers only).
    const bool gat = mode == 1 && gathers_update(S, s, gather);
    if (gat) {
        auto sync = [] { asm volatile("bar.sync 1, %0;\n" :: "n"(NCW * 32) : "memory"); };
        sync();                                        // every consumer is done reading the ring
        for (int e = tid; e < T * T; e += NCW * 32) sA[e] = 0.0;
        const int rb = tiles[blockIdx.x].rect;
        add_tile_rects<T>(S, Ust, rects + rb, tiles[blockIdx.x + 1].rect - rb, u.ti * T, u.tj * T, sA,
                          reinterpret_cast<int*>(empty + TSTAGES), tid, NCW * 32, sync);
    }
    double* Lp = Lst + S.panel_off[s];
    double* Us = Ust + S.upd_off[s];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
        double cv[2][2 * MI];
        double* dc[2];
        bool okc[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = u.tj * T + wn + 8 * j + 2 * t + e;
            okc[e] = col >= u.c_lo && col < u.c_hi;
            dc[e] = col < ns ? Lp + (int64_t)col * ld : Us + (int64_t)(col - ns) * nr - ns;
#pragma unroll
            for (int i = 0; i < 2 * MI; ++i) {
                const int row = u.ti * T + wm + 8 * i + g;
                cv[e][i] = !(okc[e] && row < nf && row >= col) ? 0.0
                         : gat ? sA[tile_idx<T>(row - u.ti * T, col - u.tj * T)] : dc[e][row];
            }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = u.tj * T + wn + 8 * j + 2 * t + e;
#pragma unroll
            for (int i = 0; i < 2 * MI; ++i) {
                const int row = u.ti * T + wm + 8 * i + g;
                // row group i = 2 * (m16 tile) + h  ->  acc[i >> 1][j][2 * (i & 1) + e]
                if (okc[e] && row < nf && row >= col) dc[e][row] = cv[e][i] - acc[i >> 1][j][2 * (i & 1) + e];
            }
        }
    }
}

// Pivot block J of the large fronts of a level: LDL' + inverse of the 64 x 64 diagonal block.
// Parks [inv(L_JJ) strictly lower ; d on the diagonal] in the workspace.  One CTA per front.
// 256 threads, thread (tx, ty) keeps the 4 x 4 tile (rows 4tx.., cols 4ty..) of the block AND of
// X = inv(L) in registers.  One barrier per pivot: the owners of column k publish it (and the
// owners of row k of X publish that row) in a double-buffered shared vector, then every thread
// applies the rank-1 updates  A -= a_k a_k' / d_k  and  X -= l_k X[k,:]  to its own tiles
// (inv(L) = (I - l_63 e_63') ... (I - l_0 e_0') applied to the identity, fused into the same sweep).
// The sign-based dynamic regularisation (QDLDL: D[k]*sign < eps => D[k] = delta*sign) is evaluated
// redundantly by every thread on the published pivot.
__global__ void __launch_bounds__(256)
k_piv_diag(DevSym S, const int32_t* __restrict__ batch, int J0, const double* __restrict__ Lst,
           double* __restrict__ Wst, const int64_t* __restrict__ woff, double* __restrict__ D,
           double* __restrict__ Dinv, RegParams rp, unsigned int* __restrict__ nreg) {
    __shared__ double colbuf[2][PB];            // column k of the (updated) block, unscaled
    __shared__ double rowbuf[2][PB];            // row k of X
    __shared__ double sgn[PB];
    const int s = batch[blockIdx.x];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    if (J0 >= ns) return;
    const int ld = S.ld[s];
    const int nb = min(PB, ns - J0);
    const double* Lp = Lst + S.panel_off[s];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    double a[4][4], x[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int i = 4 * tx + r, j = 4 * ty + c;
            double v = (i == j) ? 1.0 : 0.0;                     // identity beyond nb
            if (i < nb && j < nb) v = (i >= j) ? Lp[(int64_t)(J0 + j) * ld + J0 + i] : 0.0;
            a[r][c] = v;
            x[r][c] = (i == j) ? 1.0 : 0.0;
        }
    if (tid < PB) sgn[tid] = tid < nb ? (double)S.dsign[f + J0 + tid] : 1.0;
    unsigned int myreg = 0;
#pragma unroll 1
    for (int kq = 0; kq < PB / 4; ++kq) {
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
            const int k = 4 * kq + kc;
            double* cb = colbuf[k & 1];
            double* rb = rowbuf[k & 1];
            if (ty == kq) {
#pragma unroll
                for (int r = 0; r < 4; ++r) cb[4 * tx + r] = a[r][kc];
            }
            if (tx == kq) {
#pragma unroll
                for (int c = 0; c < 4; ++c) rb[4 * ty + c] = x[kc][c];
            }
            __syncthreads();
            double d = cb[k];
            const double sg = sgn[k];
            bool reg = false;
            if (k < nb && rp.enable && d * sg < rp.eps) { d = rp.delta * sg; reg = true; }
            const double dinv = 1.0 / d;
            if (tid == 0) { if (k < nb) { D[f + J0 + k] = d; Dinv[f + J0 + k] = dinv; } if (reg) { ++myreg; note_reg(rp, nreg, f + J0 + k); } }
            double li[4], cj[4], xr[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) { const int i = 4 * tx + r; li[r] = (i > k) ? cb[i] * dinv : 0.0; }
#pragma unroll
            for (int c = 0; c < 4; ++c) { const int j = 4 * ty + c; cj[c] = (j > k) ? cb[j] : 0.0; xr[c] = rb[j]; }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) { a[r][c] -= li[r] * cj[c]; x[r][c] -= li[r] * xr[c]; }
            if (ty == kq) {
#pragma unroll
                for (int r = 0; r < 4; ++r) { const int i = 4 * tx + r; if (i > k) a[r][kc] = li[r]; else if (i == k) a[r][kc] = d; }
            }
        }
    }
    (void)myreg;
    // park [inv(L_JJ) strictly lower ; d on the diagonal] (column-major 64 x 64)
    double* Wd = Wst + woff[blockIdx.x] + (int64_t)(J0 / PB) * (PB * PB);
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int i = 4 * tx + r, j = 4 * ty + c;
            double v = (i == j) ? 1.0 : 0.0;
            if (i < nb && j < nb) { if (i > j) v = x[r][c]; else if (i == j) v = a[r][c]; }
            Wd[i + j * PB] = v;
        }
}

// L[rows, J] = F[rows, J] * inv(L_JJ)' * D_J^-1 for a 64-row tile below the pivot block.
// grid (row tiles, nbatch), dynamic smem 2 * 64 * 65 doubles.
__global__ void __launch_bounds__(256)
k_piv_rows(DevSym S, const int32_t* __restrict__ batch, int J0, double* __restrict__ Lst,
           const double* __restrict__ Wst, const int64_t* __restrict__ woff,
           const double* __restrict__ Dinv) {
    extern __shared__ double smem[];
    double* Ts = smem;                                // T: 64 rows x 65 (k index fastest -> [i][k])
    double* Ms = Ts + PB * (PB + 1);                  // M[k][j], 64 x 65
    const int s = batch[blockIdx.y];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    if (J0 >= ns) return;
    const int nf = ns + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int ld = S.ld[s];
    const int nb = min(PB, ns - J0);
    const int r0 = J0 + nb + blockIdx.x * GBM;
    if (r0 >= nf) return;
    double* Lp = Lst + S.panel_off[s];
    const int tid = threadIdx.x;
    for (int e = tid; e < PB * PB; e += 256) {
        const int i = e & (PB - 1), k = e >> 6;
        const int gr = r0 + i;
        Ts[i * (PB + 1) + k] = (gr < nf && k < nb) ? Lp[(int64_t)(J0 + k) * ld + gr] : 0.0;
    }
    const double* Wd = Wst + woff[blockIdx.y] + (int64_t)(J0 / PB) * (PB * PB);
    for (int e = tid; e < PB * PB; e += 256) {
        const int jj = e % PB, kk = e / PB;          // Wd[jj + kk*PB] = inv(L_JJ)[jj][kk] (jj > kk)
        double v = 0.0;
        if (jj < nb && kk < nb) {
            if (jj > kk) v = Wd[e] * Dinv[f + J0 + jj];
            else if (jj == kk) v = Dinv[f + J0 + jj];
        }
        Ms[kk * (PB + 1) + jj] = v;                  // M[k][j] = inv(L)[j][k] * dinv[j], k <= j
    }
    __syncthreads();
    // L[rows, J] = T * M : out[i][j] = sum_{k <= j} T[i][k] M[k][j]  on the FP64 tensor-core path
    // (8 warps as 2 x 4, warp tile 32 x 16 = 4 x 2 DMMA fragments, K = 64)
    const int lane = tid & 31, wid = tid >> 5;
    const int wm = (wid & 1) * 32, wn = (wid >> 1) * 16;
    const int g = lane >> 2, t = lane & 3;
    double cf[4][2][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) { cf[i][j][0] = 0.0; cf[i][j][1] = 0.0; }
#pragma unroll 4
    for (int k4 = 0; k4 < PB; k4 += 4) {
        double af[4], bf[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) af[i] = Ts[(wm + 8 * i + g) * (PB + 1) + k4 + t];
#pragma unroll
        for (int j = 0; j < 2; ++j) bf[j] = Ms[(k4 + t) * (PB + 1) + wn + 8 * j + g];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) dmma884(cf[i][j][0], cf[i][j][1], af[i], bf[j]);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = wn + 8 * j + 2 * t + e;
            if (col >= nb) continue;
            double* cp_ = Lp + (int64_t)(J0 + col) * ld;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int gr = r0 + wm + 8 * i + g;
                if (gr < nf) cp_[gr] = cf[i][j][e];
            }
        }
}

// Finish the large fronts of a level: copy the parked blocks [inv(L_JJ) strictly lower ; d on the
// diagonal] into the panel (the solve kernels expect inverted SB x SB diagonal blocks, SB == PB).
// grid (max blocks per front, nbatch), 256 threads.
__global__ void __launch_bounds__(256)
k_finish_large(DevSym S, const int32_t* __restrict__ batch, double* __restrict__ Lst,
               const double* __restrict__ Wst, const int64_t* __restrict__ woff) {
    const int s = batch[blockIdx.y];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int kb = blockIdx.x * PB;
    if (kb >= ns) return;
    const int nf = ns + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int ld = S.ld[s];
    const int sb = min(PB, ns - kb);
    double* Lp = Lst + S.panel_off[s] + (int64_t)kb * ld + kb;
    const double* Wd = Wst + woff[blockIdx.y] + (int64_t)blockIdx.x * (PB * PB);
    for (int e = threadIdx.x; e < PB * PB; e += 256) {
        const int i = e % PB, j = e / PB;
        if (i < sb && j < sb && i >= j) Lp[i + (int64_t)j * ld] = Wd[e];
    }
}

// ------------------------------------------------------------------ scatter / regularisation
__global__ void k_scatter(const double* __restrict__ nz, const int64_t* __restrict__ amap,
                          int64_t n, double* __restrict__ Lst) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) Lst[amap[i]] = nz[i];
}

__global__ void k_diag_absmax(const double* __restrict__ nz, const int64_t* __restrict__ didx,
                              int64_t n, unsigned long long* __restrict__ out) {
    double m = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x)
        m = fmax(m, fabs(nz[didx[i]]));
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(m));
}

// eps = c + p * max|diag|   (_compute_regularizer, kktsolver_directldl.jl:297-310)
__global__ void k_compute_eps(const unsigned long long* maxbits, double c, double p, double* eps) {
    // separate rounding of the product and the sum, like the reference's scalar code
    *eps = __dadd_rn(c, __dmul_rn(p, __longlong_as_double((long long)*maxbits)));
}

// Lst[amap[didx[i]]] = nz[didx[i]] + sign_i * eps  (static regularisation, :266-273; the
// unshifted nz is kept for the refinement residuals, :283-291)
__global__ void k_shift_diag(const double* __restrict__ nz, const int64_t* __restrict__ didx,
                             const int64_t* __restrict__ amap, const int8_t* __restrict__ dsign_orig,
                             const double* __restrict__ eps, int64_t n, double* __restrict__ Lst) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) {
        const int64_t k = didx[i];
        Lst[amap[k]] = nz[k] + (dsign_orig[i] > 0 ? *eps : -*eps);
    }
}

// ------------------------------------------------------------------ G7 triangular solves
__global__ void k_pack_perm(const double* __restrict__ b, const int32_t* __restrict__ perm,
                            int64_t n, double* __restrict__ y) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) y[i] = b[perm[i]];
}
__global__ void k_unpack_perm(const double* __restrict__ y, const int32_t* __restrict__ perm,
                              int64_t n, double* __restrict__ x) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) x[perm[i]] = y[i];
}

// Forward sweep, multifrontal form (deterministic, no atomics): per supernode
//   w = [y_s ; 0] + sum_children extend(u_c);
//   for each SB block kb:  x = inv(L_kb,kb) w_kb ;  w[kb+sb:] -= L[kb+sb:, kb:kb+sb] x
//   y_s = w[0:ns],  u_s = w[ns:]
// Backward sweep:  w = [D^-1 y_s ; x[R_s]] ;  for kb descending:
//   t = w_kb - L[kb+sb:, kb:kb+sb]' w[kb+sb:] ;  w_kb = inv(L_kb,kb)' t


// ---- latency-tolerant building blocks: all global loads of a step are issued as one batch of
// independent loads (every L entry is used exactly once per solve, so the only thing that
// matters is memory-level parallelism).

// acc = sum_{j=q,q+4,...<i} row[j*ld] * w[j]   (j < SB), 16 loads in flight
__device__ __forceinline__ double diag_row_dot(const double* __restrict__ row, int64_t ld, int i, int q,
                                               const double* __restrict__ w) {
    double v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; v[u] = (j < i) ? row[(int64_t)j * ld] : 0.0; }
    double acc = 0.0;
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; if (j < i) acc += v[u] * w[j]; }
    return acc;
}

// acc = sum_{j<sb} rowp[j*ld] * x[j]   (sb <= 64), two batches of 32 loads
__device__ __forceinline__ double row_dot64(const double* __restrict__ rowp, int64_t ld, int sb,
                                            const double* __restrict__ x) {
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int jb = 0; jb < 64; jb += 32) {
        if (jb < sb) {
            double v[32];
#pragma unroll
            for (int u = 0; u < 32; ++u) v[u] = (jb + u < sb) ? rowp[(int64_t)(jb + u) * ld] : 0.0;
#pragma unroll
            for (int u = 0; u < 32; u += 2) { a0 += v[u] * x[jb + u]; a1 += v[u + 1] * x[jb + u + 1]; }
        }
    }
    return a0 + a1;
}

// Transposed products for 8 consecutive columns at once: out[u] = sum_{r=r0+lane,+32,..<r1} col_u[r]*w[r]
// (warp-level; result valid on all lanes after the shuffles)
// Sum 8 per-lane partial sums over the warp through shared memory: lane u (< 8) returns sum_u.
// (Shuffle trees inside loops whose trip count comes from memory are wrapped in WARPSYNC.COLLECTIVE
// by the compiler; `red` is 8 x 33 doubles owned by the warp.)
__device__ __forceinline__ double warp_sum8_smem(const double (&a)[8], double* red, int lane) {
#pragma unroll
    for (int u = 0; u < 8; ++u) red[u * 33 + lane] = a[u];
    __syncwarp();
    double s = 0.0;
    if (lane < 8) {
#pragma unroll
        for (int l = 0; l < 32; ++l) s += red[lane * 33 + l];
    }
    __syncwarp();
    return s;
}

// Transposed products for 8 consecutive columns at once: sum_{r=r0+lane,+32,..<r1} col_u[r]*w[r];
// lane u (< 8) returns the sum of column u.
__device__ __forceinline__ double cols8_dot(const double* __restrict__ base, int64_t ld, int ncol,
                                            int r0, int r1, const double* __restrict__ w, int lane,
                                            double* red) {
    double a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] = 0.0;
    for (int r = r0 + lane; r < r1; r += 64) {
        double v0[8], v1[8];
        const bool two = (r + 32) < r1;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            v0[u] = (u < ncol) ? base[(int64_t)u * ld + r] : 0.0;
            v1[u] = (u < ncol && two) ? base[(int64_t)u * ld + r + 32] : 0.0;
        }
        const double w0 = w[r], w1 = two ? w[r + 32] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; ++u) a[u] += v0[u] * w0 + v1[u] * w1;
    }
    return warp_sum8_smem(a, red, lane);
}

// --- supernodes with a single pivot column and a short front: one thread per supernode
__global__ void __launch_bounds__(128)
k_fwd_leaf(DevSym S, const int32_t* __restrict__ batch, int count, const double* __restrict__ Lst,
           double* __restrict__ y, double* __restrict__ uvec) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int s = batch[idx];
    const int f = S.sn_first[s];
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const double* Lp = Lst + S.panel_off[s];
    if (S.child_ptr[s + 1] == S.child_ptr[s]) {          // true leaf: no contributions to gather
        const double x = y[f];
        for (int i = 0; i < nr; ++i) uvec[rp + i] = -Lp[1 + i] * x;
        return;
    }
    const int32_t* cp = S.asm_colptr + S.front_ptr[s];
    const int64_t base = S.asm_base[s];
    double x = y[f];
    for (int e = cp[0]; e < cp[1]; ++e) x += uvec[S.asm_src[base + e]];
    y[f] = x;
    for (int i = 0; i < nr; ++i) {
        double acc = 0.0;
        for (int e = cp[1 + i]; e < cp[2 + i]; ++e) acc += uvec[S.asm_src[base + e]];
        uvec[rp + i] = acc - Lp[1 + i] * x;
    }
}
__global__ void __launch_bounds__(128)
k_bwd_leaf(DevSym S, const int32_t* __restrict__ batch, int count, const double* __restrict__ Lst,
           const double* __restrict__ Dinv, double* __restrict__ y) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int s = batch[idx];
    const int f = S.sn_first[s];
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const double* Lp = Lst + S.panel_off[s];
    double acc = y[f] * Dinv[f];
    for (int i = 0; i < nr; ++i) acc -= Lp[1 + i] * y[S.rows[rp + i]];
    y[f] = acc;
}

// --- narrow supernodes (ns <= 32, nf <= 192): one warp per supernode, WPB warps per CTA.
// Every L entry is used exactly once per sweep, so what matters is memory-level parallelism: each
// phase issues ALL its loads (up to 32 per lane, one per pivot column, coalesced across lanes)
// before the first use; a supernode costs ~4 dependent memory latencies instead of ~ns.
constexpr int WPB = 8;

// lane l <- sum over lanes of p[l]  (32 accumulators per lane, 31 shuffles, fixed order => deterministic)
__device__ __forceinline__ double warp_transpose_reduce(double (&p)[32], int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool hi = (lane & off) != 0;
#pragma unroll
        for (int idx = 0; idx < off; ++idx) {
            const double send = hi ? p[idx] : p[idx + off];
            const double keep = hi ? p[idx + off] : p[idx];
            p[idx] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return p[0];
}

// Everything a narrow-supernode solve step needs to know about its supernode, packed so that the
// level-scheduled kernels fetch it with ONE round trip (batch position -> descriptor) instead of two
// (batch position -> supernode id -> seven separate arrays).  64 bytes, built per batch entry.
struct SolveDesc {
    int32_t f, ns, nr, ld;
    int32_t nchild, pad;
    int64_t panel_off, rows_ptr, front_ptr, asm_base;
    int64_t pad2;
};
struct SnView {                 // the same data as raw pointers
    int f, ns, nr, ld; bool has_children;
    const double* Lp; int64_t rp; const int32_t* cp; const int32_t* asrc; const int32_t* rows;
};
__device__ __forceinline__ SnView view_of(const DevSym& S, const SolveDesc& d, const double* Lst) {
    SnView v; v.f = d.f; v.ns = d.ns; v.nr = d.nr; v.ld = d.ld; v.has_children = d.nchild != 0;
    v.Lp = Lst + d.panel_off; v.rp = d.rows_ptr; v.cp = S.asm_colptr + d.front_ptr; v.asrc = S.asm_src + d.asm_base;
    v.rows = S.rows + d.rows_ptr;
    return v;
}
__device__ __forceinline__ SnView view_of(const DevSym& S, int s, const double* Lst) {
    SnView v; v.f = S.sn_first[s]; v.ns = S.sn_first[s + 1] - v.f; v.rp = S.rows_ptr[s];
    v.nr = (int)(S.rows_ptr[s + 1] - v.rp); v.ld = S.ld[s]; v.has_children = S.child_ptr[s + 1] != S.child_ptr[s];
    v.Lp = Lst + S.panel_off[s]; v.cp = S.asm_colptr + S.front_ptr[s]; v.asrc = S.asm_src + S.asm_base[s];
    v.rows = S.rows + v.rp;
    return v;
}

// Forward step of one narrow supernode (ns <= NW) by one warp.  Y / U are the solution / contribution
// vectors addressed with GLOBAL indices: in the level-scheduled kernels they are the global arrays, in
// the subtree kernels they are shared-memory windows shifted by the window origin.
template <int NW>
__device__ __forceinline__ void fwd_warp_body(const SnView& V, double* Y, double* U, double* w, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    // Row `lane` of the first 32 panel rows, all of it in flight before anything else: for lane < ns that
    // is the inverted triangle (columns j < lane), for ns <= lane < nf the first chunk of L21 (all ns
    // columns).  Fronts with nf <= 32 - the bottom level, most of the bytes of this class - then need no
    // further L round trip.  The loads do not depend on the gathered right-hand side.
    double v[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) v[j] = (j < lane && j < ns && lane < nf) ? Lp[(int64_t)j * ld + lane] : 0.0;
    if (V.has_children) {
        for (int i = lane; i < nf; i += 32) {
            double acc = i < ns ? Y[f + i] : 0.0;
            for (int e = V.cp[i]; e < V.cp[i + 1]; ++e) acc += U[V.asrc[e]];
            w[i] = acc;
        }
    } else {
        for (int i = lane; i < nf; i += 32) w[i] = i < ns ? Y[f + i] : 0.0;
    }
    __syncwarp();
    // x = inv(L11) w_top : x_i = w_i + sum_{j<i} X[i][j] w_j
    double xi = 0.0;
    if (lane < ns) {
        xi = w[lane];
#pragma unroll
        for (int j = 0; j < NW; ++j) if (j < ns) xi += v[j] * w[j];
    }
    __syncwarp();
    if (lane < ns) { w[lane] = xi; Y[f + lane] = xi; }
    __syncwarp();
    // u = w_bot - L21 x : rows ns..31 from the registers loaded above
    if (lane >= ns && lane < nf) {
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < NW; j += 2) { if (j < ns) a0 += v[j] * w[j]; if (j + 1 < ns) a1 += v[j + 1] * w[j + 1]; }
        U[V.rp + lane - ns] = w[lane] - (a0 + a1);
    }
    // rows 32.. : one row per lane, all ns column loads of a row in flight together
    for (int r = 32 + lane; r < nf; r += 32) {
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns) ? Lp[(int64_t)j * ld + r] : 0.0;
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < NW; j += 2) { if (j < ns) a0 += v[j] * w[j]; if (j + 1 < ns) a1 += v[j + 1] * w[j + 1]; }
        U[V.rp + r - ns] = w[r] - (a0 + a1);
    }
}

// Backward step of one narrow supernode by one warp.  Columns in [win_lo, win_hi) are read from the
// window Y, all others (ancestors outside a subtree) from the global solution vector yg.
// The transposed products go through a 32 x (NW+1) shared tile (coalesced loads by rows, conflict-free
// reads by columns) instead of shuffle reductions: inside the loops of the subtree kernel the compiler
// cannot prove warp convergence and wraps every shuffle in WARPSYNC.COLLECTIVE (tens of cycles each).
constexpr int BT_LD = 33;
template <int NW>
__device__ __forceinline__ void bwd_warp_body(const SnView& V, const double* __restrict__ Dinv, double* Y,
                                              const double* yg, int win_lo, int win_hi, double* w,
                                              double* tile, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    constexpr int TL = NW + 1;
    // row `lane` of the first 32 panel rows (see fwd_warp_body): triangle X[lane][j], j < lane, for
    // lane < ns; first chunk of L21 for ns <= lane < nf.  Independent of the gather below.
    double xr[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) xr[j] = (j < lane && j < ns && lane < nf) ? Lp[(int64_t)j * ld + lane] : 0.0;
    for (int i = lane; i < nf; i += 32) {
        double val;
        if (i < ns) val = Y[f + i] * Dinv[f + i];
        else { const int c = V.rows[i - ns]; val = (c >= win_lo && c < win_hi) ? Y[c] : yg[c]; }
        w[i] = val;
    }
#pragma unroll
    for (int j = 0; j < NW; ++j) tile[lane * TL + j] = xr[j];
    __syncwarp();
    // t_j = w_j - sum_{r >= ns} L[r][j] w_r   (lane j owns column j); rows ns..31 sit in the tile already
    double acc = 0.0;
    if (lane < NW) {
#pragma unroll
        for (int rr = 0; rr < 32; ++rr) if (rr >= ns && rr < nf) acc += tile[rr * TL + lane] * w[rr];
    }
    for (int r0 = 32; r0 < nf; r0 += 32) {
        const int r = r0 + lane;
        double v[NW];
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns && r < nf) ? Lp[(int64_t)j * ld + r] : 0.0;
        __syncwarp();                              // the previous tile has been consumed
#pragma unroll
        for (int j = 0; j < NW; ++j) tile[lane * TL + j] = v[j];
        __syncwarp();
        if (lane < NW) {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) if (r0 + rr < nf) acc += tile[rr * TL + lane] * w[r0 + rr];
        }
    }
    const double tj = (lane < ns) ? w[lane] - acc : 0.0;
    // x_j = t_j + sum_{i>j} X[i][j] t_i
    __syncwarp();                                  // everyone has read w[0..nf) and the last tile
    if (nf > 32) {
#pragma unroll
        for (int j = 0; j < NW; ++j) tile[lane * TL + j] = xr[j];
    }
    w[lane] = tj;                                  // t (zero beyond ns)
    __syncwarp();
    double corr = 0.0;
    if (lane < NW) {
#pragma unroll
        for (int i = 0; i < NW; ++i) if (i < ns) corr += tile[i * TL + lane] * w[i];
    }
    if (lane < ns) Y[f + lane] = tj + corr;
    __syncwarp();
}

// The previous formulation (triangle and L21 rows loaded in two separate phases): kept selectable
// (CB200_SPLIT_ROWS=1) so that the merged-load bodies above can be measured against it on the same build.
template <int NW>
__device__ __forceinline__ void fwd_warp_body_split(const SnView& V, double* Y, double* U, double* w, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    // the triangle loads do not depend on the gathered right-hand side: issue them first
    double v[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) v[j] = (j < lane && lane < ns) ? Lp[(int64_t)j * ld + lane] : 0.0;
    if (V.has_children) {
        for (int i = lane; i < nf; i += 32) {
            double acc = i < ns ? Y[f + i] : 0.0;
            for (int e = V.cp[i]; e < V.cp[i + 1]; ++e) acc += U[V.asrc[e]];
            w[i] = acc;
        }
    } else {
        for (int i = lane; i < nf; i += 32) w[i] = i < ns ? Y[f + i] : 0.0;
    }
    __syncwarp();
    // x = inv(L11) w_top : x_i = w_i + sum_{j<i} X[i][j] w_j
    double xi = (lane < ns) ? w[lane] : 0.0;
#pragma unroll
    for (int j = 0; j < NW; ++j) if (j < ns) xi += v[j] * w[j];
    __syncwarp();
    if (lane < ns) { w[lane] = xi; Y[f + lane] = xi; }
    __syncwarp();
    // u = w_bot - L21 x : one row per lane, all ns column loads of a row in flight together
    for (int r = ns + lane; r < nf; r += 32) {
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns) ? Lp[(int64_t)j * ld + r] : 0.0;
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < NW; j += 2) { if (j < ns) a0 += v[j] * w[j]; if (j + 1 < ns) a1 += v[j + 1] * w[j + 1]; }
        U[V.rp + r - ns] = w[r] - (a0 + a1);
    }
}

template <int NW>
__device__ __forceinline__ void bwd_warp_body_split(const SnView& V, const double* __restrict__ Dinv, double* Y,
                                              const double* yg, int win_lo, int win_hi, double* w,
                                              double* tile, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    constexpr int TL = NW + 1;
    // the triangle (row `lane`): X[lane][j], j < lane - independent of the gather below
    double xr[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) xr[j] = (j < lane && lane < ns) ? Lp[(int64_t)j * ld + lane] : 0.0;
    for (int i = lane; i < nf; i += 32) {
        double val;
        if (i < ns) val = Y[f + i] * Dinv[f + i];
        else { const int c = V.rows[i - ns]; val = (c >= win_lo && c < win_hi) ? Y[c] : yg[c]; }
        w[i] = val;
    }
    __syncwarp();
    // t_j = w_j - sum_{r >= ns} L[r][j] w_r   (lane j owns column j)
    double acc = 0.0;
    for (int r0 = ns; r0 < nf; r0 += 32) {
        const int r = r0 + lane;
        double v[NW];
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns && r < nf) ? Lp[(int64_t)j * ld + r] : 0.0;
#pragma unroll
        for (int j = 0; j < NW; ++j) tile[lane * TL + j] = v[j];
        __syncwarp();
        if (lane < NW) {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) { const double wr = (r0 + rr < nf) ? w[r0 + rr] : 0.0; acc += tile[rr * TL + lane] * wr; }
        }
        __syncwarp();
    }
    const double tj = (lane < ns) ? w[lane] - acc : 0.0;
    // x_j = t_j + sum_{i>j} X[i][j] t_i
#pragma unroll
    for (int j = 0; j < NW; ++j) tile[lane * TL + j] = xr[j];
    __syncwarp();                                  // everyone has read w[0..ns) above
    w[lane] = tj;                                  // t (zero beyond ns)
    __syncwarp();
    double corr = 0.0;
    if (lane < NW) {
#pragma unroll
        for (int i = 0; i < NW; ++i) corr += tile[i * TL + lane] * w[i];
    }
    if (lane < ns) Y[f + lane] = tj + corr;
    __syncwarp();
}

template <int NW, bool MERGED>
__global__ void __launch_bounds__(WPB * 32, NW == 16 ? (MERGED ? 3 : 4) : 2)
k_fwd_warp(DevSym S, const SolveDesc* __restrict__ desc, int count, int maxnf,
           const double* __restrict__ Lst, double* __restrict__ y, double* __restrict__ uvec) {
    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int idx = blockIdx.x * WPB + wid;
    if (idx >= count) return;
    const SolveDesc d = desc[idx];
    if constexpr (MERGED) fwd_warp_body<NW>(view_of(S, d, Lst), y, uvec, smem + (size_t)wid * maxnf, lane);
    else fwd_warp_body_split<NW>(view_of(S, d, Lst), y, uvec, smem + (size_t)wid * maxnf, lane);
}

template <int NW, bool MERGED>
__global__ void __launch_bounds__(WPB * 32, NW == 16 ? (MERGED ? 3 : 4) : 2)
k_bwd_warp(DevSym S, const SolveDesc* __restrict__ desc, int count, int maxnf,
           const double* __restrict__ Lst, const double* __restrict__ Dinv, double* __restrict__ y) {
    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int idx = blockIdx.x * WPB + wid;
    if (idx >= count) return;
    const SolveDesc d = desc[idx];
    double* base = smem + (size_t)wid * (maxnf + 32 + 32 * (NW + 1));    // w (padded to >= 32) then the tile
    if constexpr (MERGED) bwd_warp_body<NW>(view_of(S, d, Lst), Dinv, y, y, 0, 0x7fffffff, base, base + maxnf + 32, lane);
    else bwd_warp_body_split<NW>(view_of(S, d, Lst), Dinv, y, y, 0, 0x7fffffff, base, base + maxnf + 32, lane);
}

// --- whole subtrees of narrow supernodes: one CTA per subtree, no level barrier across the grid.
// The bottom of the assembly tree holds > 99 % of the supernodes; level-scheduled launches make every
// one of them pay a chain of dependent global round trips per sweep with only a wave of warps in
// flight.  Here a CTA owns a complete subtree (contiguous in postorder => contiguous columns, rows,
// panels): its slice of the solution and of the children-contribution vector live in SHARED memory
// for the whole sweep, the warps walk the subtree level by level (block barriers only), and only L is
// streamed from HBM.  Deterministic (same arithmetic as the level-scheduled kernels).
struct SubTrees {
    const int32_t* sn0;        // [nsub] first supernode of the subtree
    const int32_t* sn1;        // [nsub] its root (last supernode)
    const int32_t* order;      // supernodes of all subtrees, per subtree sorted by level
    const int64_t* order_ptr;  // [nsub+1]
    const int32_t* lvl_off;    // [nsub * (nlev+1)] offsets into the subtree's slice of `order`
    int32_t nlev;              // levels a subtree can span
    int32_t maxcols, maxrows;  // window sizes (doubles) the shared memory is dimensioned for
};
constexpr int SUB_MAXNF = 192;

__global__ void __launch_bounds__(256, 2)
k_fwd_subtree(DevSym S, SubTrees T, const double* __restrict__ Lst, double* __restrict__ y,
              double* __restrict__ uvec) {
    extern __shared__ double smem[];
    double* ysm = smem;
    double* usm = ysm + T.maxcols;
    double* wsm = usm + T.maxrows;
    const int t = blockIdx.x;
    const int a = T.sn0[t], b = T.sn1[t];
    const int col_lo = S.sn_first[a], col_hi = S.sn_first[b + 1];
    const int64_t u_lo = S.rows_ptr[a];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < col_hi - col_lo; i += 256) ysm[i] = y[col_lo + i];
    __syncthreads();
    double* Y = ysm - col_lo;
    double* U = usm - u_lo;
    const int32_t* ord = T.order + T.order_ptr[t];
    const int32_t* lo = T.lvl_off + (int64_t)t * (T.nlev + 1);
    double* w = wsm + wid * SUB_MAXNF;
    for (int l = 0; l < T.nlev; ++l) {
        const int e0 = lo[l], e1 = lo[l + 1];
        if (e0 == e1) continue;                                // (uniform) nothing on this level
        for (int k = e0 + wid; k < e1; k += 8) fwd_warp_body<32>(view_of(S, ord[k], Lst), Y, U, w, lane);
        __syncthreads();
    }
    for (int i = tid; i < col_hi - col_lo; i += 256) y[col_lo + i] = ysm[i];
    // only the root's contribution leaves the subtree
    const int64_t r0 = S.rows_ptr[b], r1 = S.rows_ptr[b + 1];
    for (int64_t q = r0 + tid; q < r1; q += 256) uvec[q] = usm[q - u_lo];
}

__global__ void __launch_bounds__(256, 2)
k_bwd_subtree(DevSym S, SubTrees T, const double* __restrict__ Lst, const double* __restrict__ Dinv,
              double* __restrict__ y) {
    extern __shared__ double smem[];
    double* ysm = smem;
    double* wsm = ysm + T.maxcols;
    const int t = blockIdx.x;
    const int a = T.sn0[t], b = T.sn1[t];
    const int col_lo = S.sn_first[a], col_hi = S.sn_first[b + 1];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < col_hi - col_lo; i += 256) ysm[i] = y[col_lo + i];
    __syncthreads();
    double* Y = ysm - col_lo;
    const int32_t* ord = T.order + T.order_ptr[t];
    const int32_t* lo = T.lvl_off + (int64_t)t * (T.nlev + 1);
    double* w = wsm + wid * (SUB_MAXNF + 32 * BT_LD);
    double* tile = w + SUB_MAXNF;
    for (int l = T.nlev - 1; l >= 0; --l) {
        const int e0 = lo[l], e1 = lo[l + 1];
        if (e0 == e1) continue;
        for (int k = e0 + wid; k < e1; k += 8) bwd_warp_body<32>(view_of(S, ord[k], Lst), Dinv, Y, y, col_lo, col_hi, w, tile, lane);
        __syncthreads();
    }
    for (int i = tid; i < col_hi - col_lo; i += 256) y[col_lo + i] = ysm[i];
}

// --- wide supernodes: one CTA (256 threads) per supernode, blocked over SB pivot columns
__global__ void __launch_bounds__(256)
k_fwd_cta(DevSym S, const SolveDesc* __restrict__ desc, const double* __restrict__ Lst,
          double* __restrict__ y, double* __restrict__ uvec) {
    extern __shared__ double w[];
    __shared__ double xs[SB];
    __shared__ double part[4][SB];
    const SolveDesc d = desc[blockIdx.x];        // one round trip instead of batch -> id -> six arrays
    const int f = d.f, ns = d.ns, nr = d.nr, nf = ns + nr, ld = d.ld;
    const int64_t rp = d.rows_ptr;
    const int tid = threadIdx.x;
    {
        const int32_t* cp = S.asm_colptr + d.front_ptr;
        const int64_t base = d.asm_base;
        for (int i = tid; i < nf; i += 256) {
            double acc = i < ns ? y[f + i] : 0.0;
            for (int e = cp[i]; e < cp[i + 1]; ++e) acc += uvec[S.asm_src[base + e]];
            w[i] = acc;
        }
    }
    __syncthreads();
    const double* Lp = Lst + d.panel_off;
    for (int kb = 0; kb < ns; kb += SB) {
        const int sb = min(SB, ns - kb);
        const double* blk = Lp + (int64_t)kb * ld;
        // the first row below the block this thread updates: its loads do not depend on x_kb and are
        // issued BEFORE the block solve (one memory latency per block instead of three)
        const int r1 = kb + sb + tid;
        const bool has1 = r1 < nf;
        double v[SB];
#pragma unroll
        for (int u = 0; u < SB; ++u) v[u] = (has1 && u < sb) ? blk[(int64_t)u * ld + r1] : 0.0;
        // diagonal block: x_i = w_i + sum_{j<i} Linv[i,j] w_j ; 4 threads per row split j
        {
            const int i = tid & 63, qd = tid >> 6;
            double acc = 0.0;
            if (i < sb) acc = diag_row_dot(Lp + (int64_t)kb * ld + kb + i, ld, i, qd, w + kb);
            part[qd][i] = acc;
        }
        __syncthreads();
        if (tid < SB) {
            // zero beyond sb: row_dot64 multiplies the whole 64-entry window (its L loads are zero there), and
            // 0 * uninitialised shared memory is NaN when those bits happen to be a NaN or an infinity
            double x = 0.0;
            if (tid < sb) x = w[kb + tid] + part[0][tid] + part[1][tid] + part[2][tid] + part[3][tid];
            xs[tid] = x;
        }
        __syncthreads();
        if (tid < sb) w[kb + tid] = xs[tid];
        // rows below the block
        if (has1) {
            double a0 = 0.0, a1 = 0.0;
#pragma unroll
            for (int u = 0; u < SB; u += 2) { if (u < sb) a0 += v[u] * xs[u]; if (u + 1 < sb) a1 += v[u + 1] * xs[u + 1]; }
            w[r1] -= a0 + a1;
        }
        for (int r = r1 + 256; r < nf; r += 256) w[r] -= row_dot64(blk + r, ld, sb, xs);
        __syncthreads();
    }
    for (int i = tid; i < nf; i += 256) {
        if (i < ns) y[f + i] = w[i]; else uvec[rp + i - ns] = w[i];
    }
}

__global__ void __launch_bounds__(256)
k_bwd_cta(DevSym S, const int32_t* __restrict__ batch, const double* __restrict__ Lst,
          const double* __restrict__ Dinv, double* __restrict__ y) {
    extern __shared__ double w[];
    __shared__ double ts[SB];
    __shared__ double red8[8][8 * 33];
    // (the packed descriptors of the warp kernels were measured slower here: the per-supernode index arrays
    // are L2-resident, the 64-byte descriptors are not)
    const int s = batch[blockIdx.x];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = tid; i < nf; i += 256) w[i] = i < ns ? y[f + i] * Dinv[f + i] : y[S.rows[rp + i - ns]];
    __syncthreads();
    const double* Lp = Lst + S.panel_off[s];
    const int nblk = (ns + SB - 1) / SB;
    for (int bi = nblk - 1; bi >= 0; --bi) {
        const int kb = bi * SB;
        const int sb = min(SB, ns - kb);
        // t_j = w_j - sum_{r >= kb+sb} L[r, kb+j] w_r : one warp per column, 8 columns at a time
        {   // warp `wid` owns columns 8*wid .. 8*wid+7 of the block
            const int j0 = wid * 8;
            if (j0 < sb) {
                const double o = cols8_dot(Lp + (int64_t)(kb + j0) * ld, ld, min(8, sb - j0), kb + sb, nf, w, lane, red8[wid]);
                if (lane < 8 && j0 + lane < sb) ts[j0 + lane] = w[kb + j0 + lane] - o;
            }
        }
        __syncthreads();
        {   // x_j = t_j + sum_{i>j} Linv[i,j] t_i
            const int j0 = wid * 8;
            if (j0 < sb) {
                double a[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int j = j0 + u;
                    double v0 = 0.0, v1 = 0.0;
                    if (j < sb) {
                        const double* cj = Lp + (int64_t)(kb + j) * ld + kb;
                        const int i0 = lane, i1 = lane + 32;
                        if (i0 > j && i0 < sb) v0 = cj[i0] * ts[i0];
                        if (i1 > j && i1 < sb) v1 = cj[i1] * ts[i1];
                    }
                    a[u] = v0 + v1;
                }
                const double v = warp_sum8_smem(a, red8[wid], lane);
                if (lane < 8 && j0 + lane < sb) w[kb + j0 + lane] = ts[j0 + lane] + v;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < ns; i += 256) y[f + i] = w[i];
}

// --- big supernodes: several CTAs per supernode, one launch per kernel and level whatever ns is.
// The work vector lives in place: top part in y[f..f+ns), bottom part in uvec[rows_ptr[s]..).
//   L11: one CTA per (front, 64-block).  The blocks of a front form a chain (forward: block i needs
//        x_0..x_{i-1}; backward: block j needs x_{j+1}..); a CTA streams its strip of L while the
//        chain advances and waits on a per-block ready flag before each product.  CTAs take their
//        block from an atomic ticket in an order (built by build_plans) where every block of a front
//        comes before the blocks that wait on it, so a CTA only ever waits on blocks that running
//        CTAs hold: no deadlock, whatever the residency or the block scheduler's order.
//   L21: 64-row tiles of every front of the level in one grid (forward: after the chain, with all of
//        x known; backward: before it, into per-tile partial sums reduced in a fixed order).
// Every sum runs in a fixed order, so the solves stay bitwise reproducible.
constexpr int BRT = 64;                     // rows per CTA in the GEMV kernels
constexpr unsigned BIG_SPIN_MAX = 1u << 22; // polls of one ready flag (~1 s) before the solve is declared failed

// One item of the big-solve work lists: {supernode, 64-block (L11) or first row (L21 tile),
// first ready flag of the front, partial-sum offset (backward L11: of the front, L21: of the tile)}.
using BigItem = int4;

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
// x of another CTA of the same launch: a coherent (L2) load, never the non-coherent path
__device__ __forceinline__ double ld_relaxed_gpu(const double* p) {
    double v;
    asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}

// Block-wide: thread 0 polls `flag` (acquire) until it is set.  false (on every thread) when the
// spin bound is exceeded or another CTA has already failed; the error word is then set.
__device__ __forceinline__ bool big_wait(const unsigned* flag, unsigned* err) {
    int ok = 0;
    if (threadIdx.x == 0) {
        for (unsigned it = 0; it < BIG_SPIN_MAX; ++it) {
            if (ld_acquire_gpu(flag)) { ok = 1; break; }
            if (*(volatile unsigned*)err) break;
            __nanosleep(64);
        }
        if (!ok) atomicOr(err, 1u);
    }
    return __syncthreads_or(ok);
}

// Block-wide, after the caller's writes are visible block-wide (a preceding __syncthreads): publish.
__device__ __forceinline__ void big_publish(unsigned* flag) {
    if (threadIdx.x == 0) { __threadfence(); st_release_gpu(flag, 1u); }
}

__device__ __forceinline__ int big_ticket(unsigned* ticket) {
    __shared__ int t;
    if (threadIdx.x == 0) t = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    return t;
}

// w = [y_s ; 0] + sum of children contributions (destination-owner form).
// AL lanes cooperate on one destination row: AL = 1 (thread per row), 32 (warp per row: fronts with
// many children) or 256 (CTA per row: root fronts with ~1e5 children, ~1e3 sources per row).  The
// index loads of 8 sources are issued together, then their 8 value loads (two dependent latencies
// per 8 sources instead of 16); the cross-lane sum is a fixed-order tree => deterministic.
// grid: AL < 256: (ceil(maxnf * AL / 256), cnt) ; AL = 256: (maxnf, cnt).
template <int AL>
__global__ void __launch_bounds__(256)
k_big_asm_fwd(DevSym S, const int32_t* __restrict__ batch, double* __restrict__ y,
              double* __restrict__ uvec) {
    const int s = batch[blockIdx.y];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int i = (AL == 256) ? (int)blockIdx.x : (int)((blockIdx.x * 256 + threadIdx.x) / AL);
    const int sub = threadIdx.x % AL;
    double acc = 0.0;
    if (i < nf) {
        const int32_t* cp = S.asm_colptr + S.front_ptr[s];
        const int64_t base = S.asm_base[s];
        const int e1 = cp[i + 1];
        int e = cp[i] + sub;
        for (; e + 7 * AL < e1; e += 8 * AL) {
            int32_t q[8]; bool on[8]; double v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                q[u] = S.asm_src[base + e + u * AL];
                on[u] = !S.active || S.active[S.asm_child[base + e + u * AL]];
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = on[u] ? uvec[q[u]] : 0.0;
#pragma unroll
            for (int u = 0; u < 8; ++u) acc += v[u];
        }
        for (; e < e1; e += AL)
            if (!S.active || S.active[S.asm_child[base + e]]) acc += uvec[S.asm_src[base + e]];
    }
    if (AL == 256) {
        __shared__ double red[8];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0 && i < nf) {
            double t = 0.0;
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) t += red[w8];
            if (i < ns) y[f + i] += t; else uvec[rp + i - ns] = t;
        }
    } else {
#pragma unroll
        for (int o = AL / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (i < nf && sub == 0) {
            if (i < ns) y[f + i] += acc; else uvec[rp + i - ns] = acc;
        }
    }
}

// forward, L11: one CTA per (front, 64-block i); grid = the level's blocks, order from `ticket`.
// t = w_i - sum_{j<i} L[i,j] x_j (ascending j, each after flag j) ; x_i = inv(L_ii) t -> y ; flag i.
// 256 threads = 64 rows x 4 column quarters; the L loads of block j+1 are in flight while the CTA
// waits for x_j, so a hop of the chain costs a flag hand-off, not an HBM round trip.
__global__ void __launch_bounds__(256)
k_big_tri_fwd(DevSym S, const BigItem* __restrict__ work, unsigned* ticket, unsigned* flags, unsigned* err,
              const double* __restrict__ Lst, double* y) {
    __shared__ double ts[SB];
    __shared__ double part[4][SB];
    const BigItem it = work[big_ticket(ticket)];
    const int s = it.x, bi = it.y;
    flags += it.z;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int ld = S.ld[s];
    const double* Lp = Lst + S.panel_off[s];
    const int kb = bi * SB, sb = min(SB, ns - kb);
    const int tid = threadIdx.x, r = tid & (SB - 1), q = tid >> 6;
    const bool has_r = r < sb;
    // row r of the inverted diagonal block, columns q, q+4, .. < r
    double vd[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; vd[u] = (has_r && j < r) ? Lp[(int64_t)(kb + j) * ld + kb + r] : 0.0; }
    const double wr = (tid < sb) ? y[f + kb + tid] : 0.0;      // own rows: written by earlier launches only
    // row r of the strip left of the block, columns jb*64 + q*16 + u
    const double* rowp = Lp + (int64_t)(q * 16) * ld + kb + r;
    double v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) v[u] = (bi > 0 && has_r) ? rowp[(int64_t)u * ld] : 0.0;
    double a0 = 0.0, a1 = 0.0;
    for (int jb = 0; jb < bi; ++jb) {
        double vn[16];
        const bool more = jb + 1 < bi && has_r;
#pragma unroll
        for (int u = 0; u < 16; ++u) vn[u] = more ? rowp[(int64_t)((jb + 1) * SB + u) * ld] : 0.0;
        if (!big_wait(flags + jb, err)) return;
        const double* xj = y + f + jb * SB + q * 16;          // a full block: only the last one is partial
        double xv[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) xv[u] = ld_relaxed_gpu(xj + u);
#pragma unroll
        for (int u = 0; u < 16; u += 2) { a0 += v[u] * xv[u]; a1 += v[u + 1] * xv[u + 1]; }
#pragma unroll
        for (int u = 0; u < 16; ++u) v[u] = vn[u];
    }
    part[q][r] = a0 + a1;
    __syncthreads();
    if (tid < sb) ts[tid] = wr - ((part[0][tid] + part[1][tid]) + (part[2][tid] + part[3][tid]));
    __syncthreads();
    {   // x_r = t_r + sum_{j<r} Linv[r,j] t_j
        double acc = 0.0;
#pragma unroll
        for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; if (has_r && j < r) acc += vd[u] * ts[j]; }
        part[q][r] = acc;
    }
    __syncthreads();
    if (tid < sb) y[f + kb + tid] = ts[tid] + ((part[0][tid] + part[1][tid]) + (part[2][tid] + part[3][tid]));
    __syncthreads();
    big_publish(flags + bi);
}

// forward, L21: w[r] -= sum_{j<ns} L[r, j] x_j for the rows r >= ns of one 64-row tile; grid = the
// level's tiles.  256 threads = 64 rows x 4 column quarters of 256-column chunks of x.
__global__ void __launch_bounds__(256)
k_big_gemv_fwd(DevSym S, const BigItem* __restrict__ tiles, const double* __restrict__ Lst,
               const double* __restrict__ y, double* __restrict__ uvec) {
    constexpr int XC = 256;
    __shared__ double xs[XC];
    __shared__ double red[4][BRT];
    const BigItem it = tiles[blockIdx.x];
    const int s = it.x, r0 = it.y;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int ld = S.ld[s];
    const int tid = threadIdx.x;
    const int rl = tid & (BRT - 1), q = tid / BRT;          // row in tile, column quarter
    const int r = r0 + rl;
    const double* rowp = Lst + S.panel_off[s] + r;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    for (int c0 = 0; c0 < ns; c0 += XC) {
        const int cw = min(XC, ns - c0);
        __syncthreads();                                     // the previous chunk has been consumed
        for (int j = tid; j < cw; j += 256) xs[j] = y[f + c0 + j];
        __syncthreads();
        if (r < nf) {
            const int j0 = q * (XC / 4), j1 = min(cw, j0 + XC / 4);
            int j = j0;
            for (; j + 16 <= j1; j += 16) {        // (batches of 32 were measured slower: 246 registers)
                double v[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) v[u] = rowp[(int64_t)(c0 + j + u) * ld];
#pragma unroll
                for (int u = 0; u < 16; u += 4) {
                    a0 += v[u] * xs[j + u]; a1 += v[u + 1] * xs[j + u + 1];
                    a2 += v[u + 2] * xs[j + u + 2]; a3 += v[u + 3] * xs[j + u + 3];
                }
            }
            for (; j < j1; ++j) a0 += rowp[(int64_t)(c0 + j) * ld] * xs[j];
        }
    }
    red[q][rl] = (a0 + a1) + (a2 + a3);
    __syncthreads();
    if (q == 0 && r < nf) uvec[rp + r - ns] -= (red[0][rl] + red[1][rl]) + (red[2][rl] + red[3][rl]);
}

// backward, L21: partial[tile][j] = sum_{r in tile} L[r, j] w_r for every pivot column j, with
// w_r = y[rows[r-ns]] (ancestors, solved by earlier launches); grid = the level's tiles
__global__ void __launch_bounds__(256)
k_big_gemvT_bwd(DevSym S, const BigItem* __restrict__ tiles, const double* __restrict__ Lst,
                const double* __restrict__ y, double* __restrict__ partial) {
    __shared__ double ws[BRT];
    __shared__ double red4[8][4 * 33];
    const BigItem it = tiles[blockIdx.x];
    const int s = it.x, r0 = it.y;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int ld = S.ld[s];
    const int nrow = min(BRT, nf - r0);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid < nrow) ws[tid] = y[S.rows[rp + r0 + tid - ns]];
    __syncthreads();
    double* out = partial + it.w;
    const double* Lp = Lst + S.panel_off[s] + r0;
    for (int j = wid * 4; j < ns; j += 32) {          // 8 warps x 4 columns per pass
        double a[4] = {0.0, 0.0, 0.0, 0.0};
        for (int i = lane; i < nrow; i += 32) {
            const double wv = ws[i];
#pragma unroll
            for (int u = 0; u < 4; ++u) if (j + u < ns) a[u] += Lp[(int64_t)(j + u) * ld + i] * wv;
        }
        // cross-lane sums through shared memory (shuffles in this loop would be WARPSYNC.COLLECTIVE'd)
#pragma unroll
        for (int u = 0; u < 4; ++u) red4[wid][u * 33 + lane] = a[u];
        __syncwarp();
        if (lane < 4) {
            double v = 0.0;
#pragma unroll
            for (int l = 0; l < 32; ++l) v += red4[wid][lane * 33 + l];
            if (j + lane < ns) out[j + lane] = v;
        }
        __syncwarp();
    }
}

// sum over the 64 rows r of a[u] held by thread (r = tid & 63, q = tid >> 6) for column q*16+u, in a
// fixed order; thread c < 64 returns the sum of column c.  Ends with the shared tiles free again.
__device__ __forceinline__ double big_colsum(const double (&a)[16], double (*red)[SB + 1], double (*red2)[SB]) {
    const int tid = threadIdx.x, r = tid & (SB - 1), q = tid >> 6;
#pragma unroll
    for (int u = 0; u < 16; ++u) red[q * 16 + u][r] = a[u];
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 16; ++k) s += red[r][q * 16 + k];   // column r, rows q*16..q*16+15
    red2[q][r] = s;
    __syncthreads();
    const double t = tid < SB ? (red2[0][tid] + red2[1][tid]) + (red2[2][tid] + red2[3][tid]) : 0.0;
    __syncthreads();
    return t;
}

// backward, L11: one CTA per (front, 64-column block j); grid = the level's blocks, descending j per
// front by the ticket order.  t = D^-1 y_j - sum_tiles partial (tile order) - sum_{i>j} L[i,j]' x_i
// (descending i, each after flag i) ; x_j = inv(L_jj)' t -> y ; flag j.
// 256 threads = 64 rows (of block i) x 4 column quarters; a thread needs only its own x_i entry.
__global__ void __launch_bounds__(256)
k_big_tri_bwd(DevSym S, const BigItem* __restrict__ work, unsigned* ticket, unsigned* flags, unsigned* err,
              const double* __restrict__ Lst, const double* __restrict__ Dinv,
              const double* __restrict__ partial, double* y) {
    __shared__ double red[SB][SB + 1];
    __shared__ double red2[4][SB];
    __shared__ double ts[SB];
    const BigItem it = work[big_ticket(ticket)];
    const int s = it.x, bj = it.y;
    flags += it.z;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int nf = ns + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    const int ld = S.ld[s];
    const double* Lp = Lst + S.panel_off[s];
    const int nb = (ns + SB - 1) / SB;
    const int kb = bj * SB, sb = min(SB, ns - kb);
    const int tid = threadIdx.x, r = tid & (SB - 1), q = tid >> 6;
    // column q*16+u of this block in block row bi (rows bi*64 + r); for bi = bj the inverted diagonal
    // block (row r > column).  The diagonal block comes last: it is fetched while the last wait runs.
    const double* colp = Lp + (int64_t)(kb + q * 16) * ld + r;
    auto fetch = [&](int bi, double (&v)[16]) {
#pragma unroll
        for (int u = 0; u < 16; ++u)
            v[u] = (bi == bj ? (r < sb && r > q * 16 + u) : bi * SB + r < ns) ? colp[(int64_t)u * ld + bi * SB] : 0.0;
    };
    // ... D^-1 y_j minus the L21 partial sums of the tiles, in tile order
    double t0 = 0.0;
    if (tid < sb) {
        t0 = y[f + kb + tid] * Dinv[f + kb + tid];
        const double* pp = partial + it.w + kb + tid;
        const int ntiles = (nf - ns + BRT - 1) / BRT;
        for (int t = 0; t < ntiles; ++t) t0 -= pp[(int64_t)t * ns];
    }
    // ... and the blocks i > j below it
    double acc[16], v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) acc[u] = 0.0;
    fetch(nb - 1, v);
    for (int bi = nb - 1; bi > bj; --bi) {
        double vn[16];
        fetch(bi - 1, vn);
        if (!big_wait(flags + bi, err)) return;
        const int ri = bi * SB + r;
        const double xr = ri < ns ? ld_relaxed_gpu(y + f + ri) : 0.0;
#pragma unroll
        for (int u = 0; u < 16; ++u) { acc[u] += v[u] * xr; v[u] = vn[u]; }
    }
    const double o = big_colsum(acc, red, red2);
    if (tid < sb) ts[tid] = t0 - o;
    __syncthreads();
    {   // x_c = t_c + sum_{r>c} Linv[r,c] t_r
        const double tr = r < sb ? ts[r] : 0.0;
#pragma unroll
        for (int u = 0; u < 16; ++u) acc[u] = v[u] * tr;      // v: the diagonal block
    }
    const double c = big_colsum(acc, red, red2);
    if (tid < sb) y[f + kb + tid] = ts[tid] + c;
    __syncthreads();
    big_publish(flags + bj);
}

// ------------------------------------------------------------------ G8 residual e = b - K x
// K symmetric, stored as upper CSC (cp, ri, nz) plus the row-wise index of the same entries
// (tp, tc, tpos: entries (j, c > j) of row j, value nz[tpos]).  RL lanes cooperate on one row
// (KKT rows are short: ~5 + 5 entries; dense cone rows just loop), 256/RL rows per CTA.
constexpr int LONG_ROW = 2048;     // rows with more entries are handled by k_residual_long (CTA per row)
template <int RL>
__global__ void __launch_bounds__(256)
k_residual(int64_t N, const int64_t* __restrict__ cp, const int32_t* __restrict__ ri,
           const double* __restrict__ nz, const int64_t* __restrict__ tp,
           const int32_t* __restrict__ tc, const int64_t* __restrict__ tpos,
           const double* __restrict__ x, const double* __restrict__ b, double* __restrict__ e,
           unsigned long long* __restrict__ norm_bits) {
    const int sub = threadIdx.x % RL;
    const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / RL;
    double r = 0.0;
    double acc = 0.0;
    const bool is_long = row < N && (cp[row + 1] - cp[row]) + (tp[row + 1] - tp[row]) > LONG_ROW;
    if (row < N && !is_long) {
        for (int64_t p = cp[row] + sub; p < cp[row + 1]; p += RL) acc += nz[p] * x[ri[p]];
        for (int64_t p = tp[row] + sub; p < tp[row + 1]; p += RL) acc += nz[tpos[p]] * x[tc[p]];
    }
#pragma unroll
    for (int o = RL / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (row < N && !is_long) {
        r = b[row] - acc;
        if (sub == 0) e[row] = r;
    }
    double m = fabs(r);
    if (!(m == m)) m = __longlong_as_double(0x7ff0000000000000LL);   // NaN -> +inf
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ double sm[8];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int q = 0; q < 8; ++q) t = fmax(t, sm[q]);
        atomicMax(norm_bits, (unsigned long long)__double_as_longlong(t));
    }
}

// dense rows (budget / linking constraints): one CTA per row, fixed-order tree reduction
__global__ void __launch_bounds__(256)
k_residual_long(const int32_t* __restrict__ rows, const int64_t* __restrict__ cp,
                const int32_t* __restrict__ ri, const double* __restrict__ nz,
                const int64_t* __restrict__ tp, const int32_t* __restrict__ tc,
                const int64_t* __restrict__ tpos, const double* __restrict__ x,
                const double* __restrict__ b, double* __restrict__ e,
                unsigned long long* __restrict__ norm_bits) {
    __shared__ double sm[8];
    const int64_t row = rows[blockIdx.x];
    double acc = 0.0;
    for (int64_t p = cp[row] + threadIdx.x; p < cp[row + 1]; p += 256) acc += nz[p] * x[ri[p]];
    for (int64_t p = tp[row] + threadIdx.x; p < tp[row + 1]; p += 256) acc += nz[tpos[p]] * x[tc[p]];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int q = 0; q < 8; ++q) t += sm[q];
        const double r = b[row] - t;
        e[row] = r;
        double m = fabs(r);
        if (!(m == m)) m = __longlong_as_double(0x7ff0000000000000LL);
        atomicMax(norm_bits, (unsigned long long)__double_as_longlong(m));
    }
}

__global__ void k_absmax(const double* __restrict__ v, int64_t n, unsigned long long* __restrict__ out) {
    double m = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        double a = fabs(v[i]);
        if (!(a == a)) a = __longlong_as_double(0x7ff0000000000000LL);
        m = fmax(m, a);
    }
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(m));
}

// multi-GPU helpers: zero the panels of a list of supernodes / zero or mask entries of y
__global__ void k_zero_panels(DevSym S, const int32_t* __restrict__ list, double* __restrict__ Lst) {
    const int s = list[blockIdx.y];
    const int64_t ns = S.sn_first[s + 1] - S.sn_first[s];
    const int64_t nf = S.ld[s];
    double* Lp = Lst + S.panel_off[s];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nf * ns;
         i += (int64_t)gridDim.x * blockDim.x) Lp[i] = 0.0;
}
__global__ void k_mask_vec(double* __restrict__ y, const int8_t* __restrict__ keep, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n && !keep[i]) y[i] = 0.0;
}

__global__ void k_axpy1(double* __restrict__ dx, const double* __restrict__ x, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) dx[i] += x[i];
}

__global__ void k_build_rhs(const double* __restrict__ rx, const double* __restrict__ rz,
                            int64_t n, int64_t m, int64_t N, double* __restrict__ b) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < N) b[i] = i < n ? rx[i] : (i < n + m ? rz[i - n] : 0.0);
}

// update_values!/scale_values! on the device copy (inner boundary)
__global__ void k_update_values(double* __restrict__ nz, const int64_t* __restrict__ idx,
                                const double* __restrict__ v, int64_t n, int64_t base) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) nz[idx[i] - base] = v[i];
}
__global__ void k_scale_values(double* __restrict__ nz, const int64_t* __restrict__ idx,
                               double sc, int64_t n, int64_t base) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) nz[idx[i] - base] *= sc;
}

// ------------------------------------------------------------------ G1 cone -> K values
// Diagonal Hs entries (Zero, NN, sparse SOC): nz[map] = -Hs.
//   kind 0: 0 ; 1: w^2 (NN, coneops_nncone.jl:91-101) ; 2: eta^2 (sparse SOC tail) ;
//   3: eta^2 * d (sparse SOC head, coneops_socone.jl:161-166)
__global__ void k_hs_diag(int64_t n, const int8_t* __restrict__ kind, const int32_t* __restrict__ midx,
                          const int32_t* __restrict__ cone, const int64_t* __restrict__ map,
                          const double* __restrict__ w, const double* __restrict__ eta,
                          const double* __restrict__ dd, double* __restrict__ nz) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int k = kind[i];
    double v = 0.0;
    if (k == 1) { const double t = w[midx[i]]; v = t * t; }
    else if (k >= 2) { const double e = eta[cone[i]]; v = e * e; if (k == 3) v *= dd[cone[i]]; }
    nz[map[i]] = -v;
}

// Dense SOC blocks (dim <= 4): packed triu of eta^2 (2ww' - J), Hs[0] = (sqrt2 w0 - 1)(sqrt2 w0 + 1)
// (coneops_socone.jl:168-187).  One thread per cone.
__global__ void k_hs_soc_dense(int32_t ncone, const int32_t* __restrict__ moff,
                               const int32_t* __restrict__ dim, const int32_t* __restrict__ socid,
                               const int64_t* __restrict__ hoff, const int64_t* __restrict__ map,
                               const double* __restrict__ w, const double* __restrict__ eta,
                               double* __restrict__ nz) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncone) return;
    const double* wc = w + moff[i];
    const int d = dim[i];
    const double e = eta[socid[i]];
    const double e2 = e * e;
    const int64_t* mp = map + hoff[i];
    const double s2 = sqrt(2.0);
    // explicit _rn intrinsics: no FMA contraction, so the values are bit-identical to the
    // reference's scalar arithmetic
    const double sw = __dmul_rn(s2, wc[0]);
    nz[mp[0]] = -__dmul_rn(__dmul_rn(__dadd_rn(sw, -1.0), __dadd_rn(sw, 1.0)), e2);
    int h = 1;
    for (int col = 1; col < d; ++col)
        for (int row = 0; row <= col; ++row) {
            double v = __dmul_rn(__dmul_rn(2.0, wc[row]), wc[col]);
            if (row == col) v = __dadd_rn(v, 1.0);
            nz[mp[h++]] = -__dmul_rn(v, e2);
        }
}

// Sparse SOC expansion columns: nz[map_u] = u * (-eta^2), nz[map_v] = v * (-eta^2)
// (directldl_datamaps.jl:61-79: update then scale by -eta^2), D = (-eta^2, +eta^2).
__global__ void k_soc_expansion(int64_t n, const int32_t* __restrict__ src, const int32_t* __restrict__ cone,
                                const int64_t* __restrict__ mapu, const int64_t* __restrict__ mapv,
                                const double* __restrict__ u, const double* __restrict__ v,
                                const double* __restrict__ eta, double* __restrict__ nz) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double e = eta[cone[i]];
    const double me2 = -(e * e);
    nz[mapu[i]] = u[src[i]] * me2;
    nz[mapv[i]] = v[src[i]] * me2;
}
__global__ void k_soc_D(int32_t n, const int32_t* __restrict__ cone, const int64_t* __restrict__ mapD,
                        const double* __restrict__ eta, double* __restrict__ nz) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double e = eta[cone[i]];
    nz[mapD[2 * i]] = -(e * e);
    nz[mapD[2 * i + 1]] = e * e;
}

// ------------------------------------------------------------------ G2 PSD: Hs = (RR') (x)_s (RR')
// k_psd_rrt: A = R R' per cone (n x n, column-major), one CTA per cone.
__global__ void __launch_bounds__(256)
k_psd_rrt(const int32_t* __restrict__ side, const int64_t* __restrict__ roff,
          const double* __restrict__ R, double* __restrict__ A) {
    const int c = blockIdx.x;
    const int n = side[c];
    const double* Rc = R + roff[c];
    double* Ac = A + roff[c];
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
        const int i = e % n, j = e / n;
        double acc = 0.0;
        for (int k = 0; k < n; ++k) acc += Rc[i + k * n] * Rc[j + k * n];
        Ac[e] = acc;
    }
}
// k_psd_skron: grid (column tiles, cones).  Column q=(k,l), row p=(i,j) of triu(A (x)_s A)
// (skron!, coneops_psdtrianglecone.jl:502-540); writes -value through the Hs map.
// A is read through the read-only cache rather than staged in shared memory: it is 8 n^2 bytes
// per cone and stays in L1 / L2, and staging would cap the side at what one block's shared
// memory holds (n = 170 on an H100).
__global__ void __launch_bounds__(256)
k_psd_skron(const int32_t* __restrict__ side, const int64_t* __restrict__ roff,
            const int64_t* __restrict__ hoff, const double* __restrict__ A,
            const int64_t* __restrict__ map, double* __restrict__ nz) {
    const int c = blockIdx.y;
    const int n = side[c];
    const int ne = n * (n + 1) / 2;
    const double* Ac = A + roff[c];
    const int64_t* mp = map + hoff[c];
    const double s2 = sqrt(2.0);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int q = blockIdx.x * 8 + wid; q < ne; q += gridDim.x * 8) {
        // column q -> (k <= l)
        int l = (int)((sqrt(8.0 * q + 1.0) - 1.0) * 0.5);
        while ((l + 1) * (l + 2) / 2 <= q) ++l;
        while (l * (l + 1) / 2 > q) --l;
        const int k = q - l * (l + 1) / 2;
        const bool kl = (k == l);
        const int64_t cbase = (int64_t)q * (q + 1) / 2;
        // rows p = 0..q, p -> (i <= j)
        for (int p = lane; p <= q; p += 32) {
            int j = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
            while ((j + 1) * (j + 2) / 2 <= p) ++j;
            while (j * (j + 1) / 2 > p) --j;
            const int i = p - j * (j + 1) / 2;
            const bool ij = (i == j);
            const double Ajl = __ldg(Ac + j + l * n), Ajk = __ldg(Ac + j + k * n);
            double v;
            if (!ij && !kl) v = __ldg(Ac + i + k * n) * Ajl + __ldg(Ac + i + l * n) * Ajk;
            else if (ij && !kl) v = s2 * Ajl * Ajk;
            else if (!ij && kl) v = s2 * __ldg(Ac + i + l * n) * Ajk;
            else v = Ajl * Ajl;
            nz[mp[cbase + p]] = -v;
        }
    }
}

}  // namespace cb200
