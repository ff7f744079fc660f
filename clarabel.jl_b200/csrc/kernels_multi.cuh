// Multi-right-hand-side forms of the G7 solve kernels and the G8 residual (sm_90a).
//
// A sweep carries R (2 or 4) independent columns.  The work vectors are interleaved: entry i of column r is
// y[i * R + r] (likewise uvec, the per-tile partial sums of k_big_gemvT_bwd and the refinement vectors), so
// a front row or an asm_src gather reads R consecutive doubles, and every L entry is loaded once and used R
// times from registers.  For every column the arithmetic is that of the single-column kernel in
// kernels.cuh - the same operations in the same order, written with the same expression shapes so that the
// compiler contracts the same products - which makes column r bitwise equal to a single-column solve.
// R = 1 is not instantiated here: the single-column kernels are that case.
#pragma once
#include "kernels.cuh"

namespace cb200 {

// y[i*R + r] = src[perm[i]*rs + r*cs] for r < k, 0 for the padding columns k <= r < R
__global__ void k_pack_perm_multi(const double* __restrict__ src, int64_t rs, int64_t cs, int k, int R,
                                  const int32_t* __restrict__ perm, int64_t n, double* __restrict__ y) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * R) return;
    const int64_t i = t / R; const int r = (int)(t - i * R);
    y[t] = r < k ? src[(int64_t)perm[i] * rs + r * cs] : 0.0;
}
__global__ void k_unpack_perm_multi(const double* __restrict__ y, int k, int R, const int32_t* __restrict__ perm,
                                    int64_t n, double* __restrict__ dst, int64_t rs, int64_t cs) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * R) return;
    const int64_t i = t / R; const int r = (int)(t - i * R);
    if (r < k) dst[(int64_t)perm[i] * rs + r * cs] = y[t];
}
// interleaved (R) -> column-major (ld): the accepted refinement iterates -> the caller's layout
__global__ void k_deinterleave(const double* __restrict__ src, int k, int R, int64_t n, double* __restrict__ dst, int64_t ld) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * R) return;
    const int64_t i = t / R; const int r = (int)(t - i * R);
    if (r < k) dst[i + r * ld] = src[t];
}
// b = [rx; rz; 0] per column, interleaved; rx / rz column-major (n x k, m x k)
__global__ void k_build_rhs_multi(const double* __restrict__ rx, const double* __restrict__ rz, int64_t n, int64_t m,
                                  int64_t N, int k, int R, double* __restrict__ b) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= N * R) return;
    const int64_t i = t / R; const int r = (int)(t - i * R);
    b[t] = r >= k ? 0.0 : (i < n ? rx[i + r * n] : (i < n + m ? rz[i - n + r * m] : 0.0));
}
// dx += x (every column: a stopped column's slot is computed but never read back)
__global__ void k_axpy_multi(double* __restrict__ dx, const double* __restrict__ x, int64_t len) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < len) dx[i] += x[i];
}
// dst[:, r] = src[:, r] for the columns r whose bit is set in `mask` (the per-column form of the single
// path's pointer swap)
__global__ void k_select_cols(double* __restrict__ dst, const double* __restrict__ src, int64_t n, int R, unsigned mask) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * R) return;
    if ((mask >> (int)(t % R)) & 1u) dst[t] = src[t];
}
// out[r] = max_i |v[i*R + r]| (NaN -> +inf), as bits
template <int R>
__global__ void k_absmax_multi(const double* __restrict__ v, int64_t n, unsigned long long* __restrict__ out) {
    double m[R];
#pragma unroll
    for (int r = 0; r < R; ++r) m[r] = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            double a = fabs(v[i * R + r]);
            if (!(a == a)) a = __longlong_as_double(0x7ff0000000000000LL);
            m[r] = fmax(m[r], a);
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        for (int o = 16; o > 0; o >>= 1) m[r] = fmax(m[r], __shfl_xor_sync(0xffffffffu, m[r], o));
        if ((threadIdx.x & 31) == 0) atomicMax(out + r, (unsigned long long)__double_as_longlong(m[r]));
    }
}

// ---- leaves (k_fwd_leaf / k_bwd_leaf)
template <int R>
__global__ void __launch_bounds__(128)
k_fwd_leaf_multi(DevSym S, const int32_t* __restrict__ batch, int count, const double* __restrict__ Lst,
                 double* __restrict__ y, double* __restrict__ uvec) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int s = batch[idx];
    const int f = S.sn_first[s];
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const double* Lp = Lst + S.panel_off[s];
    double x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) x[r] = y[(int64_t)f * R + r];
    if (S.child_ptr[s + 1] == S.child_ptr[s]) {
        for (int i = 0; i < nr; ++i) {
            const double l = Lp[1 + i];
#pragma unroll
            for (int r = 0; r < R; ++r) uvec[(rp + i) * R + r] = -l * x[r];
        }
        return;
    }
    const int32_t* cp = S.asm_colptr + S.front_ptr[s];
    const int64_t base = S.asm_base[s];
    for (int e = cp[0]; e < cp[1]; ++e) {
        const int64_t q = (int64_t)S.asm_src[base + e] * R;
#pragma unroll
        for (int r = 0; r < R; ++r) x[r] += uvec[q + r];
    }
#pragma unroll
    for (int r = 0; r < R; ++r) y[(int64_t)f * R + r] = x[r];
    for (int i = 0; i < nr; ++i) {
        double acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0.0;
        for (int e = cp[1 + i]; e < cp[2 + i]; ++e) {
            const int64_t q = (int64_t)S.asm_src[base + e] * R;
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] += uvec[q + r];
        }
        const double l = Lp[1 + i];
#pragma unroll
        for (int r = 0; r < R; ++r) uvec[(rp + i) * R + r] = acc[r] - l * x[r];
    }
}
template <int R>
__global__ void __launch_bounds__(128)
k_bwd_leaf_multi(DevSym S, const int32_t* __restrict__ batch, int count, const double* __restrict__ Lst,
                 const double* __restrict__ Dinv, double* __restrict__ y) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int s = batch[idx];
    const int f = S.sn_first[s];
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const double* Lp = Lst + S.panel_off[s];
    const double dv = Dinv[f];
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = y[(int64_t)f * R + r] * dv;
    for (int i = 0; i < nr; ++i) {
        const double l = Lp[1 + i];
        const int64_t c = (int64_t)S.rows[rp + i] * R;
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] -= l * y[c + r];
    }
#pragma unroll
    for (int r = 0; r < R; ++r) y[(int64_t)f * R + r] = acc[r];
}

// ---- narrow supernodes, one warp each (fwd_warp_body / bwd_warp_body).  The split-load bodies of the
// single-column path (CB200_MERGED_ROWS=0) compute the same sums - their extra terms are products of exact
// zeros - so this one merged-load form serves both settings.
template <int NW, int R>
__device__ __forceinline__ void fwd_warp_body_multi(const SnView& V, double* Y, double* U, double* w, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    double v[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) v[j] = (j < lane && j < ns && lane < nf) ? Lp[(int64_t)j * ld + lane] : 0.0;
    if (V.has_children) {
        for (int i = lane; i < nf; i += 32) {
            double acc[R];
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = i < ns ? Y[(int64_t)(f + i) * R + r] : 0.0;
            for (int e = V.cp[i]; e < V.cp[i + 1]; ++e) {
                const int64_t q = (int64_t)V.asrc[e] * R;
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += U[q + r];
            }
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = acc[r];
        }
    } else {
        for (int i = lane; i < nf; i += 32) {
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = i < ns ? Y[(int64_t)(f + i) * R + r] : 0.0;
        }
    }
    __syncwarp();
    double xi[R];
#pragma unroll
    for (int r = 0; r < R; ++r) xi[r] = 0.0;
    if (lane < ns) {
#pragma unroll
        for (int r = 0; r < R; ++r) xi[r] = w[lane * R + r];
#pragma unroll
        for (int j = 0; j < NW; ++j)
            if (j < ns) {
#pragma unroll
                for (int r = 0; r < R; ++r) xi[r] += v[j] * w[j * R + r];
            }
    }
    __syncwarp();
    if (lane < ns) {
#pragma unroll
        for (int r = 0; r < R; ++r) { w[lane * R + r] = xi[r]; Y[(int64_t)(f + lane) * R + r] = xi[r]; }
    }
    __syncwarp();
    auto row_update = [&](int row) {
        double a0[R], a1[R];
#pragma unroll
        for (int r = 0; r < R; ++r) { a0[r] = 0.0; a1[r] = 0.0; }
#pragma unroll
        for (int j = 0; j < NW; j += 2) {
            if (j < ns) {
#pragma unroll
                for (int r = 0; r < R; ++r) a0[r] += v[j] * w[j * R + r];
            }
            if (j + 1 < ns) {
#pragma unroll
                for (int r = 0; r < R; ++r) a1[r] += v[j + 1] * w[(j + 1) * R + r];
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) U[(V.rp + row - ns) * R + r] = w[row * R + r] - (a0[r] + a1[r]);
    };
    if (lane >= ns && lane < nf) row_update(lane);
    for (int r = 32 + lane; r < nf; r += 32) {
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns) ? Lp[(int64_t)j * ld + r] : 0.0;
        row_update(r);
    }
}

// w: (maxnf + 32) * R doubles, tile: 32 x (NW + 1)
template <int NW, int R>
__device__ __forceinline__ void bwd_warp_body_multi(const SnView& V, const double* __restrict__ Dinv, double* Y,
                                                    double* w, double* tile, int lane) {
    const int f = V.f, ns = V.ns, nf = V.ns + V.nr, ld = V.ld;
    const double* Lp = V.Lp;
    constexpr int TL = NW + 1;
    double xr[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) xr[j] = (j < lane && j < ns && lane < nf) ? Lp[(int64_t)j * ld + lane] : 0.0;
    for (int i = lane; i < nf; i += 32) {
        if (i < ns) {
            const double dv = Dinv[f + i];
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = Y[(int64_t)(f + i) * R + r] * dv;
        } else {
            const int64_t c = (int64_t)V.rows[i - ns] * R;
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = Y[c + r];
        }
    }
#pragma unroll
    for (int j = 0; j < NW; ++j) tile[lane * TL + j] = xr[j];
    __syncwarp();
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0;
    if (lane < NW) {
#pragma unroll
        for (int rr = 0; rr < 32; ++rr)
            if (rr >= ns && rr < nf) {
                const double t = tile[rr * TL + lane];
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += t * w[rr * R + r];
            }
    }
    for (int r0 = 32; r0 < nf; r0 += 32) {
        const int row = r0 + lane;
        double v[NW];
#pragma unroll
        for (int j = 0; j < NW; ++j) v[j] = (j < ns && row < nf) ? Lp[(int64_t)j * ld + row] : 0.0;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < NW; ++j) tile[lane * TL + j] = v[j];
        __syncwarp();
        if (lane < NW) {
#pragma unroll
            for (int rr = 0; rr < 32; ++rr)
                if (r0 + rr < nf) {
                    const double t = tile[rr * TL + lane];
#pragma unroll
                    for (int r = 0; r < R; ++r) acc[r] += t * w[(r0 + rr) * R + r];
                }
        }
    }
    double tj[R];
#pragma unroll
    for (int r = 0; r < R; ++r) tj[r] = (lane < ns) ? w[lane * R + r] - acc[r] : 0.0;
    __syncwarp();
    if (nf > 32) {
#pragma unroll
        for (int j = 0; j < NW; ++j) tile[lane * TL + j] = xr[j];
    }
#pragma unroll
    for (int r = 0; r < R; ++r) w[lane * R + r] = tj[r];
    __syncwarp();
    double corr[R];
#pragma unroll
    for (int r = 0; r < R; ++r) corr[r] = 0.0;
    if (lane < NW) {
#pragma unroll
        for (int i = 0; i < NW; ++i)
            if (i < ns) {
                const double t = tile[i * TL + lane];
#pragma unroll
                for (int r = 0; r < R; ++r) corr[r] += t * w[i * R + r];
            }
    }
    if (lane < ns) {
#pragma unroll
        for (int r = 0; r < R; ++r) Y[(int64_t)(f + lane) * R + r] = tj[r] + corr[r];
    }
    __syncwarp();
}

template <int NW, int R>
__global__ void __launch_bounds__(WPB * 32, NW == 16 ? 2 : 1)
k_fwd_warp_multi(DevSym S, const SolveDesc* __restrict__ desc, int count, int maxnf,
                 const double* __restrict__ Lst, double* __restrict__ y, double* __restrict__ uvec) {
    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int idx = blockIdx.x * WPB + wid;
    if (idx >= count) return;
    const SolveDesc d = desc[idx];
    fwd_warp_body_multi<NW, R>(view_of(S, d, Lst), y, uvec, smem + (size_t)wid * maxnf * R, lane);
}
template <int NW, int R>
__global__ void __launch_bounds__(WPB * 32, NW == 16 ? 2 : 1)
k_bwd_warp_multi(DevSym S, const SolveDesc* __restrict__ desc, int count, int maxnf,
                 const double* __restrict__ Lst, const double* __restrict__ Dinv, double* __restrict__ y) {
    extern __shared__ double smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int idx = blockIdx.x * WPB + wid;
    if (idx >= count) return;
    const SolveDesc d = desc[idx];
    double* base = smem + (size_t)wid * ((size_t)(maxnf + 32) * R + 32 * (NW + 1));
    bwd_warp_body_multi<NW, R>(view_of(S, d, Lst), Dinv, y, base, base + (size_t)(maxnf + 32) * R, lane);
}
// dynamic shared memory of the warp kernels per CTA (R = 1: the single-column kernels)
inline size_t fwd_warp_smem(int maxnf, int R) { return (size_t)WPB * maxnf * R * sizeof(double); }
inline size_t bwd_warp_smem(int maxnf, int NW, int R) {
    return (size_t)WPB * ((size_t)(maxnf + 32) * R + 32 * (NW + 1)) * sizeof(double);
}

// ---- wide supernodes, one CTA each (k_fwd_cta / k_bwd_cta)
template <int R>
__device__ __forceinline__ void diag_row_dot_multi(const double* __restrict__ row, int64_t ld, int i, int q,
                                                   const double* __restrict__ w, double (&acc)[R]) {
    double v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; v[u] = (j < i) ? row[(int64_t)j * ld] : 0.0; }
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0;
#pragma unroll
    for (int u = 0; u < 16; ++u) {
        const int j = q + 4 * u;
        if (j < i) {
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] += v[u] * w[j * R + r];
        }
    }
}
template <int R>
__device__ __forceinline__ void row_dot64_multi(const double* __restrict__ rowp, int64_t ld, int sb,
                                                const double* __restrict__ x, double (&out)[R]) {
    double a0[R], a1[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { a0[r] = 0.0; a1[r] = 0.0; }
#pragma unroll 1
    for (int jb = 0; jb < 64; jb += 32) {
        if (jb < sb) {
            double v[32];
#pragma unroll
            for (int u = 0; u < 32; ++u) v[u] = (jb + u < sb) ? rowp[(int64_t)(jb + u) * ld] : 0.0;
#pragma unroll
            for (int u = 0; u < 32; u += 2) {
#pragma unroll
                for (int r = 0; r < R; ++r) { a0[r] += v[u] * x[(jb + u) * R + r]; a1[r] += v[u + 1] * x[(jb + u + 1) * R + r]; }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) out[r] = a0[r] + a1[r];
}

template <int R>
__global__ void __launch_bounds__(256)
k_fwd_cta_multi(DevSym S, const SolveDesc* __restrict__ desc, const double* __restrict__ Lst,
                double* __restrict__ y, double* __restrict__ uvec) {
    extern __shared__ double w[];
    __shared__ double xs[SB * R];
    __shared__ double part[4][SB * R];
    const SolveDesc d = desc[blockIdx.x];
    const int f = d.f, ns = d.ns, nr = d.nr, nf = ns + nr, ld = d.ld;
    const int64_t rp = d.rows_ptr;
    const int tid = threadIdx.x;
    {
        const int32_t* cp = S.asm_colptr + d.front_ptr;
        const int64_t base = d.asm_base;
        for (int i = tid; i < nf; i += 256) {
            double acc[R];
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = i < ns ? y[(int64_t)(f + i) * R + r] : 0.0;
            for (int e = cp[i]; e < cp[i + 1]; ++e) {
                const int64_t q = (int64_t)S.asm_src[base + e] * R;
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += uvec[q + r];
            }
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = acc[r];
        }
    }
    __syncthreads();
    const double* Lp = Lst + d.panel_off;
    for (int kb = 0; kb < ns; kb += SB) {
        const int sb = min(SB, ns - kb);
        const double* blk = Lp + (int64_t)kb * ld;
        {
            const int i = tid & 63, qd = tid >> 6;
            double acc[R];
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = 0.0;
            if (i < sb) diag_row_dot_multi<R>(Lp + (int64_t)kb * ld + kb + i, ld, i, qd, w + kb * R, acc);
#pragma unroll
            for (int r = 0; r < R; ++r) part[qd][i * R + r] = acc[r];
        }
        __syncthreads();
        if (tid < SB) {             // zero beyond sb, as in k_fwd_cta: row_dot64 reads the whole 64-entry window
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int k = tid * R + r;
                double x = 0.0;
                if (tid < sb) x = w[(kb + tid) * R + r] + part[0][k] + part[1][k] + part[2][k] + part[3][k];
                xs[k] = x;
            }
        }
        __syncthreads();
        if (tid < sb) {
#pragma unroll
            for (int r = 0; r < R; ++r) w[(kb + tid) * R + r] = xs[tid * R + r];
        }
        // rows below the block.  The single-column kernel prefetches a thread's first row before the block
        // solve and sums only its sb products; with R columns that row's 64 registers would spill.  row_dot64
        // sums the same products in the same order, plus products of a zero L entry and a zero xs entry
        // beyond sb, which leave a sum that starts at +0 unchanged.
        #pragma unroll 1
        for (int row = kb + sb + tid; row < nf; row += 256) {
            double o[R];
            row_dot64_multi<R>(blk + row, ld, sb, xs, o);
#pragma unroll
            for (int r = 0; r < R; ++r) w[row * R + r] -= o[r];
        }
        __syncthreads();
    }
    for (int i = tid; i < nf; i += 256) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (i < ns) y[(int64_t)(f + i) * R + r] = w[i * R + r];
            else uvec[(rp + i - ns) * R + r] = w[i * R + r];
        }
    }
}

// warp_sum8_smem for 8 x R sums: lane t < 8R returns the sum of (column t / R, right-hand side t % R)
template <int R>
__device__ __forceinline__ double warp_sum8_multi(const double (&a)[8][R], double* red, int lane) {
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int r = 0; r < R; ++r) red[(u * R + r) * 33 + lane] = a[u][r];
    __syncwarp();
    double s = 0.0;
    if (lane < 8 * R) {
#pragma unroll
        for (int l = 0; l < 32; ++l) s += red[lane * 33 + l];
    }
    __syncwarp();
    return s;
}
// dynamic shared memory: w (maxnf * R) then 8 warps x 8R x 33 reduction slots
inline size_t bwd_cta_smem(int maxnf, int R) { return ((size_t)maxnf * R + 8 * 8 * R * 33) * sizeof(double); }

template <int R>
__global__ void __launch_bounds__(256)
k_bwd_cta_multi(DevSym S, const int32_t* __restrict__ batch, const double* __restrict__ Lst,
                const double* __restrict__ Dinv, double* __restrict__ y) {
    extern __shared__ double w[];
    __shared__ double ts[SB * R];
    const int s = batch[blockIdx.x];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nr = (int)(S.rows_ptr[s + 1] - rp);
    const int nf = ns + nr;
    const int ld = S.ld[s];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    double* red = w + (size_t)nf * R + (size_t)wid * 8 * R * 33;
    for (int i = tid; i < nf; i += 256) {
        if (i < ns) {
            const double dv = Dinv[f + i];
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = y[(int64_t)(f + i) * R + r] * dv;
        } else {
            const int64_t c = (int64_t)S.rows[rp + i - ns] * R;
#pragma unroll
            for (int r = 0; r < R; ++r) w[i * R + r] = y[c + r];
        }
    }
    __syncthreads();
    const double* Lp = Lst + S.panel_off[s];
    const int nblk = (ns + SB - 1) / SB;
    for (int bi = nblk - 1; bi >= 0; --bi) {
        const int kb = bi * SB;
        const int sb = min(SB, ns - kb);
        {   // t_j = w_j - sum_{r >= kb+sb} L[r, kb+j] w_r   (cols8_dot)
            const int j0 = wid * 8;
            if (j0 < sb) {
                const double* base = Lp + (int64_t)(kb + j0) * ld;
                const int ncol = min(8, sb - j0), r0 = kb + sb, r1 = nf;
                double a[8][R];
#pragma unroll
                for (int u = 0; u < 8; ++u)
#pragma unroll
                    for (int r = 0; r < R; ++r) a[u][r] = 0.0;
                for (int row = r0 + lane; row < r1; row += 64) {
                    double v0[8], v1[8];
                    const bool two = (row + 32) < r1;
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        v0[u] = (u < ncol) ? base[(int64_t)u * ld + row] : 0.0;
                        v1[u] = (u < ncol && two) ? base[(int64_t)u * ld + row + 32] : 0.0;
                    }
                    double w0[R], w1[R];
#pragma unroll
                    for (int r = 0; r < R; ++r) { w0[r] = w[row * R + r]; w1[r] = two ? w[(row + 32) * R + r] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u)
#pragma unroll
                        for (int r = 0; r < R; ++r) a[u][r] += v0[u] * w0[r] + v1[u] * w1[r];
                }
                const double o = warp_sum8_multi<R>(a, red, lane);
                const int u = lane / R, r = lane % R;
                if (lane < 8 * R && j0 + u < sb) ts[(j0 + u) * R + r] = w[(kb + j0 + u) * R + r] - o;
            }
        }
        __syncthreads();
        {   // x_j = t_j + sum_{i>j} Linv[i,j] t_i
            const int j0 = wid * 8;
            if (j0 < sb) {
                double a[8][R];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int j = j0 + u;
                    double c0 = 0.0, c1 = 0.0;
                    const int i0 = lane, i1 = lane + 32;
                    const bool on0 = j < sb && i0 > j && i0 < sb, on1 = j < sb && i1 > j && i1 < sb;
                    if (j < sb) {
                        const double* cj = Lp + (int64_t)(kb + j) * ld + kb;
                        if (on0) c0 = cj[i0];
                        if (on1) c1 = cj[i1];
                    }
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        double v0 = 0.0, v1 = 0.0;
                        if (on0) v0 = c0 * ts[i0 * R + r];
                        if (on1) v1 = c1 * ts[i1 * R + r];
                        a[u][r] = v0 + v1;
                    }
                }
                const double v = warp_sum8_multi<R>(a, red, lane);
                const int u = lane / R, r = lane % R;
                if (lane < 8 * R && j0 + u < sb) w[(kb + j0 + u) * R + r] = ts[(j0 + u) * R + r] + v;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < ns; i += 256) {
#pragma unroll
        for (int r = 0; r < R; ++r) y[(int64_t)(f + i) * R + r] = w[i * R + r];
    }
}

// ---- big supernodes (k_big_asm_fwd, k_big_tri_fwd, k_big_gemv_fwd, k_big_gemvT_bwd, k_big_tri_bwd): same
// work lists, tickets, flags and block order as the single-column kernels
template <int AL, int R>
__global__ void __launch_bounds__(256)
k_big_asm_fwd_multi(DevSym S, const int32_t* __restrict__ batch, double* __restrict__ y,
                    double* __restrict__ uvec) {
    const int s = batch[blockIdx.y];
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int i = (AL == 256) ? (int)blockIdx.x : (int)((blockIdx.x * 256 + threadIdx.x) / AL);
    const int sub = threadIdx.x % AL;
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0;
    if (i < nf) {
        const int32_t* cp = S.asm_colptr + S.front_ptr[s];
        const int64_t base = S.asm_base[s];
        const int e1 = cp[i + 1];
        int e = cp[i] + sub;
        for (; e + 7 * AL < e1; e += 8 * AL) {
            int32_t q[8]; bool on[8]; double v[8][R];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                q[u] = S.asm_src[base + e + u * AL];
                on[u] = !S.active || S.active[S.asm_child[base + e + u * AL]];
            }
#pragma unroll
            for (int u = 0; u < 8; ++u)
#pragma unroll
                for (int r = 0; r < R; ++r) v[u][r] = on[u] ? uvec[(int64_t)q[u] * R + r] : 0.0;
#pragma unroll
            for (int u = 0; u < 8; ++u)
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += v[u][r];
        }
        for (; e < e1; e += AL)
            if (!S.active || S.active[S.asm_child[base + e]]) {
                const int64_t q = (int64_t)S.asm_src[base + e] * R;
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += uvec[q + r];
            }
    }
    if (AL == 256) {
        __shared__ double red[8][R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][r] = acc[r];
        }
        __syncthreads();
        if (threadIdx.x == 0 && i < nf) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                double t = 0.0;
#pragma unroll
                for (int w8 = 0; w8 < 8; ++w8) t += red[w8][r];
                if (i < ns) y[(int64_t)(f + i) * R + r] += t; else uvec[(rp + i - ns) * R + r] = t;
            }
        }
    } else {
#pragma unroll
        for (int r = 0; r < R; ++r) {
#pragma unroll
            for (int o = AL / 2; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
        }
        if (i < nf && sub == 0) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                if (i < ns) y[(int64_t)(f + i) * R + r] += acc[r]; else uvec[(rp + i - ns) * R + r] = acc[r];
            }
        }
    }
}

// forward, L11 (k_big_tri_fwd).  The published x block is staged in shared memory (one coherent load per
// entry) instead of 16 R registers per thread.
template <int R>
__global__ void __launch_bounds__(256, 1)
k_big_tri_fwd_multi(DevSym S, const BigItem* __restrict__ work, unsigned* ticket, unsigned* flags, unsigned* err,
                    const double* __restrict__ Lst, double* y) {
    __shared__ double ts[SB * R];
    __shared__ double part[4][SB * R];
    __shared__ double xsm[SB * R];
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
    double vd[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) { const int j = q + 4 * u; vd[u] = (has_r && j < r) ? Lp[(int64_t)(kb + j) * ld + kb + r] : 0.0; }
    double wr[R];
#pragma unroll
    for (int c = 0; c < R; ++c) wr[c] = (tid < sb) ? y[(int64_t)(f + kb + tid) * R + c] : 0.0;
    const double* rowp = Lp + (int64_t)(q * 16) * ld + kb + r;
    double v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) v[u] = (bi > 0 && has_r) ? rowp[(int64_t)u * ld] : 0.0;
    double a0[R], a1[R];
#pragma unroll
    for (int c = 0; c < R; ++c) { a0[c] = 0.0; a1[c] = 0.0; }
    for (int jb = 0; jb < bi; ++jb) {
        double vn[16];
        const bool more = jb + 1 < bi && has_r;
#pragma unroll
        for (int u = 0; u < 16; ++u) vn[u] = more ? rowp[(int64_t)((jb + 1) * SB + u) * ld] : 0.0;
        if (!big_wait(flags + jb, err)) return;              // (a barrier: the previous block's xsm is consumed)
        for (int k = tid; k < SB * R; k += 256) xsm[k] = ld_relaxed_gpu(y + (int64_t)(f + jb * SB) * R + k);
        __syncthreads();
        const double* xv = xsm + q * 16 * R;
#pragma unroll
        for (int u = 0; u < 16; u += 2) {
#pragma unroll
            for (int c = 0; c < R; ++c) { a0[c] += v[u] * xv[u * R + c]; a1[c] += v[u + 1] * xv[(u + 1) * R + c]; }
        }
#pragma unroll
        for (int u = 0; u < 16; ++u) v[u] = vn[u];
    }
#pragma unroll
    for (int c = 0; c < R; ++c) part[q][r * R + c] = a0[c] + a1[c];
    __syncthreads();
    if (tid < sb) {
#pragma unroll
        for (int c = 0; c < R; ++c) {
            const int k = tid * R + c;
            ts[k] = wr[c] - ((part[0][k] + part[1][k]) + (part[2][k] + part[3][k]));
        }
    }
    __syncthreads();
    {
        double acc[R];
#pragma unroll
        for (int c = 0; c < R; ++c) acc[c] = 0.0;
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const int j = q + 4 * u;
            if (has_r && j < r) {
#pragma unroll
                for (int c = 0; c < R; ++c) acc[c] += vd[u] * ts[j * R + c];
            }
        }
#pragma unroll
        for (int c = 0; c < R; ++c) part[q][r * R + c] = acc[c];
    }
    __syncthreads();
    if (tid < sb) {
#pragma unroll
        for (int c = 0; c < R; ++c) {
            const int k = tid * R + c;
            y[(int64_t)(f + kb + tid) * R + c] = ts[k] + ((part[0][k] + part[1][k]) + (part[2][k] + part[3][k]));
        }
    }
    __syncthreads();
    big_publish(flags + bi);
}

template <int R>
__global__ void __launch_bounds__(256)
k_big_gemv_fwd_multi(DevSym S, const BigItem* __restrict__ tiles, const double* __restrict__ Lst,
                     const double* __restrict__ y, double* __restrict__ uvec) {
    constexpr int XC = 256;
    __shared__ double xs[XC * R];
    __shared__ double red[4][BRT * R];
    const BigItem it = tiles[blockIdx.x];
    const int s = it.x, r0 = it.y;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int ld = S.ld[s];
    const int tid = threadIdx.x;
    const int rl = tid & (BRT - 1), q = tid / BRT;
    const int row = r0 + rl;
    const double* rowp = Lst + S.panel_off[s] + row;
    double a0[R], a1[R], a2[R], a3[R];
#pragma unroll
    for (int c = 0; c < R; ++c) { a0[c] = 0.0; a1[c] = 0.0; a2[c] = 0.0; a3[c] = 0.0; }
    for (int c0 = 0; c0 < ns; c0 += XC) {
        const int cw = min(XC, ns - c0);
        __syncthreads();
        for (int j = tid; j < cw * R; j += 256) xs[j] = y[(int64_t)(f + c0) * R + j];
        __syncthreads();
        if (row < nf) {
            const int j0 = q * (XC / 4), j1 = min(cw, j0 + XC / 4);
            int j = j0;
            for (; j + 16 <= j1; j += 16) {
                double v[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) v[u] = rowp[(int64_t)(c0 + j + u) * ld];
#pragma unroll
                for (int u = 0; u < 16; u += 4) {
#pragma unroll
                    for (int c = 0; c < R; ++c) {
                        a0[c] += v[u] * xs[(j + u) * R + c]; a1[c] += v[u + 1] * xs[(j + u + 1) * R + c];
                        a2[c] += v[u + 2] * xs[(j + u + 2) * R + c]; a3[c] += v[u + 3] * xs[(j + u + 3) * R + c];
                    }
                }
            }
            for (; j < j1; ++j) {
                const double l = rowp[(int64_t)(c0 + j) * ld];
#pragma unroll
                for (int c = 0; c < R; ++c) a0[c] += l * xs[j * R + c];
            }
        }
    }
#pragma unroll
    for (int c = 0; c < R; ++c) red[q][rl * R + c] = (a0[c] + a1[c]) + (a2[c] + a3[c]);
    __syncthreads();
    if (q == 0 && row < nf) {
#pragma unroll
        for (int c = 0; c < R; ++c) {
            const int k = rl * R + c;
            uvec[(rp + row - ns) * R + c] -= (red[0][k] + red[1][k]) + (red[2][k] + red[3][k]);
        }
    }
}

// partial: the single-column layout times R (entry (tile, j) of column c at (it.w + j) * R + c)
template <int R>
__global__ void __launch_bounds__(256)
k_big_gemvT_bwd_multi(DevSym S, const BigItem* __restrict__ tiles, const double* __restrict__ Lst,
                      const double* __restrict__ y, double* __restrict__ partial) {
    __shared__ double ws[BRT * R];
    __shared__ double red4[8][4 * R * 33];
    const BigItem it = tiles[blockIdx.x];
    const int s = it.x, r0 = it.y;
    const int f = S.sn_first[s];
    const int ns = S.sn_first[s + 1] - f;
    const int64_t rp = S.rows_ptr[s];
    const int nf = ns + (int)(S.rows_ptr[s + 1] - rp);
    const int ld = S.ld[s];
    const int nrow = min(BRT, nf - r0);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid < nrow * R) {
        const int i = tid / R, c = tid % R;
        ws[tid] = y[(int64_t)S.rows[rp + r0 + i - ns] * R + c];
    }
    __syncthreads();
    double* out = partial + (int64_t)it.w * R;
    const double* Lp = Lst + S.panel_off[s] + r0;
    for (int j = wid * 4; j < ns; j += 32) {
        double a[4][R];
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int c = 0; c < R; ++c) a[u][c] = 0.0;
        for (int i = lane; i < nrow; i += 32) {
            double wv[R];
#pragma unroll
            for (int c = 0; c < R; ++c) wv[c] = ws[i * R + c];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (j + u < ns) {
                    const double l = Lp[(int64_t)(j + u) * ld + i];
#pragma unroll
                    for (int c = 0; c < R; ++c) a[u][c] += l * wv[c];
                }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int c = 0; c < R; ++c) red4[wid][(u * R + c) * 33 + lane] = a[u][c];
        __syncwarp();
        if (lane < 4 * R) {
            double v = 0.0;
#pragma unroll
            for (int l = 0; l < 32; ++l) v += red4[wid][lane * 33 + l];
            const int u = lane / R, c = lane % R;
            if (j + u < ns) out[(int64_t)(j + u) * R + c] = v;
        }
        __syncwarp();
    }
}

template <int R>
__global__ void __launch_bounds__(256)
k_big_tri_bwd_multi(DevSym S, const BigItem* __restrict__ work, unsigned* ticket, unsigned* flags, unsigned* err,
                    const double* __restrict__ Lst, const double* __restrict__ Dinv,
                    const double* __restrict__ partial, double* y) {
    __shared__ double red[SB][SB + 1];
    __shared__ double red2[4][SB];
    __shared__ double ts[SB * R];
    __shared__ double xsm[SB * R];
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
    const double* colp = Lp + (int64_t)(kb + q * 16) * ld + r;
    auto fetch = [&](int bi, double (&v)[16]) {
#pragma unroll
        for (int u = 0; u < 16; ++u)
            v[u] = (bi == bj ? (r < sb && r > q * 16 + u) : bi * SB + r < ns) ? colp[(int64_t)u * ld + bi * SB] : 0.0;
    };
    double t0[R];
#pragma unroll
    for (int c = 0; c < R; ++c) t0[c] = 0.0;
    if (tid < sb) {
        const double dv = Dinv[f + kb + tid];
#pragma unroll
        for (int c = 0; c < R; ++c) t0[c] = y[(int64_t)(f + kb + tid) * R + c] * dv;
        const double* pp = partial + ((int64_t)it.w + kb + tid) * R;
        const int ntiles = (nf - ns + BRT - 1) / BRT;
        for (int t = 0; t < ntiles; ++t) {
#pragma unroll
            for (int c = 0; c < R; ++c) t0[c] -= pp[(int64_t)t * ns * R + c];
        }
    }
    double acc[16][R], v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u)
#pragma unroll
        for (int c = 0; c < R; ++c) acc[u][c] = 0.0;
    fetch(nb - 1, v);
    for (int bi = nb - 1; bi > bj; --bi) {
        double vn[16];
        fetch(bi - 1, vn);
        if (!big_wait(flags + bi, err)) return;              // (a barrier: the previous block's xsm is consumed)
        for (int k = tid; k < SB * R; k += 256) {
            const int ri = bi * SB + k / R;
            xsm[k] = ri < ns ? ld_relaxed_gpu(y + (int64_t)(f + bi * SB) * R + k) : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < 16; ++u) {
#pragma unroll
            for (int c = 0; c < R; ++c) acc[u][c] += v[u] * xsm[r * R + c];
            v[u] = vn[u];
        }
    }
    double o[R];
#pragma unroll
    for (int c = 0; c < R; ++c) {
        double a[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) a[u] = acc[u][c];
        o[c] = big_colsum(a, red, red2);
    }
    if (tid < sb) {
#pragma unroll
        for (int c = 0; c < R; ++c) ts[tid * R + c] = t0[c] - o[c];
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < R; ++c) {
        const double tr = r < sb ? ts[r * R + c] : 0.0;
        double a[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) a[u] = v[u] * tr;
        const double cc = big_colsum(a, red, red2);
        if (tid < sb) y[(int64_t)(f + kb + tid) * R + c] = ts[tid * R + c] + cc;
    }
    __syncthreads();
    big_publish(flags + bj);
}

// ---- G8 residual for R columns: K is read once, e[i*R + r] = b[i*R + r] - (K x_r)_i, ||e_r||_inf -> norm_bits[r]
template <int RL, int R>
__global__ void __launch_bounds__(256)
k_residual_multi(int64_t N, const int64_t* __restrict__ cp, const int32_t* __restrict__ ri,
                 const double* __restrict__ nz, const int64_t* __restrict__ tp,
                 const int32_t* __restrict__ tc, const int64_t* __restrict__ tpos,
                 const double* __restrict__ x, const double* __restrict__ b, double* __restrict__ e,
                 unsigned long long* __restrict__ norm_bits) {
    const int sub = threadIdx.x % RL;
    const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / RL;
    double res[R], acc[R];
#pragma unroll
    for (int c = 0; c < R; ++c) { res[c] = 0.0; acc[c] = 0.0; }
    const bool is_long = row < N && (cp[row + 1] - cp[row]) + (tp[row + 1] - tp[row]) > LONG_ROW;
    if (row < N && !is_long) {
        for (int64_t p = cp[row] + sub; p < cp[row + 1]; p += RL) {
            const double l = nz[p]; const int64_t k = (int64_t)ri[p] * R;
#pragma unroll
            for (int c = 0; c < R; ++c) acc[c] += l * x[k + c];
        }
        for (int64_t p = tp[row] + sub; p < tp[row + 1]; p += RL) {
            const double l = nz[tpos[p]]; const int64_t k = (int64_t)tc[p] * R;
#pragma unroll
            for (int c = 0; c < R; ++c) acc[c] += l * x[k + c];
        }
    }
#pragma unroll
    for (int c = 0; c < R; ++c) {
#pragma unroll
        for (int o = RL / 2; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    }
    if (row < N && !is_long) {
#pragma unroll
        for (int c = 0; c < R; ++c) {
            res[c] = b[row * R + c] - acc[c];
            if (sub == 0) e[row * R + c] = res[c];
        }
    }
    __shared__ double sm[8][R];
#pragma unroll
    for (int c = 0; c < R; ++c) {
        double m = fabs(res[c]);
        if (!(m == m)) m = __longlong_as_double(0x7ff0000000000000LL);
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5][c] = m;
    }
    __syncthreads();
    if (threadIdx.x < R) {
        double t = 0.0;
        for (int q = 0; q < 8; ++q) t = fmax(t, sm[q][threadIdx.x]);
        atomicMax(norm_bits + threadIdx.x, (unsigned long long)__double_as_longlong(t));
    }
}

template <int R>
__global__ void __launch_bounds__(256)
k_residual_long_multi(const int32_t* __restrict__ rows, const int64_t* __restrict__ cp,
                      const int32_t* __restrict__ ri, const double* __restrict__ nz,
                      const int64_t* __restrict__ tp, const int32_t* __restrict__ tc,
                      const int64_t* __restrict__ tpos, const double* __restrict__ x,
                      const double* __restrict__ b, double* __restrict__ e,
                      unsigned long long* __restrict__ norm_bits) {
    __shared__ double sm[8][R];
    const int64_t row = rows[blockIdx.x];
    double acc[R];
#pragma unroll
    for (int c = 0; c < R; ++c) acc[c] = 0.0;
    for (int64_t p = cp[row] + threadIdx.x; p < cp[row + 1]; p += 256) {
        const double l = nz[p]; const int64_t k = (int64_t)ri[p] * R;
#pragma unroll
        for (int c = 0; c < R; ++c) acc[c] += l * x[k + c];
    }
    for (int64_t p = tp[row] + threadIdx.x; p < tp[row + 1]; p += 256) {
        const double l = nz[tpos[p]]; const int64_t k = (int64_t)tc[p] * R;
#pragma unroll
        for (int c = 0; c < R; ++c) acc[c] += l * x[k + c];
    }
#pragma unroll
    for (int c = 0; c < R; ++c) {
        for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
        if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5][c] = acc[c];
    }
    __syncthreads();
    if (threadIdx.x < R) {
        const int c = threadIdx.x;
        double t = 0.0;
        for (int q = 0; q < 8; ++q) t += sm[q][c];
        const double res = b[row * R + c] - t;
        e[row * R + c] = res;
        double m = fabs(res);
        if (!(m == m)) m = __longlong_as_double(0x7ff0000000000000LL);
        atomicMax(norm_bits + c, (unsigned long long)__double_as_longlong(m));
    }
}

}  // namespace cb200
