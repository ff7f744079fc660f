// G10: Nesterov-Todd scaling of the symmetric cones on the device (update_scaling!, sm_90a).
//
//   k_scale_nn        NN rows, one thread per row (coneops_nncone.jl:77-89)
//   k_scale_soc<G>    SOC, G threads per cone: G = 32 (a warp, eight cones per CTA) or G = 256 (one CTA per
//                     cone, dim > SOC_CTA_MIN_DIM - 1) (coneops_socone.jl:75-154)
//   k_scale_psd<SM>   PSD, one CTA per cone: Cholesky of S and Z, M = L2'L1, one-sided Jacobi SVD of M, R, Rinv, λ
//                     (coneops_psdtrianglecone.jl:78-143); SM = true works in shared memory, false in a per-cone
//                     global workspace (sides above the shared-memory limit)
//
// Every cross-thread sum is a fixed-shape shared-memory tree behind __syncthreads(), so repeated calls give identical
// bits, and no shuffle or warp-level barrier sits inside a loop whose trip count depends on the data.
#pragma once
#include <cstdint>
#include <cfloat>
#include <cuda_runtime.h>

namespace cb200 {

// ------------------------------------------------------------------ NN
// λ = sqrt(s z), w = sqrt(s / z), correctly rounded (bitwise what numpy computes)
__global__ void k_scale_nn(int64_t n, const int32_t* __restrict__ rows, const double* __restrict__ s,
                           const double* __restrict__ z, double* __restrict__ w, double* __restrict__ lam) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t r = rows[i];
    const double si = s[r], zi = z[r];
    lam[r] = __dsqrt_rn(__dmul_rn(si, zi));
    w[r] = __dsqrt_rn(__ddiv_rn(si, zi));
}

// ------------------------------------------------------------------ SOC
constexpr int SCALE_THREADS = 256;
constexpr int SOC_CTA_MIN_DIM = 1025;       // dim >= this: one CTA per cone

// Sum a and b over each group of G threads (fixed tree order); every thread of the CTA must call.
template <int G>
__device__ __forceinline__ void group_sum2(double (*red)[SCALE_THREADS], double& a, double& b) {
    const int tid = threadIdx.x, t = tid % G;
    red[0][tid] = a; red[1][tid] = b;
    __syncthreads();
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
        if (t < off) { red[0][tid] += red[0][tid + off]; red[1][tid] += red[1][tid + off]; }
        __syncthreads();
    }
    a = red[0][tid - t]; b = red[1][tid - t];
    __syncthreads();
}

// cones[list[q]] for q in [0, ncone): rows moff.. of s / z / w / lam (m-space), srow.. of u / v (SOC space).
// fail[0] is set when a residual of z, s or w is not > 0 (the host's test, NaN included).
template <int G>
__global__ void __launch_bounds__(SCALE_THREADS)
k_scale_soc(int32_t ncone, const int32_t* __restrict__ list, const int64_t* __restrict__ moff,
            const int32_t* __restrict__ dim, const int64_t* __restrict__ srow,
            const double* __restrict__ s, const double* __restrict__ z, double* __restrict__ w,
            double* __restrict__ lam, double* __restrict__ eta, double* __restrict__ dd,
            double* __restrict__ u, double* __restrict__ v, int* __restrict__ fail) {
    __shared__ double red[2][SCALE_THREADS];
    const int t = threadIdx.x % G;
    const int q = blockIdx.x * (SCALE_THREADS / G) + threadIdx.x / G;
    const bool live = q < ncone;
    const int c = live ? list[q] : 0;
    const int d = live ? dim[c] : 0;
    const int64_t mo = live ? moff[c] : 0;
    const double* sc = s + mo;
    const double* zc = z + mo;
    // residuals of z and s: (x0 - |x1|)(x0 + |x1|)
    double az = 0.0, as = 0.0;
    for (int i = 1 + t; i < d; i += G) { const double zi = zc[i], si = sc[i]; az += zi * zi; as += si * si; }
    group_sum2<G>(red, az, as);
    const double z0 = live ? zc[0] : 1.0, s0 = live ? sc[0] : 1.0;
    const double nz = sqrt(az), ns = sqrt(as);
    const double rz = (z0 - nz) * (z0 + nz), rs = (s0 - ns) * (s0 + ns);
    if (live && t == 0 && (!(rz > 0.0) || !(rs > 0.0))) fail[0] = 1;
    const double zscale = sqrt(rz), sscale = sqrt(rs);
    // w = s / sscale + J z / zscale, then its residual
    double aw = 0.0, unused = 0.0;
    for (int i = 1 + t; i < d; i += G) { const double wi = sc[i] / sscale - zc[i] / zscale; aw += wi * wi; }
    group_sum2<G>(red, aw, unused);
    const double w0u = s0 / sscale + z0 / zscale;
    const double nw = sqrt(aw);
    const double rw = (w0u - nw) * (w0u + nw);
    if (live && t == 0 && !(rw > 0.0)) fail[0] = 1;
    const double wscale = sqrt(rw);
    // |w1|^2 of the normalised w
    double a1 = 0.0;
    unused = 0.0;
    for (int i = 1 + t; i < d; i += G) { const double wi = (sc[i] / sscale - zc[i] / zscale) / wscale; a1 += wi * wi; }
    group_sum2<G>(red, a1, unused);
    if (!live) return;
    const double w1sq = a1;
    const double w0 = sqrt(1.0 + w1sq);
    const double gam = 0.5 * wscale;
    const double c1 = (gam + z0 / zscale) / sscale;
    const double c2 = (gam + s0 / sscale) / zscale;
    const double den = 1.0 / (s0 / sscale + z0 / zscale + 2.0 * gam);
    const double sq = sqrt(sscale * zscale);
    // sparse expansion data (computed for every cone, read for dim > 4)
    const double wsq = w0 * w0 + w1sq;
    const double wsqinv = 1.0 / wsq;
    const double dval = wsqinv / 2.0;
    const double u0 = sqrt(wsq - dval);
    const double u1 = 2.0 * w0 / u0;
    const double v1 = sqrt(2.0 * (2.0 + wsqinv) / (2.0 * wsq - wsqinv));
    const int64_t so = srow[c];
    for (int i = t; i < d; i += G) {
        const double si = sc[i], zi = zc[i];
        const double wi = i == 0 ? w0 : (si / sscale - zi / zscale) / wscale;
        w[mo + i] = wi;
        lam[mo + i] = i == 0 ? gam * sq : ((c1 * si + c2 * zi) * den) * sq;
        u[so + i] = i == 0 ? u0 : u1 * wi;
        v[so + i] = i == 0 ? 0.0 : v1 * wi;
    }
    if (t == 0) { eta[c] = sqrt(sscale / zscale); dd[c] = dval; }
}

// ------------------------------------------------------------------ PSD
struct PsdScratch {
    double part[3 * SCALE_THREADS];       // per-thread partial (|ci|^2, |cj|^2, <ci,cj>) of a Jacobi step
    double cs[2 * SCALE_THREADS];         // (cos, sin) per pair of the step chunk; sin == 0: no rotation
    int flag[2];                          // [0] a Cholesky pivot was not > 0, [1] some pair rotated in this sweep
};

// pair k of step `step` of the round-robin (circle) order over N2 (even) players; i < j
__device__ __forceinline__ void rr_pair(int step, int k, int N2, int& i, int& j) {
    int a, b;
    if (k == 0) { a = N2 - 1; b = step; }
    else { a = (step + k) % (N2 - 1); b = (step - k + (N2 - 1)) % (N2 - 1); }
    i = min(a, b); j = max(a, b);
}

// One CTA per cone list[blockIdx.x] (side n, svec rows moff..): R, Rinv (column-major n x n at roff), λ (at loff).
// SM: the four n x n work matrices (S -> L1, Z -> L2, M, V) live in dynamic shared memory, else at
// gws + woff[blockIdx.x].  fail[0]: a Cholesky pivot not > 0, or the Jacobi SVD did not converge in max_sweeps
// sweeps; fail[1]: maximum sweep count over the cones.
template <bool SM>
__global__ void __launch_bounds__(SCALE_THREADS)
k_scale_psd(const int32_t* __restrict__ list, const int32_t* __restrict__ side, const int64_t* __restrict__ moff,
            const int64_t* __restrict__ roff, const int64_t* __restrict__ loff, const int64_t* __restrict__ woff,
            const double* __restrict__ s, const double* __restrict__ z, double* __restrict__ gws,
            double* __restrict__ R, double* __restrict__ Rinv, double* __restrict__ lam, int* __restrict__ fail,
            int max_sweeps) {
    extern __shared__ double dyn[];
    __shared__ PsdScratch sc;
    const int tid = threadIdx.x;
    const int c = list[blockIdx.x];
    const int n = side[c];
    const int nn = n * n;
    double* L1 = SM ? dyn : gws + woff[blockIdx.x];
    double* L2 = L1 + nn;
    double* M = L2 + nn;
    double* V = M + nn;
    const double* sv = s + moff[c];
    const double* zv = z + moff[c];
    // 1. svec -> mat (coneops_psdtrianglecone.jl:469-483): column-major packed upper, off-diagonals / sqrt(2)
    const double rs2 = __ddiv_rn(1.0, __dsqrt_rn(2.0));
    for (int idx = tid; idx < nn; idx += SCALE_THREADS) {
        const int i = idx % n, j = idx / n;
        const int a = min(i, j), b = max(i, j);
        const int e = b * (b + 1) / 2 + a;
        const double f = a == b ? 1.0 : rs2;
        L1[idx] = sv[e] * f;
        L2[idx] = zv[e] * f;
    }
    if (tid == 0) sc.flag[0] = 0;
    __syncthreads();
    // 2. right-looking Cholesky of both (lower triangles), LAPACK potrf's pivot test
    for (int k = 0; k < n; ++k) {
        if (tid < 2) {
            double* A = tid ? L2 : L1;
            const double p = A[k + k * n];
            if (!(p > 0.0)) sc.flag[0] = 1;
            A[k + k * n] = sqrt(p);
        }
        __syncthreads();
        if (sc.flag[0]) break;
        const int r = n - k - 1;
        for (int idx = tid; idx < 2 * r; idx += SCALE_THREADS) {
            double* A = idx < r ? L1 : L2;
            const int i = k + 1 + (idx < r ? idx : idx - r);
            A[i + k * n] /= A[k + k * n];
        }
        __syncthreads();
        for (int idx = tid; idx < 2 * r * r; idx += SCALE_THREADS) {
            const int rem = idx < r * r ? idx : idx - r * r;
            double* A = idx < r * r ? L1 : L2;
            const int i = k + 1 + rem % r, j = k + 1 + rem / r;
            if (i >= j) A[i + j * n] -= A[i + k * n] * A[j + k * n];
        }
        __syncthreads();
    }
    if (sc.flag[0]) { if (tid == 0) fail[0] = 1; return; }
    // 3. M = L2' L1, V = I
    for (int idx = tid; idx < nn; idx += SCALE_THREADS) {
        const int a = idx % n, b = idx / n;
        double acc = 0.0;
        for (int r = max(a, b); r < n; ++r) acc += L2[r + a * n] * L1[r + b * n];
        M[idx] = acc;
        V[idx] = a == b ? 1.0 : 0.0;
    }
    __syncthreads();
    // 4. one-sided (Hestenes) Jacobi on the columns of M, round-robin pair order, rotations applied to V too
    const int N2 = n + (n & 1);
    const int npair = N2 / 2;
    const double tol = (double)n * DBL_EPSILON;
    int sweep = 0;
    bool conv = false;
    while (!conv && sweep < max_sweeps) {
        if (tid == 0) sc.flag[1] = 0;
        for (int step = 0; step < N2 - 1; ++step) {
            for (int p0 = 0; p0 < npair; p0 += SCALE_THREADS) {
                const int pc = min(npair - p0, SCALE_THREADS);
                int T = 1;
                while (T < 32 && 2 * T * pc <= SCALE_THREADS) T *= 2;
                {   // partial sums, T threads per pair
                    const int pl = tid / T, part = tid % T;
                    double a = 0.0, b = 0.0, g = 0.0;
                    if (pl < pc) {
                        int i, j; rr_pair(step, p0 + pl, N2, i, j);
                        if (j < n)
                            for (int r = part; r < n; r += T) {
                                const double ci = M[r + i * n], cj = M[r + j * n];
                                a += ci * ci; b += cj * cj; g += ci * cj;
                            }
                    }
                    sc.part[3 * tid] = a; sc.part[3 * tid + 1] = b; sc.part[3 * tid + 2] = g;
                }
                __syncthreads();
                if (tid < pc) {     // one thread per pair: the rotation
                    double a = 0.0, b = 0.0, g = 0.0;
                    for (int part = 0; part < T; ++part) {
                        const double* pp = sc.part + 3 * (tid * T + part);
                        a += pp[0]; b += pp[1]; g += pp[2];
                    }
                    double cr = 1.0, sr = 0.0;
                    if (fabs(g) > tol * sqrt(a) * sqrt(b)) {
                        const double zeta = (b - a) / (2.0 * g);
                        const double tr = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + hypot(1.0, zeta));
                        cr = 1.0 / sqrt(1.0 + tr * tr);
                        sr = cr * tr;
                        sc.flag[1] = 1;
                    }
                    sc.cs[2 * tid] = cr; sc.cs[2 * tid + 1] = sr;
                }
                __syncthreads();
                for (int e = tid; e < pc * n; e += SCALE_THREADS) {
                    const int pl = e / n, r = e % n;
                    const double sr = sc.cs[2 * pl + 1];
                    if (sr != 0.0) {
                        const double cr = sc.cs[2 * pl];
                        int i, j; rr_pair(step, p0 + pl, N2, i, j);
                        const double mi = M[r + i * n], mj = M[r + j * n];
                        M[r + i * n] = cr * mi - sr * mj; M[r + j * n] = sr * mi + cr * mj;
                        const double vi = V[r + i * n], vj = V[r + j * n];
                        V[r + i * n] = cr * vi - sr * vj; V[r + j * n] = sr * vi + cr * vj;
                    }
                }
                __syncthreads();
            }
        }
        ++sweep;
        conv = sc.flag[1] == 0;
        __syncthreads();            // every thread has read flag[1] before it is reset
    }
    if (tid == 0) {
        if (!conv) fail[0] = 1;
        atomicMax(fail + 1, sweep);
    }
    // 5. σ_k = |M[:, k]| (M V = U Σ), unsorted
    double* lc = lam + loff[c];
    for (int k = tid; k < n; k += SCALE_THREADS) {
        double acc = 0.0;
        for (int r = 0; r < n; ++r) { const double x = M[r + k * n]; acc += x * x; }
        lc[k] = sqrt(acc);
    }
    __syncthreads();
    // 6. R = L1 V Λ^{-1/2}, Rinv = Λ^{-1/2} U' L2' with U = M Σ^{-1}
    double* Rc = R + roff[c];
    double* Ric = Rinv + roff[c];
    for (int idx = tid; idx < nn; idx += SCALE_THREADS) {
        const int a = idx % n, k = idx / n;
        const double sk = lc[k];
        const double isq = 1.0 / sqrt(sk);
        double acc = 0.0;
        for (int r = 0; r <= a; ++r) acc += L1[a + r * n] * V[r + k * n];
        Rc[idx] = acc * isq;
        // Rinv[k, a] = isq_k / σ_k * sum_r M[r, k] L2[a, r]
        double acc2 = 0.0;
        for (int r = 0; r <= a; ++r) acc2 += M[r + k * n] * L2[a + r * n];
        Ric[k + a * n] = (acc2 / sk) * isq;
    }
}

}  // namespace cb200
