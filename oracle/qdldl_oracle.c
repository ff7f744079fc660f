/* TEST INFRASTRUCTURE ONLY — CPU oracle, never imported by the product path.
 *
 * Restatement of the LDL' engine the reference calls for its KKT path: QDLDL.jl (pure Julia,
 * compat "0.4.1" at Clarabel.jl/Project.toml:38 — NOT vendored under the Clarabel.jl repository, so
 * "parity unpinned" at this boundary; see DESIGN.md).  The algorithm restated is the published
 * QDLDL one (Stellato et al., OSQP / QDLDL: elimination tree + up-looking sparse LDL' for
 * quasidefinite matrices, after Davis' LDL) with the additions QDLDL.jl makes and the reference
 * relies on at its call sites:
 *   - directldl_qdldl.jl:18-25  qdldl(KKT; Dsigns, regularize_eps, regularize_delta, logical,
 *                               amd_dense_scale)  -> symbolic analysis on triu(P*K*P')
 *   - directldl_qdldl.jl:54     update_values!(F, index, values)   (through the AtoPAPt map)
 *   - directldl_qdldl.jl:66     scale_values!(F, index, scale)
 *   - directldl_qdldl.jl:77-79  refactor!(F); success = all(isfinite, Dinv)
 *   - directldl_qdldl.jl:94     solve!(F, x): x[perm] -> L \ . -> D^-1 -> L' \ . -> ipermute
 *   - dynamic regularisation: after pivot k is formed, if D[k]*Dsigns[k] < eps then
 *     D[k] = delta*Dsigns[k]  (settings.jl:122-124: eps 1e-13, delta 2e-7)
 * The fill-reducing permutation is passed in (QDLDL.jl accepts `perm=`); the harness obtains it
 * from the AMD-class ordering in clarabel.jl_b200/csrc/ordering.cpp (compiled into this
 * library by oracle/Makefile) because SuiteSparse AMD is not available here.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

typedef int64_t I;

typedef struct {
    I n;
    I *perm, *iperm;        /* perm[k] = original index of pivot k */
    I *Ap, *Ai; double *Ax; /* triu(P A P') */
    I *AtoPAPt;             /* original nz index -> permuted nz index */
    I nnzA;
    I *Dsigns;              /* permuted */
    double eps, delta;
    int regularize;
    I *etree, *Lnz, *Lp, *Li; double *Lx;
    double *D, *Dinv;
    I *iwork; unsigned char *bwork; double *fwork;
    I nnzL;
    I regularize_count;
    double sum_lnz_sq;      /* sum_j (Lnz_j + 1)^2 : factor flops in the CHOLMOD convention */
} qdldl_t;

static I etree_build(I n, const I *Ap, const I *Ai, I *work, I *Lnz, I *etree) {
    /* QDLDL_etree: elimination tree + column counts of L for upper-triangular A */
    I i, j, p, sum = 0;
    for (i = 0; i < n; i++) { work[i] = 0; Lnz[i] = 0; etree[i] = -1; }
    for (j = 0; j < n; j++) {
        work[j] = j;
        for (p = Ap[j]; p < Ap[j + 1]; p++) {
            i = Ai[p];
            if (i > j) return -1;
            while (work[i] != j) {
                if (etree[i] == -1) etree[i] = j;
                Lnz[i]++;
                work[i] = j;
                i = etree[i];
            }
        }
    }
    for (i = 0; i < n; i++) sum += Lnz[i];
    return sum;
}

qdldl_t *qdldl_oracle_new(I n, const I *Ap, const I *Ai, const double *Ax, const I *perm,
                          const I *Dsigns, double eps, double delta, int regularize) {
    qdldl_t *F = (qdldl_t *)calloc(1, sizeof(qdldl_t));
    I i, j, p, nnz = Ap[n];
    F->n = n; F->nnzA = nnz; F->eps = eps; F->delta = delta; F->regularize = regularize;
    F->perm = (I *)malloc(sizeof(I) * (n + 1)); F->iperm = (I *)malloc(sizeof(I) * (n + 1));
    for (i = 0; i < n; i++) F->perm[i] = perm ? perm[i] : i;
    for (i = 0; i < n; i++) F->iperm[F->perm[i]] = i;
    /* permute_symmetric: triu(P A P') with the nz map */
    F->Ap = (I *)calloc(n + 1, sizeof(I));
    F->Ai = (I *)malloc(sizeof(I) * (nnz + 1));
    F->Ax = (double *)malloc(sizeof(double) * (nnz + 1));
    F->AtoPAPt = (I *)malloc(sizeof(I) * (nnz + 1));
    I *cnt = (I *)calloc(n + 1, sizeof(I));
    for (j = 0; j < n; j++)
        for (p = Ap[j]; p < Ap[j + 1]; p++) {
            I pi = F->iperm[Ai[p]], pj = F->iperm[j];
            cnt[pi > pj ? pi : pj]++;
        }
    for (j = 0; j < n; j++) F->Ap[j + 1] = F->Ap[j] + cnt[j];
    for (j = 0; j < n; j++) cnt[j] = F->Ap[j];
    for (j = 0; j < n; j++)
        for (p = Ap[j]; p < Ap[j + 1]; p++) {
            I pi = F->iperm[Ai[p]], pj = F->iperm[j];
            I c = pi > pj ? pi : pj, r = pi > pj ? pj : pi;
            I q = cnt[c]++;
            F->Ai[q] = r; F->Ax[q] = Ax[p]; F->AtoPAPt[p] = q;
        }
    free(cnt);
    F->Dsigns = (I *)malloc(sizeof(I) * (n + 1));
    for (i = 0; i < n; i++) F->Dsigns[i] = Dsigns ? Dsigns[F->perm[i]] : 1;
    F->etree = (I *)malloc(sizeof(I) * (n + 1)); F->Lnz = (I *)malloc(sizeof(I) * (n + 1));
    F->iwork = (I *)malloc(sizeof(I) * (3 * n + 1));
    F->bwork = (unsigned char *)malloc(n + 1);
    F->fwork = (double *)malloc(sizeof(double) * (n + 1));
    F->nnzL = etree_build(n, F->Ap, F->Ai, F->iwork, F->Lnz, F->etree);
    if (F->nnzL < 0) { F->nnzL = 0; }
    F->Lp = (I *)malloc(sizeof(I) * (n + 1));
    F->Li = (I *)malloc(sizeof(I) * (F->nnzL + 1));
    F->Lx = (double *)malloc(sizeof(double) * (F->nnzL + 1));
    F->D = (double *)calloc(n + 1, sizeof(double)); F->Dinv = (double *)calloc(n + 1, sizeof(double));
    F->sum_lnz_sq = 0;
    for (i = 0; i < n; i++) F->sum_lnz_sq += (double)(F->Lnz[i] + 1) * (double)(F->Lnz[i] + 1);
    return F;
}

void qdldl_oracle_free(qdldl_t *F) {
    if (!F) return;
    free(F->perm); free(F->iperm); free(F->Ap); free(F->Ai); free(F->Ax); free(F->AtoPAPt);
    free(F->Dsigns); free(F->etree); free(F->Lnz); free(F->Lp); free(F->Li); free(F->Lx);
    free(F->D); free(F->Dinv); free(F->iwork); free(F->bwork); free(F->fwork); free(F);
}

void qdldl_oracle_update_values(qdldl_t *F, const I *idx, const double *vals, I len) {
    for (I k = 0; k < len; k++) F->Ax[F->AtoPAPt[idx[k]]] = vals[k];
}

void qdldl_oracle_scale_values(qdldl_t *F, const I *idx, I len, double scale) {
    for (I k = 0; k < len; k++) F->Ax[F->AtoPAPt[idx[k]]] *= scale;
}

static void pivot_regularize(qdldl_t *F, I k) {
    if (F->regularize && F->D[k] * (double)F->Dsigns[k] < F->eps) {
        F->D[k] = F->delta * (double)F->Dsigns[k];
        F->regularize_count++;
    }
}

/* up-looking numeric factorisation (QDLDL_factor); returns 1 if all Dinv finite else 0 */
int qdldl_oracle_refactor(qdldl_t *F) {
    const I n = F->n;
    const I *Ap = F->Ap, *Ai = F->Ai; const double *Ax = F->Ax;
    I *Lp = F->Lp, *Li = F->Li; double *Lx = F->Lx, *D = F->D, *Dinv = F->Dinv;
    const I *etree = F->etree, *Lnz = F->Lnz;
    I *yIdx = F->iwork, *elimBuffer = F->iwork + n, *LNext = F->iwork + 2 * n;
    unsigned char *yMark = F->bwork; double *yVals = F->fwork;
    I i, j, k, nnzY, nnzE, bidx, cidx, nextIdx, tmpIdx;
    F->regularize_count = 0;
    if (n == 0) return 1;
    Lp[0] = 0;
    for (i = 0; i < n; i++) {
        Lp[i + 1] = Lp[i] + Lnz[i];
        yMark[i] = 0; yVals[i] = 0.0; D[i] = 0.0; LNext[i] = Lp[i];
    }
    /* first pivot: column 0 of triu has only its diagonal (or is empty) */
    for (i = Ap[0]; i < Ap[1]; i++) if (Ai[i] == 0) D[0] = Ax[i];
    pivot_regularize(F, 0);
    Dinv[0] = 1.0 / D[0];
    for (k = 1; k < n; k++) {
        nnzY = 0;
        for (i = Ap[k]; i < Ap[k + 1]; i++) {
            bidx = Ai[i];
            if (bidx == k) { D[k] = Ax[i]; continue; }
            yVals[bidx] = Ax[i];
            nextIdx = bidx;
            if (!yMark[nextIdx]) {
                yMark[nextIdx] = 1;
                elimBuffer[0] = nextIdx; nnzE = 1;
                nextIdx = etree[bidx];
                while (nextIdx != -1 && nextIdx < k) {
                    if (yMark[nextIdx]) break;
                    yMark[nextIdx] = 1;
                    elimBuffer[nnzE++] = nextIdx;
                    nextIdx = etree[nextIdx];
                }
                while (nnzE) yIdx[nnzY++] = elimBuffer[--nnzE];
            }
        }
        for (i = nnzY - 1; i >= 0; i--) {
            cidx = yIdx[i];
            tmpIdx = LNext[cidx];
            double yc = yVals[cidx];
            for (j = Lp[cidx]; j < tmpIdx; j++) yVals[Li[j]] -= Lx[j] * yc;
            Li[tmpIdx] = k;
            Lx[tmpIdx] = yc * Dinv[cidx];
            D[k] -= yc * Lx[tmpIdx];
            LNext[cidx]++;
            yVals[cidx] = 0.0; yMark[cidx] = 0;
        }
        pivot_regularize(F, k);
        Dinv[k] = 1.0 / D[k];
    }
    for (i = 0; i < n; i++) if (!isfinite(Dinv[i])) return 0;
    return 1;
}

/* x <- K^-1 x using the permuted factors (QDLDL.jl solve!) */
void qdldl_oracle_solve(qdldl_t *F, double *x) {
    const I n = F->n; double *t = F->fwork;
    const I *Lp = F->Lp, *Li = F->Li; const double *Lx = F->Lx;
    I i, j;
    for (i = 0; i < n; i++) t[i] = x[F->perm[i]];
    for (i = 0; i < n; i++) {
        double v = t[i];
        for (j = Lp[i]; j < Lp[i + 1]; j++) t[Li[j]] -= Lx[j] * v;
    }
    for (i = 0; i < n; i++) t[i] *= F->Dinv[i];
    for (i = n - 1; i >= 0; i--) {
        double v = t[i];
        for (j = Lp[i]; j < Lp[i + 1]; j++) v -= Lx[j] * t[Li[j]];
        t[i] = v;
    }
    for (i = 0; i < n; i++) x[F->perm[i]] = t[i];
    for (i = 0; i < n; i++) t[i] = 0.0;      /* fwork doubles as yVals in refactor */
}

I qdldl_oracle_nnzL(const qdldl_t *F) { return F->nnzL; }
I qdldl_oracle_nnzA(const qdldl_t *F) { return F->nnzA; }
I qdldl_oracle_regularize_count(const qdldl_t *F) { return F->regularize_count; }
double qdldl_oracle_sum_lnz_sq(const qdldl_t *F) { return F->sum_lnz_sq; }
const double *qdldl_oracle_D(const qdldl_t *F) { return F->D; }
const double *qdldl_oracle_Dinv(const qdldl_t *F) { return F->Dinv; }
const I *qdldl_oracle_Lp(const qdldl_t *F) { return F->Lp; }
const I *qdldl_oracle_Li(const qdldl_t *F) { return F->Li; }
const double *qdldl_oracle_Lx(const qdldl_t *F) { return F->Lx; }
const I *qdldl_oracle_perm(const qdldl_t *F) { return F->perm; }
