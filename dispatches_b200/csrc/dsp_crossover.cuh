// dsp_crossover.cuh -- crossover post-pass of a solved batch (dsp_lp_crossover, include/dsp_lp.h): from the interior point (x, y)
// an interior-point kernel returned, a basic optimal solution (a vertex) of the same LP, with its basis and basis duals.
//
// For one LP  min c'x + k  s.t.  A x = b, 0 <= x <= u  (A, b, c, u with every per-problem parameter and matrix term), in the CALLER's
// column / row order.  Variables are the n columns and one artificial per row (a unit column, bounds [0, 0]); a basis holds m of them.
//   1. crash: columns strictly inside their bounds, most interior first (min(x_j, u_j - x_j), ties by index), replace the artificial
//      with the largest entry of B^-1 a_j while that entry is at least kPivot |a_j|_inf.  Columns within tol_p of a bound are put on it.
//   2. push: every remaining column inside its bounds, in index order, moves towards the bound its reduced cost favours (the nearer one
//      when |d_j| <= tol_d) with a ratio test over the basic variables; a blocking basic variable leaves the basis (artificials block
//      at once), otherwise the column lands on its bound.
//   3. reinversion, x_B = B^-1 (b - N x_N) and y = B^-T c_B, each with one step of iterative refinement.
//   4. cleanup: bounded primal simplex pivots while a reduced cost has the wrong sign (Dantzig pricing, Harris ratio test, bound flips,
//      Bland's rule after kBlandAfter degenerate pivots in a row), bounded dual simplex pivots while only primal violations remain;
//      then every basic artificial that a column can replace by a dual ratio test (an entry of at least kPivot |rho|_inf |a_j|_inf) is
//      pivoted out, and 3 is repeated.  An artificial that stays basic marks a redundant row.
// Tolerances: tol_p = kFeas sp, sp = max(1, |b|_inf, |u_finite|_inf); tol_d = kFeas sd, sd = |c|_inf (1 if c = 0).
//
// Layout: one CTA per LP, LPs handed out grid-stride.  The dense explicit inverse B^-1 (m x m, row k: basis position k) is updated by a
// rank-one product-form step per pivot and rebuilt by Gauss-Jordan elimination with partial pivoting every kRefactor updates and
// before every step 3.  B^-1 and the LP's vectors sit in one work region, in shared memory or in the handle's workspace.  Every
// output element and every intermediate vector element is summed by one thread in a fixed order, and every choice is an exact
// comparison with ties broken by index: the results do not depend on the number of threads or on where an LP sits in the batch.
//
// Plain C++ over a thread index: tests/emu compiles this file with g++ on the SIMT emulator (one warp as the CTA).
#pragma once

#include <math.h>

#include <algorithm>
#include <utility>

#include "dsp_sens.cuh"

namespace xo {

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define XOD __device__ __forceinline__
#define XOHD __host__ __device__ inline
#else
#define XOD inline
#define XOHD inline
#endif

constexpr int kMaxThreads = 256;
constexpr double kFeas = 1e-9;       // primal / dual feasibility, relative to sp / sd
constexpr double kPivot = 1e-7;      // pivot tolerance, relative to the column
constexpr int kRefactor = 64;        // product-form updates between reinversions
constexpr int kBlandAfter = 50;      // degenerate pivots in a row before Bland's rule
enum { AT_LO = 0, BASIC = 1, AT_UP = 2, INSIDE = 3 };
enum { OPTIMAL = 0, MAX_ITER = 1, NUMERICAL = 2 };

// element offsets of the crossover's own structure blob (what the sensitivity blob lacks): doubles, then int32 from ioff bytes
struct Layout {
    long long b0, bm_val, u0, um_val;                              // doubles (u0: +inf where a column has no bound)
    long long bm_ptr, bm_idx, um_ptr, um_idx, r_ptr, r_pos, r_col; // int32: b by row, u by column, the CSR of A (CSC positions)
    long long ioff, bytes;
};

struct View {
    const double *b0, *bm_val, *u0, *um_val;
    const int *bm_ptr, *bm_idx, *um_ptr, *um_idx, *r_ptr, *r_pos, *r_col;
};

XOD View view_of(const unsigned char *base, const Layout &L) {
    const double *d = (const double *)base;
    const int *i = (const int *)(base + L.ioff);
    View v;
    v.b0 = d + L.b0; v.bm_val = d + L.bm_val; v.u0 = d + L.u0; v.um_val = d + L.um_val;
    v.bm_ptr = i + L.bm_ptr; v.bm_idx = i + L.bm_idx; v.um_ptr = i + L.um_ptr; v.um_idx = i + L.um_idx;
    v.r_ptr = i + L.r_ptr; v.r_pos = i + L.r_pos; v.r_col = i + L.r_col;
    return v;
}

struct Params {
    int m, n, Pc, Pr, nnz;
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    const int *status;
    const double *x, *y;
    int max_pivots;
    double o0;
    double *obj, *x_out, *y_out;
    signed char *col_status, *row_basic;   // each may be null
    int *xstatus, *pivots;                 // pivots may be null
    const unsigned char *blob;             // the sensitivity pass's structure (sens::Layout L)
    sens::Layout L;
    const unsigned char *xblob;            // the crossover's own structure
    Layout X;
    double *ws;                            // work regions in global memory (null: shared memory)
    long long ws_stride;                   // doubles per CTA
};

// doubles of one LP's work region
XOHD long long work_doubles(int m, int n, int nnz) {
    const long long d = (long long)m * m + nnz + 4LL * n + (n + m) + 7LL * m;
    const long long i = 3LL * m + 2LL * n;
    return (d + (i + 1) / 2 + 1) / 2 * 2;
}

struct Work {
    double *B, *a, *c, *u, *d, *alr, *xv, *b, *y, *al, *t1, *t2, *t3, *t4;
    int *head, *stat, *ord, *perm;
};

XOD Work carve(double *w, int m, int n, int nnz) {
    Work W;
    W.B = w; w += (long long)m * m;
    W.a = w; w += nnz;
    W.c = w; w += n; W.u = w; w += n; W.d = w; w += n; W.alr = w; w += n; W.xv = w; w += n + m;
    W.b = w; w += m; W.y = w; w += m; W.al = w; w += m; W.t1 = w; w += m; W.t2 = w; w += m; W.t3 = w; w += m; W.t4 = w; w += m;
    int *i = (int *)w;
    W.head = i; i += m; W.stat = i; i += n + m; W.ord = i; i += n; W.perm = i;
    return W;
}

// scratch for block-wide choices and broadcasts
struct Shared {
    double k1[kMaxThreads], k2[kMaxThreads];
    int id[kMaxThreads];
    double r1, r2;
    int rid;
    int ival[4];
};

#ifndef XO_SYNC
#define XO_SYNC() __syncthreads()
#endif

// the paths of lp_body, for XO_TRACE(ev): a test build counts them (tests/emu/emu_crossover.cpp); the library compiles the hook out
enum {
    TR_PUSH_PIVOT, TR_PUSH_REINVERT, TR_PRIMAL_PIVOT, TR_PRIMAL_DEGENERATE, TR_BOUND_FLIP, TR_DUAL_PIVOT, TR_BLAND,
    TR_CLEANUP_REINVERT, TR_ARTIFICIAL_OUT, TR_REDUNDANT_ROW, TR_ROUND, TR_EVENTS
};
#ifndef XO_TRACE
#define XO_TRACE(ev) ((void)0)
#endif

constexpr int kNone = 0x7fffffff;

XOD bool better(double a1, double a2, int ai, double b1, double b2, int bi) {
    return a1 < b1 || (a1 == b1 && (a2 < b2 || (a2 == b2 && ai < bi)));
}

// the block's smallest (k1, k2, id), lexicographically; every thread passes its own best.  Result in S->r1, r2, rid.
XOD void choose(Shared *S, int tid, int nt, double k1, double k2, int id) {
    S->k1[tid] = k1; S->k2[tid] = k2; S->id[tid] = id;
    XO_SYNC();
    if (tid == 0) {
        int b = 0;
        for (int t = 1; t < nt; ++t)
            if (better(S->k1[t], S->k2[t], S->id[t], S->k1[b], S->k2[b], S->id[b])) b = t;
        S->r1 = S->k1[b]; S->r2 = S->k2[b]; S->rid = S->id[b];
    }
    XO_SYNC();
}

XOD void keep_best(double &b1, double &b2, int &bi, double k1, double k2, int i) {
    if (better(k1, k2, i, b1, b2, bi)) { b1 = k1; b2 = k2; bi = i; }
}

XOD double upper(const Work &W, int n, int v) { return v < n ? W.u[v] : 0.0; }

// al = B^-1 a_v (v >= n: the artificial of row v - n)
XOD void ftran(const Work &W, const sens::View &s, int m, int n, int v, double *al, int tid, int nt) {
    if (v >= n) {
        for (int k = tid; k < m; k += nt) al[k] = W.B[(long long)k * m + (v - n)];
    } else {
        const int e0 = sens::ld<true>(s.At_ptr + v), e1 = sens::ld<true>(s.At_ptr + v + 1);
        for (int k = tid; k < m; k += nt) {
            double r = 0.0;
            for (int e = e0; e < e1; ++e) r = fma(W.B[(long long)k * m + sens::ld<true>(s.At_idx + e)], W.a[e], r);
            al[k] = r;
        }
    }
    XO_SYNC();
}

// the product-form update: column al (= B^-1 a_q) enters at position r
XOD void update(const Work &W, int m, int r, const double *al, int tid, int nt) {
    const double p = al[r];
    for (int k = tid; k < m; k += nt) W.t4[k] = W.B[(long long)r * m + k] / p;
    XO_SYNC();
    const long long mm = (long long)m * m;
    for (long long e = tid; e < mm; e += nt) {
        const int k = (int)(e / m), i = (int)(e % m);
        W.B[e] = k == r ? W.t4[i] : fma(-al[k], W.t4[i], W.B[e]);
    }
    XO_SYNC();
}

// B^-1 from the basis head by Gauss-Jordan elimination in place with partial pivoting; false when singular
XOD bool reinvert(const Work &W, const sens::View &s, Shared *S, int m, int n, int tid, int nt) {
    const long long mm = (long long)m * m;
    for (long long e = tid; e < mm; e += nt) W.B[e] = 0.0;
    XO_SYNC();
    for (int k = tid; k < m; k += nt) {              // column k of B: the basic variable of position k (each thread owns whole columns)
        const int v = W.head[k];
        double cm = 0.0;
        if (v >= n) { W.B[(long long)(v - n) * m + k] = 1.0; cm = 1.0; }
        else
            for (int e = sens::ld<true>(s.At_ptr + v), e1 = sens::ld<true>(s.At_ptr + v + 1); e < e1; ++e) {
                W.B[(long long)sens::ld<true>(s.At_idx + e) * m + k] = W.a[e];
                cm = fmax(cm, fabs(W.a[e]));
            }
        W.t2[k] = cm;
    }
    XO_SYNC();
    for (int k = 0; k < m; ++k) {
        double b1 = INFINITY, b2 = 0.0; int bi = kNone;
        for (int i = k + tid; i < m; i += nt) keep_best(b1, b2, bi, -fabs(W.B[(long long)i * m + k]), 0.0, i);
        choose(S, tid, nt, b1, b2, bi);
        const int pr = S->rid;
        if (!(-S->r1 > 1e-12 * W.t2[k])) return false;
        if (pr != k)
            for (int j = tid; j < m; j += nt) {
                const double t = W.B[(long long)k * m + j];
                W.B[(long long)k * m + j] = W.B[(long long)pr * m + j]; W.B[(long long)pr * m + j] = t;
            }
        if (tid == 0) W.perm[k] = pr;
        XO_SYNC();
        const double piv = W.B[(long long)k * m + k];
        for (int i = tid; i < m; i += nt) W.t1[i] = W.B[(long long)i * m + k];
        XO_SYNC();
        for (int j = tid; j < m; j += nt) W.B[(long long)k * m + j] = j == k ? 1.0 / piv : W.B[(long long)k * m + j] / piv;
        XO_SYNC();
        for (long long e = tid; e < mm; e += nt) {
            const int i = (int)(e / m), j = (int)(e % m);
            if (i == k) continue;
            W.B[e] = fma(-W.t1[i], W.B[(long long)k * m + j], j == k ? 0.0 : W.B[e]);
        }
        XO_SYNC();
    }
    for (int k = m - 1; k >= 0; --k) {               // undo the row interchanges as column interchanges
        const int pr = W.perm[k];
        if (pr != k)
            for (int i = tid; i < m; i += nt) {
                const double t = W.B[(long long)i * m + k];
                W.B[(long long)i * m + k] = W.B[(long long)i * m + pr]; W.B[(long long)i * m + pr] = t;
            }
        XO_SYNC();
    }
    return true;
}

// x_B = B^-1 (b - N x_N), written into xv of the basic variables; with refine, one step of iterative refinement against A
XOD void solve_x(const Work &W, const View &X, int m, int n, bool refine, int tid, int nt) {
    for (int i = tid; i < m; i += nt) {
        double r = W.b[i];
        for (int q = sens::ld<true>(X.r_ptr + i), q1 = sens::ld<true>(X.r_ptr + i + 1); q < q1; ++q) {
            const int j = sens::ld<true>(X.r_col + q);
            if (W.stat[j] != BASIC) r = fma(-W.a[sens::ld<true>(X.r_pos + q)], W.xv[j], r);
        }
        W.t1[i] = r;
    }
    XO_SYNC();
    for (int k = tid; k < m; k += nt) {
        double r = 0.0;
        for (int i = 0; i < m; ++i) r = fma(W.B[(long long)k * m + i], W.t1[i], r);
        W.t2[k] = r;
    }
    XO_SYNC();
    for (int k = tid; k < m; k += nt) W.xv[W.head[k]] = W.t2[k];
    XO_SYNC();
    if (!refine) return;
    for (int i = tid; i < m; i += nt) {
        double r = W.b[i];
        for (int q = sens::ld<true>(X.r_ptr + i), q1 = sens::ld<true>(X.r_ptr + i + 1); q < q1; ++q)
            r = fma(-W.a[sens::ld<true>(X.r_pos + q)], W.xv[sens::ld<true>(X.r_col + q)], r);
        W.t1[i] = r - W.xv[n + i];
    }
    XO_SYNC();
    for (int k = tid; k < m; k += nt) {
        double r = 0.0;
        for (int i = 0; i < m; ++i) r = fma(W.B[(long long)k * m + i], W.t1[i], r);
        W.xv[W.head[k]] = W.t2[k] + r;
    }
    XO_SYNC();
}

// a_v' y (v >= n: y of its row)
XOD double col_dot(const Work &W, const sens::View &s, int n, int v, const double *y) {
    if (v >= n) return y[v - n];
    double r = 0.0;
    for (int e = sens::ld<true>(s.At_ptr + v), e1 = sens::ld<true>(s.At_ptr + v + 1); e < e1; ++e)
        r = fma(W.a[e], y[sens::ld<true>(s.At_idx + e)], r);
    return r;
}

// y = B^-T c_B (optionally refined), then d = c - A'y of every column
XOD void solve_y(const Work &W, const sens::View &s, int m, int n, bool refine, int tid, int nt) {
    for (int k = tid; k < m; k += nt) W.t1[k] = W.head[k] < n ? W.c[W.head[k]] : 0.0;
    XO_SYNC();
    for (int i = tid; i < m; i += nt) {
        double r = 0.0;
        for (int k = 0; k < m; ++k) r = fma(W.t1[k], W.B[(long long)k * m + i], r);
        W.y[i] = r;
    }
    XO_SYNC();
    if (refine) {
        for (int k = tid; k < m; k += nt) W.t2[k] = W.t1[k] - col_dot(W, s, n, W.head[k], W.y);
        XO_SYNC();
        for (int i = tid; i < m; i += nt) {
            double r = 0.0;
            for (int k = 0; k < m; ++k) r = fma(W.t2[k], W.B[(long long)k * m + i], r);
            W.t3[i] = W.y[i] + r;
        }
        XO_SYNC();
        for (int i = tid; i < m; i += nt) W.y[i] = W.t3[i];
        XO_SYNC();
    }
    for (int j = tid; j < n; j += nt) W.d[j] = W.c[j] - col_dot(W, s, n, j, W.y);
    XO_SYNC();
}

// the basis change: q enters at position r (al = B^-1 a_q), the leaving variable goes to value `at` with status st
XOD void pivot(const Work &W, int m, int n, int r, int q, int st, double at, int tid, int nt) {
    const int v = W.head[r];
    XO_SYNC();
    update(W, m, r, W.al, tid, nt);
    if (tid == 0) {
        W.stat[v] = st; W.xv[v] = at;
        W.head[r] = q; W.stat[q] = BASIC;
    }
    XO_SYNC();
}

XOD bool fixed_col(const Work &W, int j) { return W.u[j] <= 0.0; }

// largest primal violation of a basic variable: S->rid its position (kNone: none), S->r1 minus its size
XOD void primal_worst(const Work &W, Shared *S, int m, int n, double tolp, int tid, int nt) {
    double b1 = INFINITY, b2 = 0.0; int bi = kNone;
    for (int k = tid; k < m; k += nt) {
        const int v = W.head[k];
        const double x = W.xv[v], up = upper(W, n, v);
        const double viol = x < -tolp ? -x : x > up + tolp ? x - up : 0.0;
        if (viol > 0.0) keep_best(b1, b2, bi, -viol, 0.0, v);
    }
    choose(S, tid, nt, b1, b2, bi);
}

// the dual infeasibility of a nonbasic column (0 if none)
XOD double dual_inf(const Work &W, int j, double told) {
    if (W.stat[j] == BASIC || fixed_col(W, j)) return 0.0;
    const double dj = W.d[j];
    if (W.stat[j] == AT_LO && dj < -told) return -dj;
    if (W.stat[j] == AT_UP && dj > told) return dj;
    return 0.0;
}

// how far the reduced cost of a nonbasic column is from the wrong sign: max(d_j, 0) at 0, max(-d_j, 0) at u (a reduced cost already
// on the wrong side, within tol_d, has no slack left)
XOD double dual_slack(const Work &W, int j) { return W.stat[j] == AT_LO ? fmax(W.d[j], 0.0) : fmax(-W.d[j], 0.0); }

// dual ratio test on row r of B^-1 (alr: rho' a_j of every nonbasic column): dir > 0 chooses among the columns whose reduced cost
// limits a positive dual step, dir < 0 a negative one; Harris' two passes, the largest |alpha| (Bland: the lowest index) in the
// second.  Returns the entering column (kNone: none) and its ratio in *ratio.
XOD int dual_ratio(const Work &W, Shared *S, int n, int dir, double told, bool bland, double *ratio, int tid, int nt) {
    double b1 = INFINITY, b2 = 0.0; int bi = kNone;
    for (int j = tid; j < n; j += nt) {
        const double a = W.alr[j];
        if (a == 0.0) continue;
        const bool lo = W.stat[j] == AT_LO;
        if (!((lo && a * dir > 0.0) || (!lo && a * dir < 0.0))) continue;
        keep_best(b1, b2, bi, (dual_slack(W, j) + told) / fabs(a), 0.0, j);
    }
    choose(S, tid, nt, b1, b2, bi);
    if (S->rid == kNone) return kNone;
    const double tmax = S->r1;
    b1 = INFINITY; b2 = 0.0; bi = kNone;
    for (int j = tid; j < n; j += nt) {
        const double a = W.alr[j];
        if (a == 0.0) continue;
        const bool lo = W.stat[j] == AT_LO;
        if (!((lo && a * dir > 0.0) || (!lo && a * dir < 0.0))) continue;
        const double rt = dual_slack(W, j) / fabs(a);
        if (rt <= tmax) keep_best(b1, b2, bi, bland ? 0.0 : -fabs(a), 0.0, j);
    }
    choose(S, tid, nt, b1, b2, bi);
    const int q = S->rid;
    if (q != kNone) *ratio = dual_slack(W, q) / fabs(W.alr[q]);
    return q;
}

// alr[j] = rho' a_j for every nonbasic, non-fixed column whose entry passes the pivot tolerance (else 0), rho = row r of B^-1
XOD void row_alpha(const Work &W, const sens::View &s, Shared *S, int m, int n, int r, int tid, int nt) {
    const double *rho = W.B + (long long)r * m;
    double b1 = INFINITY, b2 = 0.0; int bi = kNone;
    for (int i = tid; i < m; i += nt) keep_best(b1, b2, bi, -fabs(rho[i]), 0.0, i);
    choose(S, tid, nt, b1, b2, bi);
    const double rmax = -S->r1;
    for (int j = tid; j < n; j += nt) {
        double a = 0.0, amax = 0.0;
        if (W.stat[j] != BASIC && !fixed_col(W, j))
            for (int e = sens::ld<true>(s.At_ptr + j), e1 = sens::ld<true>(s.At_ptr + j + 1); e < e1; ++e) {
                a = fma(rho[sens::ld<true>(s.At_idx + e)], W.a[e], a);
                amax = fmax(amax, fabs(W.a[e]));
            }
        W.alr[j] = fabs(a) >= kPivot * rmax * amax ? a : 0.0;
    }
    XO_SYNC();
}

// Harris ratio test of the primal step of column q in direction dir (al = B^-1 a_q): the blocking position (kNone: none) and the
// step length in *theta; the leaving variable's bound side in *to_up
XOD int primal_ratio(const Work &W, Shared *S, int m, int n, int dir, double tolp, bool bland, double *theta, int *to_up, int tid, int nt) {
    double b1 = INFINITY, b2 = 0.0; int bi = kNone;
    for (int k = tid; k < m; k += nt) keep_best(b1, b2, bi, -fabs(W.al[k]), 0.0, k);
    choose(S, tid, nt, b1, b2, bi);
    const double tol_piv = kPivot * -S->r1;
    b1 = INFINITY; b2 = 0.0; bi = kNone;
    for (int k = tid; k < m; k += nt) {
        const double s = dir * W.al[k];
        if (fabs(s) < tol_piv || s == 0.0) continue;
        const int v = W.head[k];
        const double x = W.xv[v], up = upper(W, n, v);
        if (s > 0.0) keep_best(b1, b2, bi, fmax(0.0, x + tolp) / s, 0.0, k);
        else if (up < INFINITY) keep_best(b1, b2, bi, fmax(0.0, up - x + tolp) / -s, 0.0, k);
    }
    choose(S, tid, nt, b1, b2, bi);
    if (S->rid == kNone) return kNone;
    const double tmax = S->r1;
    b1 = INFINITY; b2 = 0.0; bi = kNone;
    for (int k = tid; k < m; k += nt) {
        const double s = dir * W.al[k];
        if (fabs(s) < tol_piv || s == 0.0) continue;
        const int v = W.head[k];
        const double x = W.xv[v], up = upper(W, n, v);
        double rt;
        if (s > 0.0) rt = fmax(0.0, x) / s;
        else if (up < INFINITY) rt = fmax(0.0, up - x) / -s;
        else continue;
        if (rt <= tmax) keep_best(b1, b2, bi, bland ? 0.0 : -fabs(s), 0.0, v);
    }
    choose(S, tid, nt, b1, b2, bi);
    const int v = S->rid;
    int pos = kNone;
    for (int k = tid; k < m; k += nt) if (W.head[k] == v) S->ival[0] = k;
    XO_SYNC();
    pos = S->ival[0];
    const double s = dir * W.al[pos];
    const double x = W.xv[v];
    *to_up = s < 0.0;
    *theta = s > 0.0 ? fmax(0.0, x) / s : fmax(0.0, upper(W, n, v) - x) / -s;
    XO_SYNC();
    return pos;
}

// the outputs of LP p, computed by the threads tid = 0 .. nt-1 of one CTA (nt <= kMaxThreads); w: the LP's work region
XOD void lp_body(const Params &P, const sens::View &s, const View &X, double *w, Shared *S, long long p, int tid, int nt) {
    const int m = P.m, n = P.n;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    if (P.status[p] != 0) {          // not DSP_OPTIMAL: status passed through, rows of NaN, -1 in the basis
        for (int j = tid; j < n; j += nt) {
            P.x_out[p * n + j] = nan;
            if (P.col_status) P.col_status[p * n + j] = -1;
        }
        for (int i = tid; i < m; i += nt) {
            P.y_out[p * m + i] = nan;
            if (P.row_basic) P.row_basic[p * m + i] = -1;
        }
        if (tid == 0) {
            P.obj[p] = nan; P.xstatus[p] = P.status[p];
            if (P.pivots) P.pivots[p] = 0;
        }
        XO_SYNC();
        return;
    }
    const Work W = carve(w, m, n, P.nnz);
    const double *cp = P.cparams ? P.cparams + p * P.Pc : nullptr;
    const double *rp = P.rparams ? P.rparams + p * P.rstride : nullptr;
    const double *xin = P.x + p * n;
    // ---- the LP's data: c, u and A's values by column, b by row
    for (int j = tid; j < n; j += nt) {
        double c = sens::ld<true>(s.c0 + j);
        for (int e = sens::ld<true>(s.cm_ptr + j), e1 = sens::ld<true>(s.cm_ptr + j + 1); e < e1; ++e)
            c = fma(sens::ld<true>(s.cm_val + e), cp[sens::ld<true>(s.cm_idx + e)], c);
        W.c[j] = c;
        double u = sens::ld<true>(X.u0 + j);
        if (u < INFINITY)
            for (int e = sens::ld<true>(X.um_ptr + j), e1 = sens::ld<true>(X.um_ptr + j + 1); e < e1; ++e)
                u = fma(sens::ld<true>(X.um_val + e), rp[sens::ld<true>(X.um_idx + e)], u);
        W.u[j] = u < 0.0 ? 0.0 : u;
        for (int e = sens::ld<true>(s.At_ptr + j), e1 = sens::ld<true>(s.At_ptr + j + 1); e < e1; ++e) {
            double a = sens::ld<true>(s.At_val + e);
            for (int k = sens::ld<true>(s.tc_ptr + e), k1 = sens::ld<true>(s.tc_ptr + e + 1); k < k1; ++k)
                a = fma(sens::ld<true>(s.tc_coef + k), rp[sens::ld<true>(s.tc_param + k)], a);
            W.a[e] = a;
        }
    }
    for (int i = tid; i < m; i += nt) {
        double b = sens::ld<true>(X.b0 + i);
        for (int e = sens::ld<true>(X.bm_ptr + i), e1 = sens::ld<true>(X.bm_ptr + i + 1); e < e1; ++e)
            b = fma(sens::ld<true>(X.bm_val + e), rp[sens::ld<true>(X.bm_idx + e)], b);
        W.b[i] = b;
    }
    XO_SYNC();
    // ---- scales and tolerances
    double bp = INFINITY, bd = INFINITY;
    for (int j = tid; j < n; j += nt) { if (W.u[j] < INFINITY) bp = fmin(bp, -fabs(W.u[j])); bd = fmin(bd, -fabs(W.c[j])); }
    for (int i = tid; i < m; i += nt) bp = fmin(bp, -fabs(W.b[i]));
    choose(S, tid, nt, bp, 0.0, 0);
    const double sp = fmax(1.0, -S->r1);
    choose(S, tid, nt, bd, 0.0, 0);
    const double sd = -S->r1 > 0.0 ? -S->r1 : 1.0;
    const double tolp = kFeas * sp, told = kFeas * sd;
    // ---- start: columns within tol_p of a bound on it, the others inside; the all-artificial basis
    for (int j = tid; j < n; j += nt) {
        const double x = xin[j], u = W.u[j];
        if (x <= tolp || u <= 0.0) { W.xv[j] = 0.0; W.stat[j] = AT_LO; }
        else if (u - x <= tolp) { W.xv[j] = u; W.stat[j] = AT_UP; }
        else { W.xv[j] = x; W.stat[j] = INSIDE; }
    }
    for (int k = tid; k < m; k += nt) { W.head[k] = n + k; W.stat[n + k] = BASIC; W.xv[n + k] = 0.0; }
    const long long mm = (long long)m * m;
    for (long long e = tid; e < mm; e += nt) W.B[e] = (e / m) == (e % m) ? 1.0 : 0.0;
    XO_SYNC();
    // ---- 1. crash: the inside columns ranked by interiority (ties by index)
    for (int j = tid; j < n; j += nt) {
        if (W.stat[j] != INSIDE) continue;
        const double ij = fmin(W.xv[j], W.u[j] - W.xv[j]);
        int r = 0;
        for (int k = 0; k < n; ++k) {
            if (W.stat[k] != INSIDE) continue;
            const double ik = fmin(W.xv[k], W.u[k] - W.xv[k]);
            r += ik > ij || (ik == ij && k < j);
        }
        W.ord[r] = j;
    }
    if (tid == 0) {
        int cnt = 0;
        for (int j = 0; j < n; ++j) cnt += W.stat[j] == INSIDE;
        S->ival[1] = cnt;
    }
    XO_SYNC();
    const int ninside = S->ival[1];
    int nart = m;
    for (int r = 0; r < ninside && nart > 0; ++r) {
        const int j = W.ord[r];
        ftran(W, s, m, n, j, W.al, tid, nt);
        double b1 = INFINITY, b2 = 0.0; int bi = kNone;
        for (int k = tid; k < m; k += nt)
            if (W.head[k] >= n) keep_best(b1, b2, bi, -fabs(W.al[k]), 0.0, k);
        choose(S, tid, nt, b1, b2, bi);
        const int k = S->rid;
        double amax = 0.0;
        for (int e = sens::ld<true>(s.At_ptr + j), e1 = sens::ld<true>(s.At_ptr + j + 1); e < e1; ++e) amax = fmax(amax, fabs(W.a[e]));
        if (k == kNone || !(-S->r1 >= kPivot * amax)) continue;
        pivot(W, m, n, k, j, AT_LO, 0.0, tid, nt);
        --nart;
    }
    const int maxp = P.max_pivots;
    int npiv = 0, since = 0, status = OPTIMAL;
    solve_x(W, X, m, n, false, tid, nt);
    // ---- 2. push every column still inside its bounds onto a bound
    for (int j = 0; j < n && status == OPTIMAL; ++j) {
        if (W.stat[j] != INSIDE) continue;
        if (npiv >= maxp) { status = MAX_ITER; break; }
        solve_y(W, s, m, n, false, tid, nt);
        const double dj = W.d[j], x = W.xv[j], u = W.u[j];
        int dir = dj < -told ? 1 : dj > told ? -1 : (u - x < x ? 1 : -1);
        ftran(W, s, m, n, j, W.al, tid, nt);
        for (int attempt = 0; attempt < 2; ++attempt) {
            double theta = INFINITY; int to_up = 0;
            const int k = primal_ratio(W, S, m, n, dir, 0.0, false, &theta, &to_up, tid, nt);
            const double dist = dir > 0 ? u - x : x;
            if (k == kNone && dist == INFINITY) { dir = -dir; continue; }   // no block towards an infinite bound: go to 0 instead
            const double step = k != kNone && theta < dist ? theta : dist;
            for (int q = tid; q < m; q += nt) {
                const int v = W.head[q];
                W.xv[v] = fma(-step * (double)dir, W.al[q], W.xv[v]);
            }
            XO_SYNC();
            if (k != kNone && theta < dist) {
                const int v = W.head[k];
                if (tid == 0) W.xv[j] = fma(step, (double)dir, x);
                XO_SYNC();
                pivot(W, m, n, k, j, to_up ? AT_UP : AT_LO, to_up ? upper(W, n, v) : 0.0, tid, nt);
                XO_TRACE(TR_PUSH_PIVOT);
                ++npiv; ++since;
                if (since >= kRefactor) {
                    XO_TRACE(TR_PUSH_REINVERT);
                    if (!reinvert(W, s, S, m, n, tid, nt)) status = NUMERICAL;
                    since = 0;
                    solve_x(W, X, m, n, false, tid, nt);
                }
            } else {
                if (tid == 0) { W.xv[j] = dir > 0 ? u : 0.0; W.stat[j] = dir > 0 ? AT_UP : AT_LO; }
                XO_SYNC();
            }
            break;
        }
    }
    // ---- 3. and 4.: fresh inverse, cleanup pivots, artificials out, fresh inverse
    int degen = 0;
    for (int round = 0; round < 4 && status == OPTIMAL; ++round) {
        XO_TRACE(TR_ROUND);
        if (!reinvert(W, s, S, m, n, tid, nt)) { status = NUMERICAL; break; }
        since = 0;
        solve_x(W, X, m, n, true, tid, nt);
        solve_y(W, s, m, n, true, tid, nt);
        bool pivoted = false;
        for (;;) {
            primal_worst(W, S, m, n, tolp, tid, nt);
            const int pv = S->rid;
            const bool bland = degen >= kBlandAfter;
            double b1 = INFINITY, b2 = 0.0; int bi = kNone;
            for (int j = tid; j < n; j += nt) {
                const double di = dual_inf(W, j, told);
                if (di > 0.0) keep_best(b1, b2, bi, bland ? 0.0 : -di, 0.0, j);
            }
            choose(S, tid, nt, b1, b2, bi);
            const int q = S->rid;
            if (pv == kNone && q == kNone) break;
            if (pv != kNone && q != kNone) { status = NUMERICAL; break; }      // primal and dual infeasible
            if (npiv >= maxp) { status = MAX_ITER; break; }
            pivoted = true;
            if (bland) XO_TRACE(TR_BLAND);
            if (q != kNone) {                            // bounded primal simplex
                const int dir = W.stat[q] == AT_LO ? 1 : -1;
                ftran(W, s, m, n, q, W.al, tid, nt);
                double theta = INFINITY; int to_up = 0;
                const int k = primal_ratio(W, S, m, n, dir, tolp, bland, &theta, &to_up, tid, nt);
                const double range = W.u[q];
                if (k == kNone && range == INFINITY) { status = NUMERICAL; break; }
                if (k == kNone || range <= theta) {      // bound flip
                    if (tid == 0) { W.stat[q] = dir > 0 ? AT_UP : AT_LO; W.xv[q] = dir > 0 ? range : 0.0; }
                    XO_SYNC();
                    XO_TRACE(TR_BOUND_FLIP);
                    degen = 0;
                } else {
                    const int v = W.head[k];
                    pivot(W, m, n, k, q, to_up ? AT_UP : AT_LO, to_up ? upper(W, n, v) : 0.0, tid, nt);
                    XO_TRACE(TR_PRIMAL_PIVOT);
                    if (theta == 0.0) XO_TRACE(TR_PRIMAL_DEGENERATE);
                    degen = theta == 0.0 ? degen + 1 : 0;
                    ++since;
                }
            } else {                                     // bounded dual simplex: position of pv leaves at its violated bound
                int r = kNone;
                for (int k = tid; k < m; k += nt) if (W.head[k] == pv) S->ival[2] = k;
                XO_SYNC();
                r = S->ival[2];
                const bool below = W.xv[pv] < 0.0;
                row_alpha(W, s, S, m, n, r, tid, nt);
                double ratio = 0.0;
                const int e = dual_ratio(W, S, n, below ? -1 : 1, told, bland, &ratio, tid, nt);
                if (e == kNone) { status = NUMERICAL; break; }
                ftran(W, s, m, n, e, W.al, tid, nt);
                pivot(W, m, n, r, e, below ? AT_LO : AT_UP, below ? 0.0 : upper(W, n, pv), tid, nt);
                XO_TRACE(TR_DUAL_PIVOT);
                degen = ratio == 0.0 ? degen + 1 : 0;
                ++since;
            }
            ++npiv;
            if (since >= kRefactor) {
                XO_TRACE(TR_CLEANUP_REINVERT);
                if (!reinvert(W, s, S, m, n, tid, nt)) { status = NUMERICAL; break; }
                since = 0;
            }
            solve_x(W, X, m, n, false, tid, nt);
            solve_y(W, s, m, n, false, tid, nt);
        }
        if (status != OPTIMAL) break;
        // artificials out: a degenerate pivot with the dual ratio test in the direction of the smaller dual step
        for (int r = 0; r < m; ++r) {
            if (W.head[r] < n) continue;
            if (npiv >= maxp) { status = MAX_ITER; break; }
            row_alpha(W, s, S, m, n, r, tid, nt);
            double rp_ = INFINITY, rn_ = INFINITY;
            const int ep = dual_ratio(W, S, n, 1, told, false, &rp_, tid, nt);
            const int en = dual_ratio(W, S, n, -1, told, false, &rn_, tid, nt);
            const int e = ep == kNone ? en : en == kNone ? ep : (rn_ < rp_ ? en : ep);
            if (e == kNone) { XO_TRACE(TR_REDUNDANT_ROW); continue; }   // a redundant row: its artificial stays basic at 0
            ftran(W, s, m, n, e, W.al, tid, nt);
            pivot(W, m, n, r, e, AT_LO, 0.0, tid, nt);
            XO_TRACE(TR_ARTIFICIAL_OUT);
            ++npiv; ++since; pivoted = true;
            if (since >= kRefactor) {
                XO_TRACE(TR_CLEANUP_REINVERT);
                if (!reinvert(W, s, S, m, n, tid, nt)) { status = NUMERICAL; break; }
                since = 0;
            }
            solve_x(W, X, m, n, false, tid, nt);
            solve_y(W, s, m, n, false, tid, nt);
        }
        if (status != OPTIMAL || !pivoted) break;
    }
    if (status == OPTIMAL) {                             // the final basic solution, from a fresh inverse
        if (!reinvert(W, s, S, m, n, tid, nt)) status = NUMERICAL;
        else {
            solve_x(W, X, m, n, true, tid, nt);
            solve_y(W, s, m, n, true, tid, nt);
            primal_worst(W, S, m, n, tolp, tid, nt);
            const int pv = S->rid;
            double b1 = INFINITY, b2 = 0.0; int bi = kNone;
            for (int j = tid; j < n; j += nt)
                if (dual_inf(W, j, told) > 0.0) keep_best(b1, b2, bi, 0.0, 0.0, j);
            choose(S, tid, nt, b1, b2, bi);
            if (pv != kNone || S->rid != kNone) status = NUMERICAL;
        }
    }
    // ---- outputs
    for (int j = tid; j < n; j += nt) {
        P.x_out[p * n + j] = W.xv[j];
        if (P.col_status) {
            int st = W.stat[j] == INSIDE ? -1 : W.stat[j];
            if (st != BASIC && fixed_col(W, j)) st = W.d[j] < 0.0 ? AT_UP : AT_LO;   // u_j = 0: the bound the sign of d_j asks for
            P.col_status[p * n + j] = (signed char)st;
        }
    }
    for (int i = tid; i < m; i += nt) {
        P.y_out[p * m + i] = W.y[i];
        if (P.row_basic) P.row_basic[p * m + i] = (signed char)(W.stat[n + i] == BASIC);
    }
    if (tid == 0) {
        double o = P.o0;
        for (int q = 0; q < P.Pr; ++q) o = fma(sens::ld<true>(s.omap + q), rp[q], o);
        for (int q = 0; q < P.Pc; ++q) o = fma(sens::ld<true>(s.ocmap + q), cp[q], o);
        double cx = 0.0;
        for (int j = 0; j < n; ++j) cx = fma(W.c[j], W.xv[j], cx);
        P.obj[p] = cx + o;
        P.xstatus[p] = status;
        if (P.pivots) P.pivots[p] = npiv;
    }
    XO_SYNC();
}

// ---- host: the crossover's structure blob, in the caller's order (b0 and Bmap by row, u0 and Umap by column, the CSR of A with the
// CSC position of every entry, matching sens::build_blob's CSC)
inline Layout build_blob(const sens::HostTemplate &T, const std::vector<double> &b0, const std::vector<double> &u0,
                         std::vector<unsigned char> &blob) {
    const int m = T.m, n = T.n;
    std::vector<int> ccol(n), crow(m), rpos(m), kpos(n);
    for (int k = 0; k < n; ++k) ccol[k] = T.col_perm.empty() ? k : T.col_perm[k];
    for (int k = 0; k < m; ++k) crow[k] = T.row_perm.empty() ? k : T.row_perm[k];
    for (int k = 0; k < m; ++k) rpos[crow[k]] = k;
    for (int k = 0; k < n; ++k) kpos[ccol[k]] = k;
    std::vector<double> db0(m), du0(n), bmv, umv;
    std::vector<int> bmp(1, 0), bmi, ump(1, 0), umi;
    for (int R = 0; R < m; ++R) {
        db0[R] = b0[rpos[R]];
        for (int e = T.bm_ptr[rpos[R]]; e < T.bm_ptr[rpos[R] + 1]; ++e) { bmi.push_back(T.bm_idx[e]); bmv.push_back(T.bm_val[e]); }
        bmp.push_back((int)bmi.size());
    }
    for (int C = 0; C < n; ++C) {
        const int k = kpos[C];
        du0[C] = k < T.nb ? u0[k] : INFINITY;
        if (k < T.nb)
            for (int e = T.um_ptr[k]; e < T.um_ptr[k + 1]; ++e) { umi.push_back(T.um_idx[e]); umv.push_back(T.um_val[e]); }
        ump.push_back((int)umi.size());
    }
    // the CSC position of every entry: sens::build_blob pushes entries by caller row, then groups them stably by caller column
    std::vector<int> cnt(n + 1, 0);
    for (int q = 0; q < T.A_ptr[m]; ++q) cnt[ccol[T.A_idx[q]] + 1]++;
    for (int C = 0; C < n; ++C) cnt[C + 1] += cnt[C];
    std::vector<int> fill(cnt.begin(), cnt.end() - 1), rp(1, 0), rposv, rcol;
    for (int R = 0; R < m; ++R) {
        std::vector<std::pair<int, int>> row;         // (caller column, CSC position), by column
        for (int q = T.A_ptr[rpos[R]]; q < T.A_ptr[rpos[R] + 1]; ++q) { const int C = ccol[T.A_idx[q]]; row.push_back({C, fill[C]++}); }
        std::sort(row.begin(), row.end());
        for (auto &e : row) { rcol.push_back(e.first); rposv.push_back(e.second); }
        rp.push_back((int)rcol.size());
    }
    Layout L;
    std::vector<double> dv;
    std::vector<int> iv;
    auto pd = [&dv](const std::vector<double> &v) { const long long at = (long long)dv.size(); dv.insert(dv.end(), v.begin(), v.end()); return at; };
    auto pi = [&iv](const std::vector<int> &v) { const long long at = (long long)iv.size(); iv.insert(iv.end(), v.begin(), v.end()); return at; };
    L.b0 = pd(db0); L.bm_val = pd(bmv); L.u0 = pd(du0); L.um_val = pd(umv);
    L.bm_ptr = pi(bmp); L.bm_idx = pi(bmi); L.um_ptr = pi(ump); L.um_idx = pi(umi); L.r_ptr = pi(rp); L.r_pos = pi(rposv); L.r_col = pi(rcol);
    L.ioff = (long long)dv.size() * 8;
    L.bytes = (L.ioff + (long long)iv.size() * 4 + 15) / 16 * 16;
    blob.assign((size_t)L.bytes, 0);
    if (!dv.empty()) memcpy(blob.data(), dv.data(), dv.size() * 8);
    if (!iv.empty()) memcpy(blob.data() + L.ioff, iv.data(), iv.size() * 4);
    return L;
}

}  // namespace xo
