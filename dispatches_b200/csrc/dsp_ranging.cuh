// dsp_ranging.cuh -- ranging post-pass over given bases (dsp_lp_ranging, include/dsp_lp.h): for every LP and every direction k of the
// batch parameters, the interval [theta_lo, theta_hi] of theta over which the given basis stays optimal for the parameters
// (cp + theta dir_c[k], rp + theta dir_r[k]), and the objective's first and second derivative along the direction inside it.
//
// For one LP  min c'x + k  s.t.  A x = b, 0 <= x <= u  in the CALLER's column / row order (the LP dsp_lp_crossover sees) and a basis in
// its convention (col_status 0 / 1 / 2, row_basic: the row's artificial, a unit column with bounds [0, 0], is basic):
//   1. the basis head in a fixed order: the basic columns by index, then the basic artificials by row.  A basis without m members, or
//      with a column at an infinite upper bound, is DSP_NUMERICAL.
//   2. B^-1 by xo::reinvert; x_B, y and d = c - A'y with one step of iterative refinement each (crossover step 3).  A basis that is not
//      primal and dual feasible within the crossover's tol_p / tol_d is DSP_NUMERICAL.
//   3. per direction: dc = Cmap dir_c, db = Bmap dir_r, du = Umap dir_r (0 where u is infinite); dy = B^-T dc_B, dd_j = dc_j - a_j'dy;
//      dx_B = B^-1 (db - sum over columns j at u of a_j du_j), dx_j = du_j at u, 0 at 0.  Along theta every quantity g moves as
//      g + theta dg, and each of these must keep its sign:
//        x_B >= 0 and u_B - x_B >= 0 (finite u); u_j >= 0 of a column at u; d_j >= 0 at 0 and -d_j >= 0 at u, for the columns not fixed
//        at 0 along the direction (u_j = du_j = 0 imposes nothing, nor does a nonbasic artificial).  A column with u_j = 0 and
//        du_j != 0 whose d_j already has the wrong sign beyond tol_d (any bound is optimal for a fixed column) gives 0 on the side
//        where u_j(theta) > 0.  A basic artificial must stay 0: a non-negligible dx of one gives [0, 0].
//      An entry blocks at g / |dg| on the side where dg < 0 moves it towards its bound; an entry within tolerance of its bound
//      (g <= tol_p, tol_d) counts as on it and blocks at 0; an entry whose rate is negligible, |dg| <= kRate times the direction's scale
//      (max(|db|_inf, |du|_inf) on the primal side, |dc|_inf on the dual side), does not block.  The range is the block-wide minimum
//      of each side, +-inf where nothing blocks.
//      obj(theta) = obj + dobj theta + d2obj theta^2 / 2 with dobj = dc'x + c'dx + omap'dir_r + ocmap'dir_c and d2obj = 2 dc'dx.
//      A direction with a nonzero dir_r entry on a parameter that enters a matrix term gets NaN in all four outputs: A moves and the
//      objective is not piecewise quadratic along it.
//      Step 3 is rg::segment, which the parametric walk (dsp_parametric.cuh) calls for every segment of its walk.
//
// Layout: the crossover's (dsp_crossover.cuh): one CTA per LP, LPs handed out grid-stride, the work region (B^-1, the LP's vectors and
// the direction's) in shared memory or in the handle's workspace.  Every element is summed by one thread in a fixed order and every
// minimum is an exact comparison, so the results do not depend on the number of threads or on where an LP sits in the batch.
//
// Plain C++ over a thread index: tests/emu compiles this file with g++ on the SIMT emulator (one warp as the CTA).
#pragma once

#include "dsp_crossover.cuh"

namespace rg {

constexpr double kRate = 1e-9;    // a rate of change at most this, relative to the direction's scale, does not block

struct Params {
    int m, n, Pc, Pr, nnz, K;
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    const int *status;
    const signed char *col_status, *row_basic;
    const double *dir_c, *dir_r;           // [K,Pc] / [K,Pr], or [N,K,Pc] / [N,K,Pr] with dir_per_lp; each may be null (0)
    int dir_per_lp;
    double o0;
    double *lo, *hi, *dobj, *d2obj;        // [N,K]; dobj and d2obj may be null
    int *rstatus;
    const unsigned char *blob;             // the sensitivity pass's structure
    sens::Layout L;
    const unsigned char *xblob;            // the crossover's structure
    xo::Layout X;
    double *ws;                            // work regions in global memory (null: shared memory)
    long long ws_stride;                   // doubles per CTA
};

// doubles of one LP's work region: the crossover's, then dc, du, dx (n each), db, dy (m each)
XOHD long long work_doubles(int m, int n, int nnz) { return xo::work_doubles(m, n, nnz) + (3LL * n + 2LL * m + 1) / 2 * 2; }

// block kinds of the upper side (for the parametric walk, dsp_parametric.cuh): a basic column reaching 0 or its u, a basic artificial
// leaving 0, a nonbasic column at u whose u reaches 0, a reduced cost reaching 0, a fixed column unfixed at the wrong bound
enum { BK_BASIC_LO = 0, BK_BASIC_UP = 1, BK_ARTIFICIAL = 2, BK_BOUND = 3, BK_DUAL = 4, BK_UNFIX = 5 };

// the tighter of the two sides g + theta dg >= 0 may block: into *hi when dg < 0, into *lo (as a distance) when dg > 0.  The upper
// side keeps its blocking entry, the smallest (ratio, class, id) with id = variable * 8 + kind and class -1 for a fixed column
// unfixed at the wrong bound (a flip that changes no value), 0 for a primal entry, 1 for a dual one
XOD void block(double g, double dg, double tol, double rtol, double *hi, double *lo, double *hc, int *hid, double cls, int id) {
    if (!(fabs(dg) > rtol)) return;
    const double r = g <= tol ? 0.0 : g / fabs(dg);
    if (dg < 0.0) xo::keep_best(*hi, *hc, *hid, r, cls, id);
    else *lo = fmin(*lo, r);
}

// the block's largest |v| of its threads' own largest
XOD double block_max(xo::Shared *S, int tid, int nt, double v) {
    xo::choose(S, tid, nt, -v, 0.0, 0);
    return -S->r1;
}

// one range of a basis along a direction: hi / lo as distances from the current point, the blocking entry of the upper side
// (variable * 8 + kind, xo::kNone where nothing blocks), and (thread 0 only) the objective's first and second derivative
struct Segment { double hi, lo, d1, d2; int block; };

// step 3 for the direction (gc, gr) on the current basis, x_B, y and d: dc, du, db, dy, dd = dc - A'dy and dx of every column (dx_B
// also in W.al), then the ratio tests.  tolp / told: the on-bound tolerances.
XOD Segment segment(const sens::View &s, const xo::View &X, const xo::Work &W, xo::Shared *S, int m, int n, int Pc, int Pr,
                    const double *gc, const double *gr, double *dc, double *du, double *dx, double *db, double *dy, double *dd,
                    double tolp, double told, int tid, int nt) {
    double sdp = 0.0, sdd = 0.0;
    for (int j = tid; j < n; j += nt) {
        double v = 0.0;
        if (gc)
            for (int e = sens::ld<true>(s.cm_ptr + j), e1 = sens::ld<true>(s.cm_ptr + j + 1); e < e1; ++e)
                v = fma(sens::ld<true>(s.cm_val + e), gc[sens::ld<true>(s.cm_idx + e)], v);
        dc[j] = v;
        double g = 0.0;
        if (gr && sens::ld<true>(X.u0 + j) < INFINITY)
            for (int e = sens::ld<true>(X.um_ptr + j), e1 = sens::ld<true>(X.um_ptr + j + 1); e < e1; ++e)
                g = fma(sens::ld<true>(X.um_val + e), gr[sens::ld<true>(X.um_idx + e)], g);
        du[j] = g;
        sdd = fmax(sdd, fabs(v)); sdp = fmax(sdp, fabs(g));
    }
    for (int i = tid; i < m; i += nt) {
        double v = 0.0;
        if (gr)
            for (int e = sens::ld<true>(X.bm_ptr + i), e1 = sens::ld<true>(X.bm_ptr + i + 1); e < e1; ++e)
                v = fma(sens::ld<true>(X.bm_val + e), gr[sens::ld<true>(X.bm_idx + e)], v);
        db[i] = v;
        sdp = fmax(sdp, fabs(v));
    }
    sdp = block_max(S, tid, nt, sdp);
    sdd = block_max(S, tid, nt, sdd);
    // dy = B^-T dc_B, dd = dc - A'dy; the right-hand side of dx_B (into t1)
    for (int q = tid; q < m; q += nt) W.t2[q] = W.head[q] < n ? dc[W.head[q]] : 0.0;
    for (int i = tid; i < m; i += nt) {
        double r = db[i];
        for (int q = sens::ld<true>(X.r_ptr + i), q1 = sens::ld<true>(X.r_ptr + i + 1); q < q1; ++q) {
            const int j = sens::ld<true>(X.r_col + q);
            if (W.stat[j] == xo::AT_UP) r = fma(-W.a[sens::ld<true>(X.r_pos + q)], du[j], r);
        }
        W.t1[i] = r;
    }
    XO_SYNC();
    for (int i = tid; i < m; i += nt) {
        double r = 0.0;
        for (int q = 0; q < m; ++q) r = fma(W.t2[q], W.B[(long long)q * m + i], r);
        dy[i] = r;
    }
    for (int q = tid; q < m; q += nt) {
        double r = 0.0;
        for (int i = 0; i < m; ++i) r = fma(W.B[(long long)q * m + i], W.t1[i], r);
        W.al[q] = r;
    }
    XO_SYNC();
    for (int j = tid; j < n; j += nt) {
        dd[j] = dc[j] - xo::col_dot(W, s, n, j, dy);
        dx[j] = W.stat[j] == xo::AT_UP ? du[j] : 0.0;
    }
    XO_SYNC();
    for (int q = tid; q < m; q += nt) if (W.head[q] < n) dx[W.head[q]] = W.al[q];
    // the ratio tests: hi and lo as distances from 0
    const double rtp = kRate * sdp, rtd = kRate * sdd;
    double hi = INFINITY, lo = INFINITY, hc = 0.0;
    int hid = xo::kNone;
    for (int q = tid; q < m; q += nt) {
        const int v = W.head[q];
        const double x = W.xv[v], g = W.al[q];
        if (v >= n) {
            if (fabs(g) > rtp) { xo::keep_best(hi, hc, hid, 0.0, 0.0, v * 8 + BK_ARTIFICIAL); lo = 0.0; }
            continue;
        }
        block(x, g, tolp, rtp, &hi, &lo, &hc, &hid, 0.0, v * 8 + BK_BASIC_LO);
        if (W.u[v] < INFINITY) block(W.u[v] - x, du[v] - g, tolp, rtp, &hi, &lo, &hc, &hid, 0.0, v * 8 + BK_BASIC_UP);
    }
    for (int j = tid; j < n; j += nt) {
        const int st = W.stat[j];
        if (st == xo::BASIC) continue;
        if (st == xo::AT_UP) block(W.u[j], du[j], tolp, rtp, &hi, &lo, &hc, &hid, 0.0, j * 8 + BK_BOUND);
        if (W.u[j] <= 0.0) {         // fixed at 0 at theta = 0, its bound free of the sign of d_j
            if (du[j] == 0.0) continue;
            if ((st == xo::AT_LO ? W.d[j] : -W.d[j]) < -told) {     // at the wrong bound: optimal only while u_j stays 0
                if (du[j] > 0.0) xo::keep_best(hi, hc, hid, 0.0, -1.0, j * 8 + BK_UNFIX);
                else lo = 0.0;
                continue;
            }
        }
        if (st == xo::AT_LO) block(W.d[j], dd[j], told, rtd, &hi, &lo, &hc, &hid, 1.0, j * 8 + BK_DUAL);
        else block(-W.d[j], -dd[j], told, rtd, &hi, &lo, &hc, &hid, 1.0, j * 8 + BK_DUAL);
    }
    Segment g;
    xo::choose(S, tid, nt, hi, hc, hid);
    g.hi = S->r1; g.block = S->rid;
    xo::choose(S, tid, nt, lo, 0.0, 0);
    g.lo = S->r1;
    g.d1 = g.d2 = 0.0;
    if (tid == 0) {
        double d1 = 0.0, d2 = 0.0;
        for (int j = 0; j < n; ++j) {
            d1 = fma(dc[j], W.xv[j], d1);
            d1 = fma(W.c[j], dx[j], d1);
            d2 = fma(dc[j], dx[j], d2);
        }
        if (gr) for (int q = 0; q < Pr; ++q) d1 = fma(sens::ld<true>(s.omap + q), gr[q], d1);
        if (gc) for (int q = 0; q < Pc; ++q) d1 = fma(sens::ld<true>(s.ocmap + q), gc[q], d1);
        g.d1 = d1; g.d2 = 2.0 * d2;
    }
    return g;
}

// the outputs of LP p, computed by the threads tid = 0 .. nt-1 of one CTA (nt <= xo::kMaxThreads); w: the LP's work region
XOD void lp_body(const Params &P, const sens::View &s, const xo::View &X, double *w, xo::Shared *S, long long p, int tid, int nt) {
    const int m = P.m, n = P.n, K = P.K;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    auto nan_row = [&](int status) {
        for (int k = tid; k < K; k += nt) {
            P.lo[p * K + k] = nan; P.hi[p * K + k] = nan;
            if (P.dobj) P.dobj[p * K + k] = nan;
            if (P.d2obj) P.d2obj[p * K + k] = nan;
        }
        if (tid == 0) P.rstatus[p] = status;
        XO_SYNC();
    };
    if (P.status[p] != 0) { nan_row(P.status[p]); return; }     // not DSP_OPTIMAL: passed through
    const xo::Work W = xo::carve(w, m, n, P.nnz);
    double *dc = w + xo::work_doubles(m, n, P.nnz), *du = dc + n, *dx = du + n, *db = dx + n, *dy = db + m;
    const double *cp = P.cparams ? P.cparams + p * P.Pc : nullptr;
    const double *rp = P.rparams ? P.rparams + p * P.rstride : nullptr;
    // ---- the LP's data: c, u and A's values by column, b by row (as the crossover forms them)
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
    // ---- scales and tolerances (the crossover's)
    double bp = INFINITY, bd = INFINITY;
    for (int j = tid; j < n; j += nt) { if (W.u[j] < INFINITY) bp = fmin(bp, -fabs(W.u[j])); bd = fmin(bd, -fabs(W.c[j])); }
    for (int i = tid; i < m; i += nt) bp = fmin(bp, -fabs(W.b[i]));
    xo::choose(S, tid, nt, bp, 0.0, 0);
    const double sp = fmax(1.0, -S->r1);
    xo::choose(S, tid, nt, bd, 0.0, 0);
    const double sd = -S->r1 > 0.0 ? -S->r1 : 1.0;
    const double tolp = xo::kFeas * sp, told = xo::kFeas * sd;
    // ---- 1. the basis: nonbasic columns on their bound, the head in a fixed order
    const signed char *cs = P.col_status + p * n, *rb = P.row_basic + p * m;
    for (int j = tid; j < n; j += nt) {
        const int st = cs[j];
        W.stat[j] = st == 1 ? xo::BASIC : st == 2 ? xo::AT_UP : xo::AT_LO;
        W.xv[j] = st == 2 ? W.u[j] : 0.0;
    }
    for (int i = tid; i < m; i += nt) { W.stat[n + i] = rb[i] == 1 ? xo::BASIC : xo::AT_LO; W.xv[n + i] = 0.0; }
    if (tid == 0) {
        int cnt = 0, bad = 0;
        for (int j = 0; j < n; ++j) {
            const int st = cs[j];
            if (st == 1) { if (cnt < m) W.head[cnt] = j; ++cnt; }
            else if (st != 0 && !(st == 2 && W.u[j] < INFINITY)) bad = 1;
        }
        for (int i = 0; i < m; ++i) {
            if (rb[i] == 1) { if (cnt < m) W.head[cnt] = n + i; ++cnt; }
            else if (rb[i] != 0) bad = 1;
        }
        S->ival[0] = bad || cnt != m;
    }
    XO_SYNC();
    if (S->ival[0]) { nan_row(xo::NUMERICAL); return; }
    // ---- 2. B^-1, x_B, y and d; the basis must be primal and dual feasible within tolerance
    if (!xo::reinvert(W, s, S, m, n, tid, nt)) { nan_row(xo::NUMERICAL); return; }
    xo::solve_x(W, X, m, n, true, tid, nt);
    xo::solve_y(W, s, m, n, true, tid, nt);
    xo::primal_worst(W, S, m, n, tolp, tid, nt);
    const int pv = S->rid;
    {
        double b1 = INFINITY, b2 = 0.0; int bi = xo::kNone;
        for (int j = tid; j < n; j += nt)
            if (xo::dual_inf(W, j, told) > 0.0) xo::keep_best(b1, b2, bi, 0.0, 0.0, j);
        xo::choose(S, tid, nt, b1, b2, bi);
    }
    if (pv != xo::kNone || S->rid != xo::kNone) { nan_row(xo::NUMERICAL); return; }
    // ---- 3. every direction
    for (int k = 0; k < K; ++k) {
        const double *gc = P.dir_c ? P.dir_c + ((P.dir_per_lp ? p * K : 0) + k) * P.Pc : nullptr;
        const double *gr = P.dir_r ? P.dir_r + ((P.dir_per_lp ? p * K : 0) + k) * P.Pr : nullptr;
        if (tid == 0) {                  // does the direction move a parameter that enters a matrix term?
            int moves = 0;
            if (gr)
                for (int q = 0; q < P.Pr; ++q) moves |= gr[q] != 0.0 && sens::ld<true>(s.tp_ptr + q + 1) > sens::ld<true>(s.tp_ptr + q);
            S->ival[1] = moves;
        }
        XO_SYNC();
        if (S->ival[1]) {
            if (tid == 0) {
                P.lo[p * K + k] = nan; P.hi[p * K + k] = nan;
                if (P.dobj) P.dobj[p * K + k] = nan;
                if (P.d2obj) P.d2obj[p * K + k] = nan;
            }
            XO_SYNC();
            continue;
        }
        const Segment g = segment(s, X, W, S, m, n, P.Pc, P.Pr, gc, gr, dc, du, dx, db, dy, W.alr, tolp, told, tid, nt);
        if (tid == 0) {
            P.lo[p * K + k] = 0.0 - g.lo; P.hi[p * K + k] = g.hi;
            if (P.dobj) P.dobj[p * K + k] = g.d1;
            if (P.d2obj) P.d2obj[p * K + k] = g.d2;
        }
        XO_SYNC();
    }
    if (tid == 0) P.rstatus[p] = xo::OPTIMAL;
    XO_SYNC();
}

}  // namespace rg
