// dsp_parametric.cuh -- parametric simplex walk over given bases (dsp_lp_parametric, include/dsp_lp.h): for every LP and every direction
// k of the batch parameters, the exact optimal value along theta in [0, theta_end] with the parameters at (cp + theta dir_c[k],
// rp + theta dir_r[k]), as an event log of basis changes and bound flips with the objective's value and derivatives at each.
//
// For one LP  min c'x + k  s.t.  A x = b, 0 <= x <= u  in the CALLER's order (the LP dsp_lp_crossover sees) and a basis in its
// convention that is optimal at theta = 0:
//   1. set-up as dsp_ranging.cuh steps 1-2: the LP's data, the scales and tol_p / tol_d, the basis head in a fixed order, B^-1 by
//      xo::reinvert and x_B, y, d with refinement.  A basis that is not primal and dual feasible is DSP_NUMERICAL.
//   2. segment: the ranging's per-direction quantities and the upper side of its range (rg::segment), with the entry that blocks
//      there.  The event opening the segment records theta, obj(theta) = c'x + k from the current basis, and the segment's dobj and
//      d2obj.  A segment that reaches theta_end, or that nothing blocks, ends the walk DSP_OPTIMAL.
//   3. event at the breakpoint theta' = theta + hi: the parameters are formed afresh there, one fma per parameter, and c, b, u, x_B,
//      y, d and the tolerances recomputed from the basis.  Then, by the kind of block:
//        a basic variable at 0 or u_B (an artificial leaving 0): a dual simplex pivot, the variable leaving to the bound it hit.
//          The entering column, among the nonbasic columns with u > 0 or unfixed by the direction, minimises (ratio, rate, -|alpha|,
//          index), ratio = dual slack / |alpha| and rate its derivative in theta, so that the new basis stays dual feasible just past
//          theta'.  No candidate: DSP_INFEASIBLE.
//        a reduced cost at 0: a primal simplex pivot with that column entering, the leaving position minimising (ratio, rate,
//          -|alpha|, index) over x_B (ratio max(gap, 0) / |alpha|, no Harris tolerance, so that a basic variable exactly at its bound
//          leaves before one a rounding error away from it); the column flips to its other bound if it reaches it first.  Nothing
//          blocks and no other bound: DSP_UNBOUNDED.
//        a nonbasic column at u whose u reaches 0: DSP_INFEASIBLE (the library's negative-bound rule).
//        a fixed column (u = 0) that the direction unfixes at the bound its reduced cost does not ask for: a flip to the other bound,
//          a zero-length event.
//      B^-1 by product-form updates, rebuilt every xo::kRefactor events.  After xo::kBlandAfter zero-length events in a row the ties
//      of the ratio and rate go to the lowest index instead of the largest |alpha| (a lowest-index tie-break, not Bland's rule: the
//      blocking entry still comes from rg::segment's order; a walk that cycles ends DSP_MAX_ITER at S events).  A singular
//      reinversion, or a basis that is primal and dual
//      infeasible at once after an event, is DSP_NUMERICAL.  An INFEASIBLE or UNBOUNDED walk ends with an event at the breakpoint
//      that has enter = leave = -1 and NaN derivatives: the curve stops there.  S events before theta_end: DSP_MAX_ITER.
//
// Layout: one CTA per (LP, direction) pair, pairs handed out grid-stride; the work region (the ranging's, then dd and the moved
// parameters) in shared memory or in the handle's workspace.  Every element is summed by one thread in a fixed order and every
// choice is an exact comparison with ties by index, so a walk does not depend on the number of threads or on where its pair sits.
//
// Plain C++ over a thread index: tests/emu compiles this file with g++ on the SIMT emulator (one warp as the CTA).
#pragma once

#include "dsp_ranging.cuh"

namespace pm {

enum { OPTIMAL = 0, MAX_ITER = 1, NUMERICAL = 2, INFEASIBLE = 3, UNBOUNDED = 4 };

struct Params {
    int m, n, Pc, Pr, nnz, K, S;
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    const int *status;
    const signed char *col_status, *row_basic;
    const double *dir_c, *dir_r;           // [K,Pc] / [K,Pr], or [N,K,Pc] / [N,K,Pr] with dir_per_lp; each may be null (0)
    int dir_per_lp;
    const double *theta_end;               // [K], or [N,K] with dir_per_lp
    double o0;
    double *theta, *obj, *dobj, *d2obj;    // [N,K,S]; d2obj may be null
    int *enter, *leave;                    // [N,K,S], each may be null
    signed char *leave_to;                 // [N,K,S] or null
    int *count, *pstatus;                  // [N,K]
    const unsigned char *blob;             // the sensitivity pass's structure
    sens::Layout L;
    const unsigned char *xblob;            // the crossover's structure
    xo::Layout X;
    double *ws;                            // work regions in global memory (null: shared memory)
    long long ws_stride;                   // doubles per CTA
};

// doubles of one pair's work region: the ranging's, then dd (n), the parameters at theta (Pc, Pr)
XOHD long long work_doubles(int m, int n, int nnz, int Pc, int Pr) {
    return rg::work_doubles(m, n, nnz) + ((long long)n + Pc + Pr + 1) / 2 * 2;
}

// c, u (clipped at 0) and, with with_a, A's values by column; b by row: the crossover's formulas at the parameters (cp, rp)
XOD void form(const sens::View &s, const xo::View &X, const xo::Work &W, int m, int n, const double *cp, const double *rp, bool with_a,
              int tid, int nt) {
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
        if (with_a)
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
}

// the crossover's tol_p / tol_d of the LP in W
XOD void tolerances(const xo::Work &W, xo::Shared *S, int m, int n, double *tolp, double *told, int tid, int nt) {
    double bp = INFINITY, bd = INFINITY;
    for (int j = tid; j < n; j += nt) { if (W.u[j] < INFINITY) bp = fmin(bp, -fabs(W.u[j])); bd = fmin(bd, -fabs(W.c[j])); }
    for (int i = tid; i < m; i += nt) bp = fmin(bp, -fabs(W.b[i]));
    xo::choose(S, tid, nt, bp, 0.0, 0);
    const double sp = fmax(1.0, -S->r1);
    xo::choose(S, tid, nt, bd, 0.0, 0);
    const double sd = -S->r1 > 0.0 ? -S->r1 : 1.0;
    *tolp = xo::kFeas * sp; *told = xo::kFeas * sd;
}

// 0: primal and dual feasible within tolerance; 1: one of the two; 2: neither
XOD int infeasible(const xo::Work &W, xo::Shared *S, int m, int n, double tolp, double told, int tid, int nt) {
    xo::primal_worst(W, S, m, n, tolp, tid, nt);
    const int pv = S->rid;
    double b1 = INFINITY, b2 = 0.0; int bi = xo::kNone;
    for (int j = tid; j < n; j += nt)
        if (xo::dual_inf(W, j, told) > 0.0) xo::keep_best(b1, b2, bi, 0.0, 0.0, j);
    xo::choose(S, tid, nt, b1, b2, bi);
    return (pv != xo::kNone) + (S->rid != xo::kNone);
}

// xo::row_alpha over the columns that can enter just past theta: the nonbasic columns with u > 0 and those with u = 0 that the
// direction unfixes (du > 0)
XOD void row_alpha(const xo::Work &W, const sens::View &s, xo::Shared *S, int m, int n, int r, const double *du, int tid, int nt) {
    const double *rho = W.B + (long long)r * m;
    double b1 = INFINITY, b2 = 0.0; int bi = xo::kNone;
    for (int i = tid; i < m; i += nt) xo::keep_best(b1, b2, bi, -fabs(rho[i]), 0.0, i);
    xo::choose(S, tid, nt, b1, b2, bi);
    const double rmax = -S->r1;
    for (int j = tid; j < n; j += nt) {
        double a = 0.0, amax = 0.0;
        if (W.stat[j] != xo::BASIC && (W.u[j] > 0.0 || du[j] > 0.0))
            for (int e = sens::ld<true>(s.At_ptr + j), e1 = sens::ld<true>(s.At_ptr + j + 1); e < e1; ++e) {
                a = fma(rho[sens::ld<true>(s.At_idx + e)], W.a[e], a);
                amax = fmax(amax, fabs(W.a[e]));
            }
        W.alr[j] = fabs(a) >= xo::kPivot * rmax * amax ? a : 0.0;
    }
    XO_SYNC();
}

// the basis position of variable v
XOD int position(const xo::Work &W, xo::Shared *S, int m, int v, int tid, int nt) {
    for (int k = tid; k < m; k += nt) if (W.head[k] == v) S->ival[2] = k;
    XO_SYNC();
    const int r = S->ival[2];
    XO_SYNC();
    return r;
}

// the walk of pair pk = p K + k, computed by the threads tid = 0 .. nt-1 of one CTA (nt <= xo::kMaxThreads); w: its work region
XOD void pair_body(const Params &P, const sens::View &s, const xo::View &X, double *w, xo::Shared *S, long long pk, int tid, int nt) {
    const int m = P.m, n = P.n, K = P.K, NS = P.S;
    const long long p = pk / K, ev = pk * NS;
    const int k = (int)(pk % K);
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    // entries from `from` on NaN / -1, the count and the status
    auto finish = [&](int from, int status) {
        for (int e = from + tid; e < NS; e += nt) {
            P.theta[ev + e] = nan; P.obj[ev + e] = nan; P.dobj[ev + e] = nan;
            if (P.d2obj) P.d2obj[ev + e] = nan;
            if (P.enter) P.enter[ev + e] = -1;
            if (P.leave) P.leave[ev + e] = -1;
            if (P.leave_to) P.leave_to[ev + e] = -1;
        }
        if (tid == 0) { P.count[pk] = from; P.pstatus[pk] = status; }
        XO_SYNC();
    };
    if (P.status[p] != 0) { finish(0, P.status[p]); return; }     // not DSP_OPTIMAL: passed through
    const double *gc = P.dir_c ? P.dir_c + ((P.dir_per_lp ? p * K : 0) + k) * P.Pc : nullptr;
    const double *gr = P.dir_r ? P.dir_r + ((P.dir_per_lp ? p * K : 0) + k) * P.Pr : nullptr;
    if (tid == 0) {                      // does the direction move a parameter that enters a matrix term?
        int moves = 0;
        if (gr)
            for (int q = 0; q < P.Pr; ++q) moves |= gr[q] != 0.0 && sens::ld<true>(s.tp_ptr + q + 1) > sens::ld<true>(s.tp_ptr + q);
        S->ival[1] = moves;
    }
    XO_SYNC();
    if (S->ival[1]) { finish(0, NUMERICAL); return; }
    const double te = P.theta_end[P.dir_per_lp ? pk : k];
    const xo::Work W = xo::carve(w, m, n, P.nnz);
    double *dc = w + xo::work_doubles(m, n, P.nnz), *du = dc + n, *dx = du + n, *db = dx + n, *dy = db + m;
    double *dd = w + rg::work_doubles(m, n, P.nnz), *cpt = dd + n, *rpt = cpt + P.Pc;
    const double *cp = P.cparams ? P.cparams + p * P.Pc : nullptr;
    const double *rp = P.rparams ? P.rparams + p * P.rstride : nullptr;
    // the parameters at theta (exactly the LP's own at 0), then the LP there with every nonbasic column at u on its moved bound
    auto move_to = [&](double th, bool with_a) {
        for (int q = tid; q < P.Pc; q += nt) cpt[q] = gc && th != 0.0 ? fma(th, gc[q], cp[q]) : cp[q];
        for (int q = tid; q < P.Pr; q += nt) rpt[q] = gr && th != 0.0 ? fma(th, gr[q], rp[q]) : rp[q];
        XO_SYNC();
        form(s, X, W, m, n, cpt, rpt, with_a, tid, nt);
    };
    move_to(0.0, true);
    double tolp, told;
    tolerances(W, S, m, n, &tolp, &told, tid, nt);
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
    if (S->ival[0]) { finish(0, NUMERICAL); return; }
    if (!xo::reinvert(W, s, S, m, n, tid, nt)) { finish(0, NUMERICAL); return; }
    xo::solve_x(W, X, m, n, true, tid, nt);
    xo::solve_y(W, s, m, n, true, tid, nt);
    if (infeasible(W, S, m, n, tolp, told, tid, nt)) { finish(0, NUMERICAL); return; }
    // the objective c'x + k at the current parameters (thread 0)
    auto objective = [&]() {
        double o = P.o0;
        for (int q = 0; q < P.Pr; ++q) o = fma(sens::ld<true>(s.omap + q), rpt[q], o);
        for (int q = 0; q < P.Pc; ++q) o = fma(sens::ld<true>(s.ocmap + q), cpt[q], o);
        double cx = 0.0;
        for (int j = 0; j < n; ++j) cx = fma(W.c[j], W.xv[j], cx);
        return cx + o;
    };
    auto record = [&](int e, double th, double d1, double d2, int en, int lv, int lt) {
        if (tid == 0) {
            P.theta[ev + e] = th; P.obj[ev + e] = objective(); P.dobj[ev + e] = d1;
            if (P.d2obj) P.d2obj[ev + e] = d2;
            if (P.enter) P.enter[ev + e] = en;
            if (P.leave) P.leave[ev + e] = lv;
            if (P.leave_to) P.leave_to[ev + e] = (signed char)lt;
        }
    };
    double th = 0.0;
    int cnt = 0, status = OPTIMAL, en = -1, lv = -1, lt = -1, since = 0, degen = 0;
    for (;;) {
        // ---- 2. the segment from th
        const rg::Segment g = rg::segment(s, X, W, S, m, n, P.Pc, P.Pr, gc, gr, dc, du, dx, db, dy, dd, tolp, told, tid, nt);
        record(cnt++, th, g.d1, g.d2, en, lv, lt);
        XO_SYNC();
        const double tn = th + g.hi;
        if (g.block == xo::kNone || !(tn < te)) break;
        if (cnt == NS) { status = MAX_ITER; break; }
        // ---- 3. the event at tn
        degen = tn == th ? degen + 1 : 0;
        const bool low_index = degen >= xo::kBlandAfter;
        const int v = g.block / 8, kind = g.block % 8;
        const double rate_art = kind == rg::BK_ARTIFICIAL ? W.al[position(W, S, m, v, tid, nt)] : 0.0;   // dx_B of the artificial
        th = tn;
        move_to(th, false);
        tolerances(W, S, m, n, &tolp, &told, tid, nt);
        for (int j = tid; j < n; j += nt) if (W.stat[j] == xo::AT_UP) W.xv[j] = W.u[j];
        XO_SYNC();
        xo::solve_x(W, X, m, n, true, tid, nt);
        xo::solve_y(W, s, m, n, true, tid, nt);
        en = -1; lv = v; lt = -1;
        bool pivoted = false;
        if (kind == rg::BK_BOUND) {                      // an upper bound at u reaches 0: no feasible point past th
            status = INFEASIBLE;
        } else if (kind == rg::BK_UNFIX) {               // to the bound the reduced cost asks for, x unchanged (u = 0)
            const bool up = W.d[v] < 0.0;
            if (tid == 0) { W.stat[v] = up ? xo::AT_UP : xo::AT_LO; W.xv[v] = up ? W.u[v] : 0.0; }
            lt = up ? 2 : 0;
            XO_SYNC();
        } else if (kind == rg::BK_DUAL) {                // primal simplex: v enters
            const int q = v, dir = W.stat[q] == xo::AT_LO ? 1 : -1;
            xo::ftran(W, s, m, n, q, W.al, tid, nt);
            double b1 = INFINITY, b2 = 0.0; int bi = xo::kNone;
            for (int r = tid; r < m; r += nt) xo::keep_best(b1, b2, bi, -fabs(W.al[r]), 0.0, r);
            xo::choose(S, tid, nt, b1, b2, bi);
            const double tol_piv = xo::kPivot * -S->r1;
            // the ratio of position r, and its rate in theta: the step of x_q at which x_B(r) reaches the bound it moves towards
            auto ratio = [&](int r, double *rt, double *rate, double *a) {
                const double sg = dir * W.al[r];
                *a = fabs(sg);
                if (*a < tol_piv || sg == 0.0) return false;
                const int u = W.head[r];
                const double x = W.xv[u], up = xo::upper(W, n, u), dxu = u < n ? dx[u] : 0.0;
                double gap, dgap;
                if (sg > 0.0) { gap = x; dgap = dxu; }
                else if (up < INFINITY) { gap = up - x; dgap = u < n ? du[u] - dxu : 0.0; }
                else return false;
                *rt = u < n ? fmax(gap, 0.0) / *a : 0.0;          // a basic artificial is at 0 (its x_B is rounding)
                *rate = dgap / *a;
                return true;
            };
            b1 = INFINITY; b2 = 0.0; bi = xo::kNone;
            for (int r = tid; r < m; r += nt) {
                double rt, rate, a;
                if (ratio(r, &rt, &rate, &a)) xo::keep_best(b1, b2, bi, rt, rate, W.head[r]);
            }
            xo::choose(S, tid, nt, b1, b2, bi);
            const double r1 = S->r1, r2 = S->r2;
            const bool blocks = S->rid != xo::kNone;
            b1 = INFINITY; b2 = 0.0; bi = xo::kNone;
            if (blocks)
                for (int r = tid; r < m; r += nt) {
                    double rt, rate, a;
                    if (ratio(r, &rt, &rate, &a) && rt == r1 && rate == r2) xo::keep_best(b1, b2, bi, low_index ? 0.0 : -a, 0.0, W.head[r]);
                }
            xo::choose(S, tid, nt, b1, b2, bi);
            const int lvar = S->rid;
            const double uq = W.u[q], rq = uq;
            if (!blocks && uq == INFINITY) {
                status = UNBOUNDED;
            } else if (!blocks || rq < r1 || (rq == r1 && du[q] <= r2)) {     // the column reaches its other bound first: a flip
                if (tid == 0) { W.stat[q] = dir > 0 ? xo::AT_UP : xo::AT_LO; W.xv[q] = dir > 0 ? uq : 0.0; }
                lt = dir > 0 ? 2 : 0;
                XO_SYNC();
            } else {
                const int r = position(W, S, m, lvar, tid, nt);
                const bool to_up = dir * W.al[r] < 0.0;
                xo::pivot(W, m, n, r, q, to_up ? xo::AT_UP : xo::AT_LO, to_up ? xo::upper(W, n, lvar) : 0.0, tid, nt);
                en = q; lv = lvar; lt = to_up && lvar < n ? 2 : 0;       // an artificial leaves to 0
                pivoted = true;
            }
        } else {                                         // dual simplex: basic v leaves to the bound it reached
            const int r = position(W, S, m, v, tid, nt);
            const bool below = kind == rg::BK_BASIC_LO || (kind == rg::BK_ARTIFICIAL && rate_art < 0.0);
            const int dir = below ? -1 : 1;
            row_alpha(W, s, S, m, n, r, du, tid, nt);
            auto ratio = [&](int j, double *rt, double *rate, double *a) {
                const double al = W.alr[j];
                if (al == 0.0) return false;
                const bool lo = W.stat[j] == xo::AT_LO;
                if (!((lo && al * dir > 0.0) || (!lo && al * dir < 0.0))) return false;
                *a = fabs(al);
                const double sl = xo::dual_slack(W, j);
                *rt = sl / *a;
                *rate = (lo ? dd[j] : -dd[j]) / *a;
                return true;
            };
            double b1 = INFINITY, b2 = 0.0; int bi = xo::kNone;
            for (int j = tid; j < n; j += nt) {
                double rt, rate, a;
                if (ratio(j, &rt, &rate, &a)) xo::keep_best(b1, b2, bi, rt, rate, j);
            }
            xo::choose(S, tid, nt, b1, b2, bi);
            const double r1 = S->r1, r2 = S->r2;
            if (S->rid == xo::kNone) {
                status = INFEASIBLE;
            } else {
                b1 = INFINITY; b2 = 0.0; bi = xo::kNone;
                for (int j = tid; j < n; j += nt) {
                    double rt, rate, a;
                    if (ratio(j, &rt, &rate, &a) && rt == r1 && rate == r2) xo::keep_best(b1, b2, bi, low_index ? 0.0 : -a, 0.0, j);
                }
                xo::choose(S, tid, nt, b1, b2, bi);
                const int e = S->rid;
                xo::ftran(W, s, m, n, e, W.al, tid, nt);
                xo::pivot(W, m, n, r, e, below ? xo::AT_LO : xo::AT_UP, below ? 0.0 : xo::upper(W, n, v), tid, nt);
                en = e; lt = below || v >= n ? 0 : 2;            // an artificial's only bound is 0
                pivoted = true;
            }
        }
        if (status != OPTIMAL) {                         // the curve stops at th
            record(cnt++, th, nan, nan, -1, -1, -1);
            XO_SYNC();
            break;
        }
        if (pivoted && ++since >= xo::kRefactor) {
            since = 0;
            if (!xo::reinvert(W, s, S, m, n, tid, nt)) { status = NUMERICAL; break; }
        }
        xo::solve_x(W, X, m, n, true, tid, nt);
        xo::solve_y(W, s, m, n, true, tid, nt);
        if (infeasible(W, S, m, n, tolp, told, tid, nt) == 2) { status = NUMERICAL; break; }
    }
    finish(cnt, status);
}

}  // namespace pm
