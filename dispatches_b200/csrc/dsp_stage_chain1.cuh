// dsp_stage_chain1.cuh -- DESCRIPTOR-DRIVEN stage kernel for the "single storage chain" family of dispatch LPs:
//
//     one equality row per period t;  every column appears either in ONE row (a "flow" of period t: power to the electrolyser,
//     hydrogen to the pipeline / turbine, a slack ...) or in TWO CONSECUTIVE rows (the "state" of period t: tank holdup at the end
//     of t, which re-enters the balance of t+1).                     A D A' is then TRIDIAGONAL (1x1 blocks, K = 1).
//
// Members in this repo: the nuclear + PEM + hydrogen-tank dispatch LP of BASELINE config C3
// (nuclear_flowsheet_multiperiod_class.py:72-155, hydrogen_tank_simplified.py:177-184 -> templates.nuclear) and the report's LP with
// tank / turbine (price_taker_analysis.py:116-222 -> templates.nuclear_report) for T <= 96.  Nothing flowsheet-specific is
// compiled in: the host (lp_template.detect_chain1) recognises the structure of ANY LPTemplate and emits, per period, the template
// column of each of its <= NF flows and of its state, their row coefficients (as equilibrated by the template) and the row index;
// costs / right-hand sides / bounds come from the template's ordinary parameter maps.  Same algorithm, scaling and stopping rules as
// the generic band kernel (dsp_lp.cu; numpy mirror oracle/ipm_numpy.py) -- the iterates agree to rounding -- but laid out like the
// generation-2 wind+battery kernel (dsp_stage2.cuh): an LP occupies a group of L lanes, P periods per lane, iterate in registers,
// cross-pass temporaries in shared memory, partitioned elimination of the tridiagonal system (local P-1 pivots per lane + a
// twisted chain over the L separators), groups refill from the ticket counter independently, CTA-synchronised rounds.
#pragma once
#include "dsp_stage2.cuh"

namespace chain1 {
using namespace stage2;

struct Params {
    // batch
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    int Pc, Pr;
    const double *omap, *ocmap;
    double o0;
    double tol, feas_tol, step_frac, reg;
    int max_iter;
    double *obj, *x_out, *y_out;
    int *status, *iters;
    int n, m, nb;
    unsigned long long *ticket;
    // template parameter maps (device): c = c0 + Cmap cp, b = b0 + Bmap rp, u = u0 + Umap rp (first nb columns are the bounded ones)
    const double *c0, *b0, *u0;
    const int *cm_ptr, *cm_idx, *bm_ptr, *bm_idx, *um_ptr, *um_idx;
    const double *cm_val, *bm_val, *um_val;
    // chain descriptor (device): T periods, NC = NF + 1 column slots per period (flows 0..NF-1, state NF)
    int T;
    const int *col_idx;          // [T * NC] template column of (t, slot) or -1
    const int *row_idx;          // [T]
    const double *coef;          // [T * NC] row-t coefficient of (t, slot)
    const double *coef_next;     // [T] coefficient of the state of period t in row t+1 (0 for the last period)
    const int *x_perm, *y_perm;  // non-null: x_out / y_out index of template column / row (templates created from plain CSR)
};

template <int NF, int P>
struct Smem {
    static constexpr int NC = NF + 1;
    // [array][period slot][lane]
    static constexpr int A_D = 0;                 // NC scaling values d; after the corrector's recovery: dx
    static constexpr int A_RX = NC;               // NC reciprocals 1/x
    static constexpr int A_PR = 2 * NC;           // 2 NC second-order products (dx dz, ds dw)
    static constexpr int A_F = 4 * NC;            // forward-eliminated right-hand side / dy
    static constexpr int A_C = 4 * NC + 1;        // NC scaled costs
    static constexpr int A_U = 5 * NC + 1;        // NC scaled upper bounds (only read where the column is bounded)
    static constexpr int A_B = 6 * NC + 1;        // scaled right-hand side
    static constexpr int A_A = 6 * NC + 2;        // NC row coefficients (LP independent: loaded once per warp)
    static constexpr int A_HN = 7 * NC + 2;       // coefficient of the state in the next row
    static constexpr int NA_FULL = 7 * NC + 3;
    static constexpr int I_K = 0, I_G = 1, I_H = 2, NA_INT = 3;
    static constexpr int doubles_per_warp = (NA_FULL * P + NA_INT * (P > 1 ? P - 1 : 0)) * 32;
};

template <int NF>
struct Per {
    double x[NF + 1], z[NF + 1], s[NF + 1], w[NF + 1];
    double y;
};

// The trailing flag is ignored: the exit vote is always the CTA barrier on the device and the warp vote in the emulator
// (stage2::cta_all).  tests/emu/emu_chain1.cpp still passes it, so it stays in the signature.
template <int L, int P, int NF, bool = true>
__device__ void warp_body(const Params &Q, double *smw, int lane) {
    using SM = Smem<NF, P>;
    constexpr int NC = NF + 1;
#define SMF(arr, j) sm[((arr) * P + (j)) * 32]
#define SMI(arr, j) smi[((arr) * (P - 1) + (j)) * 32]
    const int gl = lane & (L - 1);
    double *sm = smw + lane;
    double *smi = smw + SM::NA_FULL * P * 32 + lane;
    const int T = Q.T;
    constexpr int r_root = L / 2;
    constexpr int kmax = (r_root - 1 > L - 2 - r_root) ? r_root - 1 : L - 2 - r_root;
    constexpr int smax = (r_root > L - 1 - r_root) ? r_root : L - 1 - r_root;

    // ---- LP-independent structure of this lane's periods: presence / boundedness flags, row coefficients
    int present[P], bounded[P];                  // bit c: slot c of period j exists / has an upper bound
    int ncols = 0, nbnd = 0;
#pragma unroll
    for (int j = 0; j < P; ++j) {
        const int t = gl * P + j;
        present[j] = 0; bounded[j] = 0;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int col = t < T ? Q.col_idx[t * NC + c] : -1;
            if (col >= 0) { present[j] |= 1 << c; ++ncols; if (col < Q.nb) { bounded[j] |= 1 << c; ++nbnd; } }
            SMF(SM::A_A + c, j) = col >= 0 ? Q.coef[t * NC + c] : 0.0;
        }
        SMF(SM::A_HN, j) = (t < T && (present[j] >> NF & 1)) ? Q.coef_next[t] : 0.0;
    }
    const double ntot_t = gsum<L>((double)(ncols + nbnd));       // template constant: n + nb

    Per<NF> pr[P];
#pragma unroll
    for (int j = 0; j < P; ++j) {
#pragma unroll
        for (int c = 0; c < NC; ++c) pr[j].x[c] = pr[j].z[c] = pr[j].s[c] = pr[j].w[c] = 0.0;
        pr[j].y = 0.0;
    }
    double nrm_b = 1.0, nrm_c = 1.0, beta_b = 1.0, beta_c = 1.0, kconst = 0.0;
    double step_frac = Q.step_frac, reg = Q.reg;
    long long p = -1;
    int it = 0, it0 = 0, attempt = 0, Tg = 0;
    int mode = 1;                     // 0 running, 1 needs a new LP, 2 retries its LP with safer parameters, 3 out of work
#define HAS(j, c) ((present[j] >> (c)) & 1)
#define BND(j, c) ((bounded[j] >> (c)) & 1)
#define ACT(j) (gl * P + (j) < Tg)

    double mu_keep = 0.0;             // complementarity measure of the group's current iterate (set by the check / the refill)
    const double ntot = ntot_t;
    double hx_left = 0.0;             // hn * x_state of the left neighbour's last period
    double y_right = 0.0;             // dual of the right neighbour's first period
    // state of the previous period enters this period's row; the next period's dual enters this period's state column
#define NEIGHBOURS()                                                                                   \
    {                                                                                                  \
        const double v_ = HAS(P - 1, NF) ? SMF(SM::A_HN, P - 1) * pr[P - 1].x[NF] : 0.0;               \
        hx_left = gup1<L>(v_, gl);                                                                     \
        y_right = gdown1<L>(pr[0].y, gl);                                                              \
    }
#define YN(j) ((j) == P - 1 ? y_right : pr[(j) < P - 1 ? (j) + 1 : 0].y)
    // residuals of one period (registers); hxp = hn * x_state of period t-1
#define RESID(j, hxp)                                                                                  \
        double rp_ = 0.0, rd_[NC], ru_[NC];                                                            \
        {                                                                                              \
            double ax = (hxp);                                                                         \
            _Pragma("unroll")                                                                          \
            for (int c = 0; c < NC; ++c) {                                                             \
                const double a_ = SMF(SM::A_A + c, j);                                                 \
                ax = fma(a_, q.x[c], ax);                                                              \
                double r_ = SMF(SM::A_C + c, j) - a_ * q.y - q.z[c];                                   \
                if (c == NF) r_ -= SMF(SM::A_HN, j) * YN(j);                                           \
                ru_[c] = 0.0;                                                                          \
                if (BND(j, c)) { r_ += q.w[c]; ru_[c] = SMF(SM::A_U + c, j) - q.x[c] - q.s[c]; }       \
                rd_[c] = HAS(j, c) ? r_ : 0.0;                                                         \
            }                                                                                          \
            rp_ = SMF(SM::A_B, j) - ax;                                                                \
        }

    for (;;) {
        // =========================================================================================== convergence check
        // before the refill (as in dsp_stage2.cuh): a group whose LP has just converged starts its next LP in this very round
        if (__any_sync(FULL, mode == 0)) {
            NEIGHBOURS();
            double pm = 0.0, dm = 0.0, mus = 0.0, po = 0.0, dob = 0.0;
            double hxc = hx_left;
#pragma unroll
            for (int j = 0; j < P; ++j) {
                const Per<NF> &q = pr[j];
                if (ACT(j)) {
                    RESID(j, hxc);
                    pm = dmax(pm, fabs(rp_));
                    dob += SMF(SM::A_B, j) * q.y;
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        if (HAS(j, c)) {
                            dm = dmax(dm, fabs(rd_[c]));
                            mus += q.x[c] * q.z[c];
                            po += SMF(SM::A_C + c, j) * q.x[c];
                            if (BND(j, c)) {
                                pm = dmax(pm, fabs(ru_[c]));
                                mus += q.s[c] * q.w[c];
                                dob -= SMF(SM::A_U + c, j) * q.w[c];
                            }
                        }
                    }
                    hxc = SMF(SM::A_HN, j) * q.x[NF];
                } else {
                    hxc = 0.0;
                }
            }
            const double res = gmax<L>(dmax(pm / nrm_b, dm / nrm_c));
            mus = gsum<L>(mus); po = gsum<L>(po); dob = gsum<L>(dob);
            const double mu = mus / ntot;
            const double den = dmax(kGapFloor2, fabs(po));
            const double gap = fabs(po - dob) / den, cgap = ntot * mu / den;
            if (mode == 0) {
                mu_keep = mu;
                int status = -1;
                if (!(mu == mu) || !(po == po) || mu > 1e100) status = DSP_NUMERICAL;
                else if (res < Q.feas_tol && gap < Q.tol) status = DSP_OPTIMAL;
                else if (cgap < Q.tol && res < 10.0 * Q.feas_tol && gap < 10.0 * Q.tol) status = DSP_OPTIMAL;
                else if (cgap < 1e-3 * Q.tol) status = (res < 100.0 * Q.feas_tol && gap < 1000.0 * Q.tol) ? DSP_OPTIMAL : DSP_NUMERICAL;
                else if (it == Q.max_iter) status = DSP_MAX_ITER;
                if (status >= 0) {
                    if (gl == 0) { Q.obj[p] = po * beta_b * beta_c + kconst; Q.status[p] = status; Q.iters[p] = it + it0; }
                    if (Q.x_out) {
                        double *xo_ = Q.x_out + p * (long long)Q.n;
#pragma unroll
                        for (int j = 0; j < P; ++j) {
                            const int t = gl * P + j;
                            if (t < T) {
#pragma unroll
                                for (int c = 0; c < NC; ++c)
                                    if (HAS(j, c)) {
                                        const int col = Q.col_idx[t * NC + c];
                                        xo_[Q.x_perm ? Q.x_perm[col] : col] = pr[j].x[c] * beta_b;
                                    }
                            }
                        }
                    }
                    if (Q.y_out) {
                        double *yo_ = Q.y_out + p * (long long)Q.m;
#pragma unroll
                        for (int j = 0; j < P; ++j) {
                            const int t = gl * P + j;
                            if (t < T) { const int row = Q.row_idx[t]; yo_[Q.y_perm ? Q.y_perm[row] : row] = pr[j].y * beta_c; }
                        }
                    }
                    if (status != DSP_OPTIMAL && attempt == 0) { mode = 2; attempt = 1; it0 = it + it0; }
                    else mode = 1;
                }
            }
        }
        // =========================================================================================== (re)fill groups
        if (__any_sync(FULL, mode == 1 || mode == 2)) {
            unsigned long long tk = 0;
            if (mode == 1 && gl == 0) tk = atomicAdd(Q.ticket, 1ULL);
            tk = __shfl_sync(FULL, tk, 0, L);
            if (mode == 1) {
                if ((long long)tk >= Q.N) { mode = 3; p = -1; Tg = 0; }
                else { p = (long long)tk; attempt = 0; it0 = 0; }
            }
            const bool ld = (mode == 1 || mode == 2);
            double kc = 0.0, bm = 0.0, cm = 0.0;
            bool bad_u = false;
            if (ld) {
                const double *cp = Q.cparams + p * (long long)Q.Pc;
                const double *rp = Q.rparams + p * Q.rstride;
                for (int r = gl; r < Q.Pr; r += L) kc += Q.omap[r] * rp[r];
                for (int r = gl; r < Q.Pc; r += L) kc += Q.ocmap[r] * cp[r];
#pragma unroll
                for (int j = 0; j < P; ++j) {
                    const int t = gl * P + j;
                    if (t < T) {
                        const int row = Q.row_idx[t];
                        double bj = Q.b0[row];
                        for (int q = Q.bm_ptr[row]; q < Q.bm_ptr[row + 1]; ++q) bj += Q.bm_val[q] * rp[Q.bm_idx[q]];
                        SMF(SM::A_B, j) = bj;
                        bm = dmax(bm, fabs(bj));
#pragma unroll
                        for (int c = 0; c < NC; ++c) {
                            double cj = 0.0, uj = 0.0;
                            if (HAS(j, c)) {
                                const int col = Q.col_idx[t * NC + c];
                                cj = Q.c0[col];
                                for (int q = Q.cm_ptr[col]; q < Q.cm_ptr[col + 1]; ++q) cj += Q.cm_val[q] * cp[Q.cm_idx[q]];
                                if (BND(j, c)) {
                                    uj = Q.u0[col];
                                    for (int q = Q.um_ptr[col]; q < Q.um_ptr[col + 1]; ++q) uj += Q.um_val[q] * rp[Q.um_idx[q]];
                                    bm = dmax(bm, uj);
                                    bad_u |= uj < 0.0;
                                }
                            }
                            SMF(SM::A_C + c, j) = cj; SMF(SM::A_U + c, j) = uj;
                            cm = dmax(cm, fabs(cj));
                        }
                    } else {
                        SMF(SM::A_B, j) = 0.0;
#pragma unroll
                        for (int c = 0; c < NC; ++c) { SMF(SM::A_C + c, j) = 0.0; SMF(SM::A_U + c, j) = 0.0; }
                    }
                }
            }
            kc = gsum<L>(kc);
            bm = gmax<L>(bm);
            cm = gmax<L>(cm);
            const double ubad = gmax<L>(bad_u ? 1.0 : 0.0);
            double infl = 0.0;
            if (ld) {
                kconst = kc + Q.o0;
                beta_b = bm > 0.0 ? bm : 1.0;
                beta_c = cm > 0.0 ? cm : 1.0;
                // a negative upper bound beyond rounding: infeasible (same rule as the band kernel)
                if (ubad > 0.0) {
#pragma unroll
                    for (int j = 0; j < P; ++j)
#pragma unroll
                        for (int c = 0; c < NC; ++c)
                            if (BND(j, c) && (gl * P + j) < T && SMF(SM::A_U + c, j) < -1e-9 * beta_b) infl = 1.0;
                }
            }
            infl = gmax<L>(infl);               // (collectives stay outside the divergent branches)
            double mu0 = 0.0;
            if (ld) {
                if (infl > 0.0) {
                    if (gl == 0) { Q.obj[p] = __longlong_as_double(0x7ff8000000000000LL); Q.status[p] = DSP_INFEASIBLE; Q.iters[p] = it0; }
                    dsp_nan_rows(Q.x_out, Q.n, Q.y_out, Q.m, p, gl, L);
                    mode = 1; Tg = 0;
#pragma unroll
                    for (int j = 0; j < P; ++j) {           // (an all-inactive group must not carry the finished LP's iterate)
#pragma unroll
                        for (int c = 0; c < NC; ++c) pr[j].x[c] = pr[j].z[c] = pr[j].s[c] = pr[j].w[c] = 0.0;
                        pr[j].y = 0.0;
                    }
                } else {
                    step_frac = attempt ? 0.99 : Q.step_frac;
                    reg = attempt ? 10.0 * Q.reg : Q.reg;
                    double bsmax = 0.0;
#pragma unroll
                    for (int j = 0; j < P; ++j) {
                        const bool act = (gl * P + j) < T;
                        const double bj = SMF(SM::A_B, j) / beta_b;
                        SMF(SM::A_B, j) = bj;
                        bsmax = dmax(bsmax, fabs(bj));
                        pr[j].y = 0.0;
#pragma unroll
                        for (int c = 0; c < NC; ++c) {
                            SMF(SM::A_C + c, j) = SMF(SM::A_C + c, j) / beta_c;
                            double xj = (act && HAS(j, c)) ? 1.0 : 0.0, sj = 0.0, wj = 0.0;
                            if (act && BND(j, c)) {
                                const double uj = dmax(SMF(SM::A_U + c, j) / beta_b, 1e-10);
                                SMF(SM::A_U + c, j) = uj;
                                xj = fmin(1.0, 0.5 * uj);
                                sj = uj - xj; wj = 1.0;
                            }
                            pr[j].x[c] = xj; pr[j].z[c] = (act && HAS(j, c)) ? 1.0 : 0.0; pr[j].s[c] = sj; pr[j].w[c] = wj;
                            if (act && HAS(j, c)) { mu0 += pr[j].x[c] * pr[j].z[c]; if (BND(j, c)) mu0 += sj * wj; }
                        }
                    }
                    nrm_b = 1.0 + bsmax;            // completed by the group maximum below
                    nrm_c = 1.0 + (cm > 0.0 ? 1.0 : 0.0);
                    Tg = T; it = 0; mode = 0;
                }
            }
            // (the group maximum of |b| for the residual norm; executed by every lane)
            nrm_b = 1.0 + gmax<L>(nrm_b - 1.0);
            mu0 = gsum<L>(mu0);
            if (ld) mu_keep = mu0 / ntot;      // (the start point is never optimal: its own convergence check is skipped)
        }
        if (cta_all(mode == 3)) break;
        if (__all_sync(FULL, mode == 3)) continue;     // out of work: leave the issue slots to the warps that still iterate

        // =========================================================================================== neighbours of the lane's block
        NEIGHBOURS();

        // =========================================================================================== pass 1
        double Dd[P], f1[P], Cn[P];        // diagonal, right-hand side, coupling with the next period
        double dl_left, ql_left;           // hn^2 d and hn d h of the left neighbour's last period
        {
            double hxc = hx_left, ddc = 0.0, qqc = 0.0;       // carried from period j-1 (ddc / qqc of the left lane are added after the loop)
#pragma unroll
            for (int j = 0; j < P; ++j) {
                const Per<NF> &q = pr[j];
                if (ACT(j)) {
                    RESID(j, hxc);
                    double diag = ddc, rhs = rp_ + qqc;
                    double dh = 0.0, hh = 0.0;
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        double dc = 0.0, rx = 0.0, hc = 0.0;
                        if (HAS(j, c)) {
                            rx = frcp(q.x[c]);
                            double tt = q.z[c] * rx + (q.x[c] > 1.0 ? reg * rx * rx : reg);
                            hc = rd_[c] + q.z[c];
                            if (BND(j, c)) {
                                const double rs = frcp(q.s[c]);
                                tt += q.w[c] * rs;
                                hc += (-q.w[c] * ru_[c]) * rs - q.w[c];
                            }
                            dc = frcp(tt);
                            const double a_ = SMF(SM::A_A + c, j);
                            diag = fma(a_ * a_, dc, diag);
                            rhs = fma(a_ * dc, hc, rhs);
                        }
                        SMF(SM::A_D + c, j) = dc; SMF(SM::A_RX + c, j) = rx;
                        if (c == NF) { dh = dc; hh = hc; }
                    }
                    const double hn = SMF(SM::A_HN, j), hs = SMF(SM::A_A + NF, j);
                    Dd[j] = diag; f1[j] = rhs;
                    Cn[j] = hs * hn * dh;
                    hxc = hn * q.x[NF]; ddc = hn * hn * dh; qqc = hn * dh * hh;
                } else {
                    Dd[j] = 1.0; f1[j] = 0.0; Cn[j] = 0.0; hxc = 0.0; ddc = 0.0; qqc = 0.0;
#pragma unroll
                    for (int c = 0; c < NC; ++c) { SMF(SM::A_D + c, j) = 0.0; SMF(SM::A_RX + c, j) = 0.0; }
                }
            }
            dl_left = gup1<L>(ddc, gl); ql_left = gup1<L>(qqc, gl);
            if (ACT(0)) { Dd[0] += dl_left; f1[0] += ql_left; }
        }
        const double mu = mu_keep;

        // =========================================================================================== factorisation + predictor solve
        double Wc, Asep, g1, Ainv, Mout = 0.0, Mout2 = 0.0, Cin;
        int fo, bo, fsrc, bsrc;
        const bool is_root = (gl == r_root);
        {
            // coupling of this lane's first period with the left separator: hs_0 * hn_left * d_left  (= Cn of the left lane's last period)
            const double c_left = gup1<L>(Cn[P - 1], gl);
            double E = ACT(0) ? c_left : 0.0;
            double dS = 0.0, dg1 = 0.0;
#pragma unroll
            for (int j = 0; j < P - 1; ++j) {
                const double Kj = frcp(Dd[j]);
                const double C = Cn[j];
                const double G = C * Kj;
                Dd[j + 1] -= G * C;
                const double Hm = E * Kj;
                dS -= Hm * E;
                dg1 -= Hm * f1[j];
                f1[j + 1] -= G * f1[j];
                SMI(SM::I_K, j) = Kj; SMI(SM::I_G, j) = G; SMI(SM::I_H, j) = Hm;
                SMF(SM::A_F, j) = f1[j];
                E = -G * E;
            }
            Wc = E;
            Asep = Dd[P - 1] + gdown1<L>(dS, gl);
            g1 = f1[P - 1] + gdown1<L>(dg1, gl);
            const double Wn = gdown1<L>(Wc, gl);
            const bool low = gl < r_root;
            fsrc = low ? (gl > 0 ? gl - 1 : 0) : (gl < L - 1 ? gl + 1 : L - 1);
            bsrc = low ? gl + 1 : gl - 1;
            fo = is_root ? (1 << 20) : (low ? gl : L - 1 - gl);
            bo = is_root ? (1 << 20) : (low ? r_root - gl : gl - r_root);
            const double Cout = low ? Wc : Wn;
            Cin = low ? Wn : Wc;
#pragma unroll
            for (int k = 1; k <= kmax; ++k) {
                const double R = gfrom<L>(Asep, fsrc), q1 = gfrom<L>(g1, fsrc);
                if (fo == k) {
                    const double X = Cout * frcp(R);
                    Asep -= X * Cout; g1 -= X * q1; Mout = X;
                }
            }
            {
                constexpr int la = r_root > 0 ? r_root - 1 : 0, lb = r_root + 1 < L ? r_root + 1 : L - 1;
                const double Ra = gfrom<L>(Asep, la), Rb = gfrom<L>(Asep, lb), a1 = gfrom<L>(g1, la), b1 = gfrom<L>(g1, lb);
                if (is_root) {
                    if (r_root >= 1) { Mout = Wc * frcp(Ra); Asep -= Mout * Wc; g1 -= Mout * a1; }
                    if (r_root + 1 <= L - 1) { Mout2 = Wn * frcp(Rb); Asep -= Mout2 * Wn; g1 -= Mout2 * b1; }
                }
            }
            Ainv = frcp(Asep);
        }
#define SEP_BACK()                                                                     \
        {                                                                              \
            double u1 = is_root ? Ainv * g1 : 0.0;                                     \
            _Pragma("unroll")                                                          \
            for (int s = 1; s <= smax; ++s) {                                          \
                const double r1 = gfrom<L>(u1, bsrc);                                  \
                if (bo == s) u1 = Ainv * (g1 - Cin * r1);                              \
            }                                                                          \
            g1 = u1;                                                                   \
        }
#define LOCAL_BACK(dy)                                                                 \
        {                                                                              \
            const double ul = gup1<L>(g1, gl);                                         \
            dy[P - 1] = g1;                                                            \
            _Pragma("unroll")                                                          \
            for (int j = P - 2; j >= 0; --j)                                           \
                dy[j] = SMI(SM::I_K, j) * SMF(SM::A_F, j) - SMI(SM::I_G, j) * dy[j + 1] - SMI(SM::I_H, j) * ul; \
        }
        double dy[P];
        SEP_BACK();
        LOCAL_BACK(dy);

        // =========================================================================================== pass 2: predictor direction
        double smu;
        {
            const double dy_right = gdown1<L>(dy[0], gl);
            double ip = 0.0, id = 0.0, S1 = 0.0, S3 = 0.0;
            double hxc = hx_left;
#pragma unroll
            for (int j = 0; j < P; ++j) {
                const Per<NF> &q = pr[j];
                if (ACT(j)) {
                    RESID(j, hxc);
                    (void)rp_;
                    const double dyn = (j == P - 1) ? dy_right : dy[j < P - 1 ? j + 1 : 0];
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        double pxz = 0.0, psw = 0.0;
                        if (HAS(j, c)) {
                            const double rx = SMF(SM::A_RX + c, j), dc = SMF(SM::A_D + c, j);
                            double hc = rd_[c] + q.z[c];
                            double rs = 0.0;
                            if (BND(j, c)) { rs = frcp(q.s[c]); hc += (-q.w[c] * ru_[c]) * rs - q.w[c]; }
                            double aty = SMF(SM::A_A + c, j) * dy[j];
                            if (c == NF) aty = fma(SMF(SM::A_HN, j), dyn, aty);
                            const double dx = dc * (aty - hc);
                            const double tx = dx * rx;
                            const double dz = -q.z[c] - q.z[c] * tx;
                            ip = dmax(ip, -tx); id = dmax(id, 1.0 + tx);
                            S1 += q.z[c] * dx;
                            pxz = dx * dz;
                            if (BND(j, c)) {
                                const double ds = ru_[c] - dx;
                                const double ts = ds * rs;
                                const double dw = -q.w[c] - q.w[c] * ts;
                                ip = dmax(ip, -ts); id = dmax(id, 1.0 + ts);
                                S1 += q.w[c] * ds;
                                psw = ds * dw;
                            }
                            S3 += pxz + psw;
                        }
                        SMF(SM::A_PR + c, j) = pxz; SMF(SM::A_PR + NC + c, j) = psw;
                    }
                    hxc = SMF(SM::A_HN, j) * q.x[NF];
                }
            }
            ip = gmax<L>(ip); id = gmax<L>(id);
            S1 = gsum<L>(S1); S3 = gsum<L>(S3);
            const double ap = ip > 1.0 ? 1.0 / ip : 1.0, ad = id > 1.0 ? 1.0 / id : 1.0;
            const double musum = mu * ntot;
            const double S2 = -musum - S1;
            const double mua = (musum + ap * S1 + ad * S2 + ap * ad * S3) / ntot;
            const double sg = mua / mu;
            smu = sg * sg * sg * mu;
        }

        // =========================================================================================== pass 3: corrector right-hand side + solve
        {
            double hxc = hx_left, qqc = 0.0;
#pragma unroll
            for (int j = 0; j < P; ++j) {
                const Per<NF> &q = pr[j];
                if (ACT(j)) {
                    RESID(j, hxc);
                    double rhs = rp_ + qqc;
                    double dh = 0.0, hh = 0.0;
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        if (HAS(j, c)) {
                            const double rx = SMF(SM::A_RX + c, j), dc = SMF(SM::A_D + c, j);
                            double hc = rd_[c] + q.z[c] - (smu - SMF(SM::A_PR + c, j)) * rx;
                            if (BND(j, c)) {
                                const double rs = frcp(q.s[c]);
                                hc += (-q.w[c] * ru_[c] + smu - SMF(SM::A_PR + NC + c, j)) * rs - q.w[c];
                            }
                            rhs = fma(SMF(SM::A_A + c, j) * dc, hc, rhs);
                            if (c == NF) { dh = dc; hh = hc; }
                        }
                    }
                    f1[j] = rhs;
                    const double hn = SMF(SM::A_HN, j);
                    hxc = hn * q.x[NF]; qqc = hn * dh * hh;
                } else {
                    f1[j] = 0.0; hxc = 0.0; qqc = 0.0;
                }
            }
            const double ql = gup1<L>(qqc, gl);
            if (ACT(0)) f1[0] += ql;
            double dg1 = 0.0;
#pragma unroll
            for (int j = 0; j < P - 1; ++j) {
                dg1 -= SMI(SM::I_H, j) * f1[j];
                f1[j + 1] -= SMI(SM::I_G, j) * f1[j];
                SMF(SM::A_F, j) = f1[j];
            }
            g1 = f1[P - 1] + gdown1<L>(dg1, gl);
#pragma unroll
            for (int k = 1; k <= kmax; ++k) {
                const double q1 = gfrom<L>(g1, fsrc);
                if (fo == k) g1 -= Mout * q1;
            }
            {
                constexpr int la = r_root > 0 ? r_root - 1 : 0, lb = r_root + 1 < L ? r_root + 1 : L - 1;
                const double a1 = gfrom<L>(g1, la), b1 = gfrom<L>(g1, lb);
                if (is_root) {
                    if (r_root >= 1) g1 -= Mout * a1;
                    if (r_root + 1 <= L - 1) g1 -= Mout2 * b1;
                }
            }
        }
        SEP_BACK();
        LOCAL_BACK(dy);

        // =========================================================================================== pass 4: corrector direction
        double ap, ad;
        {
            const double dy_right = gdown1<L>(dy[0], gl);
            double ip = 0.0, id = 0.0;
            double hxc = hx_left;
#pragma unroll
            for (int j = 0; j < P; ++j) {
                const Per<NF> &q = pr[j];
                if (ACT(j)) {
                    RESID(j, hxc);
                    (void)rp_;
                    const double dyn = (j == P - 1) ? dy_right : dy[j < P - 1 ? j + 1 : 0];
#pragma unroll
                    for (int c = 0; c < NC; ++c) {
                        double dx = 0.0;
                        if (HAS(j, c)) {
                            const double rx = SMF(SM::A_RX + c, j), dc = SMF(SM::A_D + c, j);
                            const double ax = smu - SMF(SM::A_PR + c, j);
                            double hc = rd_[c] + q.z[c] - ax * rx;
                            double rs = 0.0, as_ = 0.0;
                            if (BND(j, c)) {
                                rs = frcp(q.s[c]); as_ = smu - SMF(SM::A_PR + NC + c, j);
                                hc += (-q.w[c] * ru_[c] + as_) * rs - q.w[c];
                            }
                            double aty = SMF(SM::A_A + c, j) * dy[j];
                            if (c == NF) aty = fma(SMF(SM::A_HN, j), dyn, aty);
                            dx = dc * (aty - hc);
                            const double dz = ax * rx - q.z[c] - q.z[c] * dx * rx;
                            ip = dmax(ip, -dx * rx); id = dmax(id, -dz * frcp(q.z[c]));
                            if (BND(j, c)) {
                                const double ds = ru_[c] - dx;
                                const double dw = as_ * rs - q.w[c] - q.w[c] * ds * rs;
                                ip = dmax(ip, -ds * rs); id = dmax(id, -dw * frcp(q.w[c]));
                            }
                        }
                        SMF(SM::A_D + c, j) = dx;            // the scaling value of this column is dead now: park the direction
                    }
                    hxc = SMF(SM::A_HN, j) * q.x[NF];
                }
            }
            ip = gmax<L>(ip); id = gmax<L>(id);
            ap = step_frac < ip ? step_frac / ip : 1.0;
            ad = step_frac < id ? step_frac / id : 1.0;
        }

        // =========================================================================================== pass 5: step
#pragma unroll
        for (int j = 0; j < P; ++j) {
            Per<NF> &q = pr[j];
            if (ACT(j)) {
#pragma unroll
                for (int c = 0; c < NC; ++c) {
                    if (HAS(j, c)) {
                        const double rx = SMF(SM::A_RX + c, j), dx = SMF(SM::A_D + c, j);
                        const double dz = (smu - SMF(SM::A_PR + c, j)) * rx - q.z[c] - q.z[c] * dx * rx;
                        if (BND(j, c)) {
                            const double rs = frcp(q.s[c]);
                            const double ds = (SMF(SM::A_U + c, j) - q.x[c] - q.s[c]) - dx;
                            const double dw = (smu - SMF(SM::A_PR + NC + c, j)) * rs - q.w[c] - q.w[c] * ds * rs;
                            q.s[c] += ap * ds; q.w[c] += ad * dw;
                        }
                        q.x[c] += ap * dx; q.z[c] += ad * dz;
                    }
                }
                q.y += ad * dy[j];
            }
        }
        ++it;
    }
#undef SMF
#undef SMI
#undef HAS
#undef BND
#undef ACT
#undef YN
#undef NEIGHBOURS
#undef RESID
#undef SEP_BACK
#undef LOCAL_BACK
}

}  // namespace chain1
