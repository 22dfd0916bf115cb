// dsp_stage2_long.cuh -- the wind+battery stage algebra for LONG horizons (T > 96, up to the reference's full-year
// n_time_points = 8736 of run_pricetaker_wind_battery.py:57-58): ONE WARP PER LP, each lane owns a CONTIGUOUS chunk of
// P = ceil(T / 32) periods, and everything -- the iterate included -- lives in a per-warp region of a global workspace laid out
// [array][period slot j][lane] (every access of the warp is one coalesced 256-byte line; the working set of an LP is 65 arrays x T
// doubles = 4.5 MB at T = 8736, L2 resident).
//
// Why: on the generic band kernel this LP is a band of 35 k rows factorised by a 35 k-step sequential sweep with 4 lanes busy, three
// sweeps per IPM iteration through L2 (2.35 s per LP, round 1).  Here the per-period passes are 32-wide over P periods each, and the
// block-tridiagonal system is factorised by the PARTITIONED elimination of dsp_stage2.cuh: each lane eliminates its P-1 interior
// periods locally (all lanes busy, P sequential steps), the 32 separators form a chain eliminated from both ends with shuffles
// (16 steps).  Same algorithm, scaling, start point and stopping rules as the other two wind+battery kernels; period loops are rolled
// (the code is small), the per-period formulas are those of dsp_stage2.cuh.
// One numerical difference, measured: with explicitly inverted 2x2 pivot blocks (adjugate / determinant, fine for T <= 96 where
// the iteration counts are identical to the band kernel's) the iteration count grows with the chunk length -- 42 vs 29 at T = 2184,
// no convergence at T = 8736: block LDL' with inverted pivots is only conditionally stable and the blocks reach cond 1e12 here.
// The elimination below is therefore SCALAR (two pivots per period: u1, then u2 -- a Cholesky order, unconditionally backward
// stable); the stored multipliers replace K, G, H one for one.
#pragma once
#include "dsp_stage2.cuh"

namespace stage2long {
using namespace stage2;

// workspace arrays of a warp: [array][slot j][lane], P slots each
enum { W_X = 0,        // 7: xg xi xo xs xe xp xq
       W_Z = 7,        // 7
       W_S = 14,       // 2: si so
       W_W = 16,       // 2: wi wo
       W_Y = 18,       // 4: y1..y4
       W_C = 22, W_B4 = 23,
       W_SC = 24,      // 9 scaling values ds de dp kap dg di dq iot dO; after the corrector's recovery: dx (7), dy3, dy4
       W_RX = 33,      // 7
       W_PR = 40,      // 9
       W_D = 49,       // 3: diagonal block of the reduced system
       W_F = 52,       // 2: right-hand side / forward-eliminated right-hand side / solution dy
       W_K = 54,       // 3: pivots of the eliminated period (1/a, l = b/a, 1/(c - l b))
       W_G = 57,       // 4: scalar multipliers towards the next period (two per pivot)
       W_H = 61,       // 4: scalar multipliers towards the left separator
       NW = 65 };

struct LongParams {
    stage2::Params q;        // batch + stage structure (same fields as the short-horizon kernel)
    double *ws;              // [warps][NW][P][32]
    int P;                   // periods per lane
};

S2D void load_per(Per &q, const double *w, int P, int j) {
#define LW(a) w[((a) * P + j) * 32]
    q.xg = LW(W_X + 0); q.xi = LW(W_X + 1); q.xo = LW(W_X + 2); q.xs = LW(W_X + 3); q.xe = LW(W_X + 4); q.xp = LW(W_X + 5); q.xq = LW(W_X + 6);
    q.zg = LW(W_Z + 0); q.zi = LW(W_Z + 1); q.zo = LW(W_Z + 2); q.zs = LW(W_Z + 3); q.ze = LW(W_Z + 4); q.zp = LW(W_Z + 5); q.zq = LW(W_Z + 6);
    q.si = LW(W_S + 0); q.so = LW(W_S + 1); q.wi = LW(W_W + 0); q.wo = LW(W_W + 1);
    q.y1 = LW(W_Y + 0); q.y2 = LW(W_Y + 1); q.y3 = LW(W_Y + 2); q.y4 = LW(W_Y + 3);
#undef LW
}
S2D void store_per(const Per &q, double *w, int P, int j) {
#define LW(a) w[((a) * P + j) * 32]
    LW(W_X + 0) = q.xg; LW(W_X + 1) = q.xi; LW(W_X + 2) = q.xo; LW(W_X + 3) = q.xs; LW(W_X + 4) = q.xe; LW(W_X + 5) = q.xp; LW(W_X + 6) = q.xq;
    LW(W_Z + 0) = q.zg; LW(W_Z + 1) = q.zi; LW(W_Z + 2) = q.zo; LW(W_Z + 3) = q.zs; LW(W_Z + 4) = q.ze; LW(W_Z + 5) = q.zp; LW(W_Z + 6) = q.zq;
    LW(W_S + 0) = q.si; LW(W_S + 1) = q.so; LW(W_W + 0) = q.wi; LW(W_W + 1) = q.wo;
    LW(W_Y + 0) = q.y1; LW(W_Y + 1) = q.y2; LW(W_Y + 2) = q.y3; LW(W_Y + 3) = q.y4;
#undef LW
}

// solves LP p with the whole warp; returns 0 when optimal, else (iterations so far + 1) for the second attempt
__device__ int solve_long(const LongParams &LQ, double *wsw, long long p, int lane, double step_frac, double reg, int it0) {
    const stage2::Params &Q = LQ.q;
    const int P = LQ.P, T = Q.T;
    constexpr int L = 32;
    double *w = wsw + lane;
#define WS(a, j) w[((a) * P + (j)) * 32]
#define LSCAL(j) make_scal(WS(W_SC + 0, j), WS(W_SC + 1, j), WS(W_SC + 2, j), WS(W_SC + 3, j), WS(W_SC + 4, j), WS(W_SC + 5, j), WS(W_SC + 6, j), WS(W_SC + 7, j), WS(W_SC + 8, j), dl)
    Cst K;
    K.a = Q.a; K.binv = Q.binv; K.hf = Q.hf; K.dl = Q.dl;
    const double a = K.a, binv = K.binv, hf = K.hf, dl = K.dl;
    constexpr int r_root = L / 2;
    constexpr int kmax = (r_root - 1 > L - 2 - r_root) ? r_root - 1 : L - 2 - r_root;
    constexpr int smax = (r_root > L - 1 - r_root) ? r_root : L - 1 - r_root;
    const int t0 = lane * P;                      // first period of this lane
#define ACT(j) (t0 + (j) < T)
#define HAS_S(j) (t0 + (j) < T - 1)

    // ---- load, scale, start point
    const double *cp = Q.cparams + p * (long long)Q.Pc;
    const double *rp = Q.rparams + p * Q.rstride;
    double kc = 0.0, b4m = 0.0, cm = 0.0;
    for (int r = lane; r < Q.Pr; r += 32) kc += Q.omap[r] * rp[r];
    for (int r = lane; r < Q.Pc; r += 32) kc += Q.ocmap[r] * cp[r];
    const double Pw = rp[Q.p_off];
    for (int j = 0; j < P; ++j) {
        const int t = t0 + j;
        const double cj = t < T ? Q.krev * cp[t] : 0.0, bj = t < T ? rp[Q.wcf_off + t] : 0.0;
        WS(W_C, j) = cj; WS(W_B4, j) = bj;
        b4m = dmax(b4m, fabs(bj)); cm = dmax(cm, fabs(cj));
    }
    kc = gsum<L>(kc); b4m = gmax<L>(b4m); cm = gmax<L>(cm);
    const double kconst = kc + Q.o0;
    if (Pw < 0.0) {
        if (lane == 0) { Q.obj[p] = __longlong_as_double(0x7ff8000000000000LL); Q.status[p] = DSP_INFEASIBLE; Q.iters[p] = it0; }
        return 0;
    }
    const double b3u = Q.dur * Pw;
    double beta_b = dmax(dmax(fabs(b3u), b4m), Pw);
    beta_b = beta_b > 0.0 ? beta_b : 1.0;
    const double beta_c = cm > 0.0 ? cm : 1.0;
    const double b3 = b3u / beta_b, u = dmax(Pw / beta_b, 1e-10);
    const double nrm_b = 1.0 + dmax(fabs(b3), b4m / beta_b), nrm_c = 1.0 + (cm > 0.0 ? 1.0 : 0.0);
    const double ntot = (double)(9 * (long long)T - 1);
    {
        const double x0 = fmin(1.0, 0.5 * u);
        for (int j = 0; j < P; ++j) {
            const bool act = ACT(j), has_s = HAS_S(j);
            WS(W_C, j) = WS(W_C, j) / beta_c; WS(W_B4, j) = WS(W_B4, j) / beta_b;
            const double one = act ? 1.0 : 0.0;
            Per q;
            q.xg = one; q.xi = act ? x0 : 0.0; q.xo = q.xi; q.xs = has_s ? 1.0 : 0.0; q.xe = one; q.xp = one; q.xq = one;
            q.zg = one; q.zi = one; q.zo = one; q.zs = has_s ? 1.0 : 0.0; q.ze = one; q.zp = one; q.zq = one;
            q.si = act ? u - x0 : 0.0; q.so = q.si; q.wi = one; q.wo = one;
            q.y1 = q.y2 = q.y3 = q.y4 = 0.0;
            store_per(q, w, P, j);
        }
    }

    int status = DSP_MAX_ITER, it = 0;
    double po_last = 0.0;
    for (it = 0; it <= Q.max_iter; ++it) {
        // neighbours of the lane's chunk: state of the left lane's last period, duals of the right lane's first period
        const double xs_left = gup1<L>(WS(W_X + 3, P - 1), lane), xe_left = gup1<L>(WS(W_X + 4, P - 1), lane);
        const double y1_right = gdown1<L>(WS(W_Y + 0, 0), lane), y2_right = gdown1<L>(WS(W_Y + 1, 0), lane);
#define Y1N(j) ((j) == P - 1 ? y1_right : WS(W_Y + 0, (j) + 1))
#define Y2N(j) ((j) == P - 1 ? y2_right : WS(W_Y + 1, (j) + 1))

        // =========================================================================================== pass 1
        double pm = 0.0, dm = 0.0, mus = 0.0, po = 0.0, dob = 0.0;
        double s11l, s22l, s12l;
        {
            double s11c = 0.0, s22c = 0.0, s12c = 0.0, ph1c = 0.0, ph2c = 0.0, xsp = xs_left, xep = xe_left;
            for (int j = 0; j < P; ++j) {
                const bool act = ACT(j), has_s = HAS_S(j);
                Sym2 D; double f1, f2;
                if (act) {
                    Per q; load_per(q, w, P, j);
                    const double cj = WS(W_C, j), b4j = WS(W_B4, j);
                    Res r;
                    residuals(q, cj, b4j, xsp, xep, Y1N(j), Y2N(j), b3, u, K, act, has_s, r);
                    pm = dmax(pm, dmax(dmax(dmax(fabs(r.rp1), fabs(r.rp2)), dmax(fabs(r.rp3), fabs(r.rp4))), dmax(fabs(r.rui), fabs(r.ruo))));
                    dm = dmax(dm, dmax(dmax(dmax(fabs(r.rdg), fabs(r.rdi)), dmax(fabs(r.rdo), fabs(r.rds))),
                                       dmax(dmax(fabs(r.rde), fabs(r.rdp)), fabs(r.rdq))));
                    mus += q.xg * q.zg + q.xi * q.zi + q.xo * q.zo + q.xs * q.zs + q.xe * q.ze + q.xp * q.zp + q.xq * q.zq
                           + q.si * q.wi + q.so * q.wo;
                    po += cj * (q.xg + q.xo);
                    dob += b3 * q.y3 + b4j * q.y4 - u * (q.wi + q.wo);
                    const double rxg = frcp(q.xg), rxi = frcp(q.xi), rxo = frcp(q.xo), rxe = frcp(q.xe), rxp = frcp(q.xp), rxq = frcp(q.xq);
                    const double rxs = has_s ? frcp(q.xs) : 0.0;
                    const double rsi = frcp(q.si), rso = frcp(q.so);
                    const double qg = q.xg > 1.0 ? reg * rxg * rxg : reg, qe = q.xe > 1.0 ? reg * rxe * rxe : reg;
                    const double qp = q.xp > 1.0 ? reg * rxp * rxp : reg, qq = q.xq > 1.0 ? reg * rxq * rxq : reg;
                    const double qs = q.xs > 1.0 ? reg * rxs * rxs : reg;
                    const double dg = q.xg * frcp(fma(qg, q.xg, q.zg)), de = q.xe * frcp(fma(qe, q.xe, q.ze));
                    const double dp = q.xp * frcp(fma(qp, q.xp, q.zp)), dq = q.xq * frcp(fma(qq, q.xq, q.zq));
                    const double ds = has_s ? q.xs * frcp(fma(qs, q.xs, q.zs)) : 0.0;
                    const double di = frcp(fma(q.zi, rxi, q.wi * rsi) + reg), dO = frcp(fma(q.zo, rxo, q.wo * rso) + reg);
                    const double kap = frcp(ds + dl * dl * de + dp);
                    const double iot = frcp(dg + di + dq);
                    const Scal sc = make_scal(ds, de, dp, kap, dg, di, dq, iot, dO, dl);
                    const double s11 = sc.s11, s22 = sc.s22, s12 = sc.s12, tau = sc.tau, dsk = sc.dsk, dek = sc.dek, dii = sc.dii;
                    D.a = s11 + s11c + a * a * tau + binv * binv * dO;
                    D.c = s22 + s22c + hf * hf * (tau + dO);
                    D.b = a * hf * tau - hf * binv * dO - s12 - s12c;
                    const double hg = r.rdg + q.zg, he = r.rde + q.ze, hp = r.rdp + q.zp, hq = r.rdq + q.zq;
                    const double hs = has_s ? r.rds + q.zs : 0.0;
                    const double hi = r.rdi + q.zi + (-q.wi * r.rui) * rsi - q.wi;
                    const double ho = r.rdo + q.zo + (-q.wo * r.ruo) * rso - q.wo;
                    const double w3 = r.rp3 + dp * hp;
                    const double ph1 = s11 * hs - s12 * he - dsk * w3;
                    const double ph2 = s22 * he - s12 * hs - dek * w3;
                    const double w4 = r.rp4 + dg * hg + dq * hq;
                    const double psi = tau * hi - dii * w4;
                    const double doh = dO * ho;
                    f1 = r.rp1 + ph1 - ph1c - a * psi + binv * doh;
                    f2 = r.rp2 + ph2 - ph2c - hf * psi - hf * doh;
                    WS(W_SC + 0, j) = ds; WS(W_SC + 1, j) = de; WS(W_SC + 2, j) = dp; WS(W_SC + 3, j) = kap;
                    WS(W_SC + 4, j) = dg; WS(W_SC + 5, j) = di; WS(W_SC + 6, j) = dq; WS(W_SC + 7, j) = iot; WS(W_SC + 8, j) = dO;
                    WS(W_RX + 0, j) = rxg; WS(W_RX + 1, j) = rxi; WS(W_RX + 2, j) = rxo; WS(W_RX + 3, j) = rxs;
                    WS(W_RX + 4, j) = rxe; WS(W_RX + 5, j) = rxp; WS(W_RX + 6, j) = rxq;
                    s11c = has_s ? s11 : 0.0; s22c = has_s ? s22 : 0.0; s12c = has_s ? s12 : 0.0; ph1c = ph1; ph2c = ph2;
                    xsp = q.xs; xep = q.xe;
                } else {
                    D.a = 1.0; D.b = 0.0; D.c = 1.0; f1 = 0.0; f2 = 0.0;
                    for (int k = 0; k < 16; ++k) WS(W_SC + k, j) = 0.0;
                    s11c = s22c = s12c = ph1c = ph2c = 0.0; xsp = 0.0; xep = 0.0;
                }
                WS(W_D + 0, j) = D.a; WS(W_D + 1, j) = D.b; WS(W_D + 2, j) = D.c;
                WS(W_F + 0, j) = f1; WS(W_F + 1, j) = f2;
            }
            s11l = gup1<L>(s11c, lane); s22l = gup1<L>(s22c, lane); s12l = gup1<L>(s12c, lane);
            const double ph1l = gup1<L>(ph1c, lane), ph2l = gup1<L>(ph2c, lane);
            if (ACT(0)) {
                WS(W_D + 0, 0) += s11l; WS(W_D + 2, 0) += s22l; WS(W_D + 1, 0) -= s12l;
                WS(W_F + 0, 0) -= ph1l; WS(W_F + 1, 0) -= ph2l;
            }
        }
        const double res = gmax<L>(dmax(pm / nrm_b, dm / nrm_c));
        mus = gsum<L>(mus); po = gsum<L>(po); dob = gsum<L>(dob);
        po_last = po;
        const double mu = mus / ntot;
        {
            const double den = dmax(kGapFloor2, fabs(po));
            const double gap = fabs(po - dob) / den, cgap = ntot * mu / den;
#if !defined(__CUDA_ARCH__) && defined(DSP_EMU_TRACE)
            if (lane == 0) printf("it %2d  res %.2e (p %.2e d %.2e)  gap %.2e  cgap %.2e  mu %.2e\n", it, res, gmax<1>(pm) / nrm_b, dm / nrm_c, gap, cgap, mu);
#endif
            if (!(mu == mu) || !(po == po) || mu > 1e100) { status = DSP_NUMERICAL; break; }
            if (res < Q.feas_tol && gap < Q.tol) { status = DSP_OPTIMAL; break; }
            if (cgap < Q.tol && res < 10.0 * Q.feas_tol && gap < 10.0 * Q.tol) { status = DSP_OPTIMAL; break; }
            if (cgap < 1e-3 * Q.tol) { status = (res < 100.0 * Q.feas_tol && gap < 1000.0 * Q.tol) ? DSP_OPTIMAL : DSP_NUMERICAL; break; }
            if (it == Q.max_iter) break;
        }

        // =========================================================================================== factorisation (+ forward part of the predictor solve)
        Mat2 Wc, Mout, Mout2, Cin;       // Mout / Mout2 + mo4 / mo24: the five multipliers (l, m1a, m1b, m2a, m2b) of a separator elimination
        Sym2 Asep, Ainv;                 // Ainv: (1/a, l, 1/c') of the separator's final pivot block
        double g1, g2, mo4 = 0.0, mo24 = 0.0;
        int fo, bo, fsrc, bsrc;
        const bool is_root = (lane == r_root);
        {
            Mat2 E;
            {
                const bool cpl = (lane > 0) && ACT(0);
                E.a = cpl ? -s11l : 0.0; E.d = cpl ? -s22l : 0.0; E.b = cpl ? s12l : 0.0; E.c = E.b;
            }
            Sym2 dS; dS.a = dS.b = dS.c = 0.0;
            double dg1 = 0.0, dg2 = 0.0;
            Sym2 Dc; Dc.a = WS(W_D + 0, 0); Dc.b = WS(W_D + 1, 0); Dc.c = WS(W_D + 2, 0);
            double fa = WS(W_F + 0, 0), fb = WS(W_F + 1, 0);
            for (int j = 0; j < P - 1; ++j) {
                const Scal sc = LSCAL(j);
                const bool cn = HAS_S(j);
                // coupling (next period, this period): symmetric 2x2, entries [k][m] = equation (next, k), unknown (this, m)
                const double Ca = cn ? -sc.s11 : 0.0, Cb = cn ? sc.s12 : 0.0, Cd = cn ? -sc.s22 : 0.0;
                Sym2 Dn; Dn.a = WS(W_D + 0, j + 1); Dn.b = WS(W_D + 1, j + 1); Dn.c = WS(W_D + 2, j + 1);
                double fn1 = WS(W_F + 0, j + 1), fn2 = WS(W_F + 1, j + 1);
                // ---- pivot 1: unknown u1 of this period
                const double i1 = frcp(Dc.a);
                const double l = Dc.b * i1;
                const double mn1 = Ca * i1, mn2 = Cb * i1;                 // column 0 of C over the pivot
                const double ms1 = E.a * i1, ms2 = E.b * i1;               // row 0 of E (= column 0 of the (separator, this) block)
                const double c2 = fma(-l, Dc.b, Dc.c);
                const double Cb1 = fma(-mn1, Dc.b, Cb), Cd1 = fma(-mn2, Dc.b, Cd);     // column 1 of C after the first elimination
                const double Ec1 = fma(-ms1, Dc.b, E.c), Ed1 = fma(-ms2, Dc.b, E.d);   // row 1 of E after it
                Dn.a = fma(-mn1, Ca, Dn.a); Dn.b = fma(-mn1, Cb, Dn.b); Dn.c = fma(-mn2, Cb, Dn.c);
                dS.a = fma(-ms1, E.a, dS.a); dS.b = fma(-ms1, E.b, dS.b); dS.c = fma(-ms2, E.b, dS.c);
                Mat2 En;                                                    // fill (next period, separator)
                En.a = -Ca * ms1; En.b = -Ca * ms2; En.c = -Cb * ms1; En.d = -Cb * ms2;
                const double fb1 = fma(-l, fa, fb);
                fn1 = fma(-mn1, fa, fn1); fn2 = fma(-mn2, fa, fn2);
                dg1 = fma(-ms1, fa, dg1); dg2 = fma(-ms2, fa, dg2);
                // ---- pivot 2: unknown u2
                const double i2 = frcp(c2);
                const double mq1 = Cb1 * i2, mq2 = Cd1 * i2;
                const double mt1 = Ec1 * i2, mt2 = Ed1 * i2;
                Dn.a = fma(-mq1, Cb1, Dn.a); Dn.b = fma(-mq1, Cd1, Dn.b); Dn.c = fma(-mq2, Cd1, Dn.c);
                dS.a = fma(-mt1, Ec1, dS.a); dS.b = fma(-mt1, Ed1, dS.b); dS.c = fma(-mt2, Ed1, dS.c);
                En.a = fma(-Cb1, mt1, En.a); En.b = fma(-Cb1, mt2, En.b); En.c = fma(-Cd1, mt1, En.c); En.d = fma(-Cd1, mt2, En.d);
                fn1 = fma(-mq1, fb1, fn1); fn2 = fma(-mq2, fb1, fn2);
                dg1 = fma(-mt1, fb1, dg1); dg2 = fma(-mt2, fb1, dg2);
                WS(W_K + 0, j) = i1; WS(W_K + 1, j) = l; WS(W_K + 2, j) = i2;
                WS(W_G + 0, j) = mn1; WS(W_G + 1, j) = mn2; WS(W_G + 2, j) = mq1; WS(W_G + 3, j) = mq2;
                WS(W_H + 0, j) = ms1; WS(W_H + 1, j) = ms2; WS(W_H + 2, j) = mt1; WS(W_H + 3, j) = mt2;
                WS(W_F + 0, j) = fa; WS(W_F + 1, j) = fb1;
                E = En; Dc = Dn; fa = fn1; fb = fn2;
            }
            Wc = E; Asep = Dc; g1 = fa; g2 = fb;
            Asep.a += gdown1<L>(dS.a, lane); Asep.b += gdown1<L>(dS.b, lane); Asep.c += gdown1<L>(dS.c, lane);
            g1 += gdown1<L>(dg1, lane); g2 += gdown1<L>(dg2, lane);
            Mat2 Wn;
            Wn.a = gdown1<L>(Wc.a, lane); Wn.b = gdown1<L>(Wc.b, lane); Wn.c = gdown1<L>(Wc.c, lane); Wn.d = gdown1<L>(Wc.d, lane);
            const bool low = lane < r_root;
            fsrc = low ? (lane > 0 ? lane - 1 : 0) : (lane < L - 1 ? lane + 1 : L - 1);
            bsrc = low ? lane + 1 : lane - 1;
            fo = is_root ? (1 << 20) : (low ? lane : L - 1 - lane);
            bo = is_root ? (1 << 20) : (low ? r_root - lane : lane - r_root);
            const Mat2 Cout = low ? Wc : transp(Wn);
            Cin = low ? transp(Wn) : Wc;
            // eliminating a neighbouring separator R (right-hand side q) from this one through the coupling Co (rows: this, columns: R):
            // two scalar pivots; the multipliers (l, m1a, m1b, m2a, m2b) are kept for the corrector's forward solve
#define SEP_ELIM(Co, R, q1, q2, M)                                                                    \
            {                                                                                         \
                const double i1_ = frcp(R.a), l_ = R.b * i1_;                                         \
                const double m1a = Co.a * i1_, m1b = Co.c * i1_;                                      \
                const double c2_ = fma(-l_, R.b, R.c);                                                \
                const double ka_ = fma(-m1a, R.b, Co.b), kb_ = fma(-m1b, R.b, Co.d);                  \
                const double i2_ = frcp(c2_);                                                         \
                const double m2a = ka_ * i2_, m2b = kb_ * i2_;                                        \
                Asep.a -= fma(m1a, Co.a, m2a * ka_); Asep.b -= fma(m1a, Co.c, m2a * kb_); Asep.c -= fma(m1b, Co.c, m2b * kb_); \
                const double q2_ = fma(-l_, q1, q2);                                                  \
                g1 -= fma(m1a, q1, m2a * q2_); g2 -= fma(m1b, q1, m2b * q2_);                         \
                M[0] = l_; M[1] = m1a; M[2] = m1b; M[3] = m2a; M[4] = m2b;                            \
            }
            double Mo[5] = {0, 0, 0, 0, 0}, Mo2[5] = {0, 0, 0, 0, 0};
            for (int k = 1; k <= kmax; ++k) {
                Sym2 R;
                R.a = gfrom<L>(Asep.a, fsrc); R.b = gfrom<L>(Asep.b, fsrc); R.c = gfrom<L>(Asep.c, fsrc);
                const double q1 = gfrom<L>(g1, fsrc), q2 = gfrom<L>(g2, fsrc);
                if (fo == k) SEP_ELIM(Cout, R, q1, q2, Mo)
            }
            {
                constexpr int la = r_root - 1, lb = r_root + 1;
                Sym2 Ra, Rb;
                Ra.a = gfrom<L>(Asep.a, la); Ra.b = gfrom<L>(Asep.b, la); Ra.c = gfrom<L>(Asep.c, la);
                Rb.a = gfrom<L>(Asep.a, lb); Rb.b = gfrom<L>(Asep.b, lb); Rb.c = gfrom<L>(Asep.c, lb);
                const double a1 = gfrom<L>(g1, la), a2 = gfrom<L>(g2, la), b1 = gfrom<L>(g1, lb), b2 = gfrom<L>(g2, lb);
                if (is_root) {
                    SEP_ELIM(Wc, Ra, a1, a2, Mo)
                    const Mat2 Wt = transp(Wn);
                    SEP_ELIM(Wt, Rb, b1, b2, Mo2)
                }
            }
#undef SEP_ELIM
            // the final pivot block of every separator, as scalar pivots too
            Ainv.a = frcp(Asep.a); Ainv.b = Asep.b * Ainv.a; Ainv.c = frcp(fma(-Ainv.b, Asep.b, Asep.c));     // (1/a, l, 1/c')
            Mout.a = Mo[0]; Mout.b = Mo[1]; Mout.c = Mo[2]; Mout.d = Mo[3]; Mout2.a = Mo2[0]; Mout2.b = Mo2[1]; Mout2.c = Mo2[2]; Mout2.d = Mo2[3];
            mo4 = Mo[4]; mo24 = Mo2[4];
        }
        // separator back substitution + local back substitution; the solution dy overwrites W_F
#define SEP_SOLVE(t1, t2, o1, o2) { const double t2_ = fma(-Ainv.b, (t1), (t2)); o2 = t2_ * Ainv.c; o1 = fma((t1), Ainv.a, -Ainv.b * o2); }
#define BACK_ALL()                                                                                    \
        {                                                                                             \
            double u1 = 0.0, u2 = 0.0;                                                                \
            if (is_root) SEP_SOLVE(g1, g2, u1, u2)                                                    \
            for (int s = 1; s <= smax; ++s) {                                                         \
                const double r1 = gfrom<L>(u1, bsrc), r2 = gfrom<L>(u2, bsrc);                        \
                if (bo == s) {                                                                        \
                    const double t1 = g1 - fma(Cin.a, r1, Cin.b * r2);                                \
                    const double t2 = g2 - fma(Cin.c, r1, Cin.d * r2);                                \
                    SEP_SOLVE(t1, t2, u1, u2)                                                         \
                }                                                                                     \
            }                                                                                         \
            const double ul1 = gup1<L>(u1, lane), ul2 = gup1<L>(u2, lane);                            \
            double n1 = u1, n2 = u2;                                                                  \
            WS(W_F + 0, P - 1) = u1; WS(W_F + 1, P - 1) = u2;                                         \
            for (int j = P - 2; j >= 0; --j) {                                                        \
                const double i1 = WS(W_K + 0, j), l = WS(W_K + 1, j), i2 = WS(W_K + 2, j);            \
                const double mn1 = WS(W_G + 0, j), mn2 = WS(W_G + 1, j), mq1 = WS(W_G + 2, j), mq2 = WS(W_G + 3, j); \
                const double ms1 = WS(W_H + 0, j), ms2 = WS(W_H + 1, j), mt1 = WS(W_H + 2, j), mt2 = WS(W_H + 3, j); \
                const double e1 = WS(W_F + 0, j), e2 = WS(W_F + 1, j);                                \
                const double v2 = e2 * i2 - fma(mq1, n1, mq2 * n2) - fma(mt1, ul1, mt2 * ul2);        \
                const double v1 = e1 * i1 - l * v2 - fma(mn1, n1, mn2 * n2) - fma(ms1, ul1, ms2 * ul2); \
                WS(W_F + 0, j) = v1; WS(W_F + 1, j) = v2;                                             \
                n1 = v1; n2 = v2;                                                                     \
            }                                                                                         \
        }
        BACK_ALL();

        // =========================================================================================== pass 2: predictor direction
        double smu;
        {
            const double dy1_right = gdown1<L>(WS(W_F + 0, 0), lane), dy2_right = gdown1<L>(WS(W_F + 1, 0), lane);
            double ip = 0.0, id = 0.0, S1 = 0.0, S3 = 0.0, xsp = xs_left, xep = xe_left;
            for (int j = 0; j < P; ++j) {
                if (!ACT(j)) continue;
                const bool has_s = HAS_S(j);
                Per q; load_per(q, w, P, j);
                Res r;
                residuals(q, WS(W_C, j), WS(W_B4, j), xsp, xep, Y1N(j), Y2N(j), b3, u, K, true, has_s, r);
                xsp = q.xs; xep = q.xe;
                const double rxg = WS(W_RX + 0, j), rxi = WS(W_RX + 1, j), rxo = WS(W_RX + 2, j), rxs = WS(W_RX + 3, j);
                const double rxe = WS(W_RX + 4, j), rxp = WS(W_RX + 5, j), rxq = WS(W_RX + 6, j);
                const double rsi = frcp(q.si), rso = frcp(q.so);
                const Scal sc = LSCAL(j);
                const double s11 = sc.s11, s22 = sc.s22, s12 = sc.s12, dsk = sc.dsk, dek = sc.dek;
                const double kap = sc.kap, tau = sc.tau, dii = sc.dii, iot = sc.iot, dO = sc.dO;
                const double dg = sc.dg, dq = sc.dq, dp = sc.dp, di = sc.di;
                const double hg = r.rdg + q.zg, he = r.rde + q.ze, hp = r.rdp + q.zp, hq = r.rdq + q.zq;
                const double hs = has_s ? r.rds + q.zs : 0.0;
                const double hi = r.rdi + q.zi + (-q.wi * r.rui) * rsi - q.wi;
                const double ho = r.rdo + q.zo + (-q.wo * r.ruo) * rso - q.wo;
                const double w3 = r.rp3 + dp * hp, w4 = r.rp4 + dg * hg + dq * hq;
                const double dy1 = WS(W_F + 0, j), dy2 = WS(W_F + 1, j);
                const double d1n = (j == P - 1) ? dy1_right : WS(W_F + 0, j + 1);
                const double d2n = (j == P - 1) ? dy2_right : WS(W_F + 1, j + 1);
                const double e1 = dy1 - d1n - hs, e2 = dy2 - d2n - he;
                const double v = a * dy1 + hf * dy2;
                const double dxs = has_s ? s11 * e1 - s12 * e2 + dsk * w3 : 0.0;
                const double dxe = s22 * e2 - s12 * e1 + dek * w3;
                const double dxi = -tau * (v + hi) + dii * w4;
                const double dxo = dO * (binv * dy1 - hf * dy2 - ho);
                const double dxg = dg * iot * (r.rp4 + di * (hi - hg + v) + dq * (hq - hg));
                const double dy3 = kap * w3 - dsk * e1 - dek * e2;
                const double dy4 = iot * w4 + dii * (hi + v);
                const double dxp = dp * (dy3 - hp), dxq = dq * (dy4 - hq);
                const double tg = dxg * rxg, ti = dxi * rxi, to = dxo * rxo, ts = dxs * rxs, te = dxe * rxe, tp = dxp * rxp, tq = dxq * rxq;
                const double dzg = -q.zg - q.zg * tg, dzi = -q.zi - q.zi * ti, dzo = -q.zo - q.zo * to, dzs = has_s ? -q.zs - q.zs * ts : 0.0;
                const double dze = -q.ze - q.ze * te, dzp = -q.zp - q.zp * tp, dzq = -q.zq - q.zq * tq;
                const double dsi = r.rui - dxi, dso = r.ruo - dxo;
                const double tsi = dsi * rsi, tso = dso * rso;
                const double dwi = -q.wi - q.wi * tsi, dwo = -q.wo - q.wo * tso;
                ip = dmax(ip, dmax(dmax(dmax(-tg, -ti), dmax(-to, -ts)), dmax(dmax(-te, -tp), dmax(-tq, dmax(-tsi, -tso)))));
                id = dmax(id, dmax(dmax(dmax(1.0 + tg, 1.0 + ti), dmax(1.0 + to, has_s ? 1.0 + ts : 0.0)),
                                   dmax(dmax(1.0 + te, 1.0 + tp), dmax(1.0 + tq, dmax(1.0 + tsi, 1.0 + tso)))));
                S1 += q.zg * dxg + q.zi * dxi + q.zo * dxo + q.zs * dxs + q.ze * dxe + q.zp * dxp + q.zq * dxq + q.wi * dsi + q.wo * dso;
                const double cg = dxg * dzg, ci = dxi * dzi, co = dxo * dzo, cs = dxs * dzs, ce = dxe * dze, cpp = dxp * dzp, cq = dxq * dzq;
                const double csi = dsi * dwi, cso = dso * dwo;
                S3 += cg + ci + co + cs + ce + cpp + cq + csi + cso;
                WS(W_PR + 0, j) = cg; WS(W_PR + 1, j) = ci; WS(W_PR + 2, j) = co; WS(W_PR + 3, j) = cs; WS(W_PR + 4, j) = ce;
                WS(W_PR + 5, j) = cpp; WS(W_PR + 6, j) = cq; WS(W_PR + 7, j) = csi; WS(W_PR + 8, j) = cso;
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
            double ph1c = 0.0, ph2c = 0.0, xsp = xs_left, xep = xe_left;
            double dg1 = 0.0, dg2 = 0.0, fpa = 0.0, fpb = 0.0;      // forward elimination runs along: (fpa, fpb) = eliminated rhs of j-1
            double f1_0 = 0.0, f2_0 = 0.0;
            // first the raw right-hand sides (period 0 needs the left lane's ph after the loop)
            for (int j = 0; j < P; ++j) {
                double f1 = 0.0, f2 = 0.0;
                if (ACT(j)) {
                    const bool has_s = HAS_S(j);
                    Per q; load_per(q, w, P, j);
                    Res r;
                    residuals(q, WS(W_C, j), WS(W_B4, j), xsp, xep, Y1N(j), Y2N(j), b3, u, K, true, has_s, r);
                    xsp = q.xs; xep = q.xe;
                    const double rsi = frcp(q.si), rso = frcp(q.so);
                    const Scal sc = LSCAL(j);
                    const double hg = r.rdg + q.zg - (smu - WS(W_PR + 0, j)) * WS(W_RX + 0, j);
                    const double hs = has_s ? r.rds + q.zs - (smu - WS(W_PR + 3, j)) * WS(W_RX + 3, j) : 0.0;
                    const double he = r.rde + q.ze - (smu - WS(W_PR + 4, j)) * WS(W_RX + 4, j);
                    const double hp = r.rdp + q.zp - (smu - WS(W_PR + 5, j)) * WS(W_RX + 5, j);
                    const double hq = r.rdq + q.zq - (smu - WS(W_PR + 6, j)) * WS(W_RX + 6, j);
                    const double asi = -q.wi * r.rui + smu - WS(W_PR + 7, j), aso = -q.wo * r.ruo + smu - WS(W_PR + 8, j);
                    const double hi = r.rdi + q.zi - (smu - WS(W_PR + 1, j)) * WS(W_RX + 1, j) + asi * rsi - q.wi;
                    const double ho = r.rdo + q.zo - (smu - WS(W_PR + 2, j)) * WS(W_RX + 2, j) + aso * rso - q.wo;
                    const double w3 = r.rp3 + sc.dp * hp;
                    const double ph1 = sc.s11 * hs - sc.s12 * he - sc.dsk * w3;
                    const double ph2 = sc.s22 * he - sc.s12 * hs - sc.dek * w3;
                    const double w4 = r.rp4 + sc.dg * hg + sc.dq * hq;
                    const double psi = sc.tau * hi - sc.dii * w4;
                    const double doh = sc.dO * ho;
                    f1 = r.rp1 + ph1 - ph1c - a * psi + binv * doh;
                    f2 = r.rp2 + ph2 - ph2c - hf * psi - hf * doh;
                    ph1c = ph1; ph2c = ph2;
                } else {
                    ph1c = 0.0; ph2c = 0.0; xsp = 0.0; xep = 0.0;
                }
                WS(W_F + 0, j) = f1; WS(W_F + 1, j) = f2;
            }
            const double ph1l = gup1<L>(ph1c, lane), ph2l = gup1<L>(ph2c, lane);
            if (ACT(0)) { WS(W_F + 0, 0) -= ph1l; WS(W_F + 1, 0) -= ph2l; }
            (void)fpa; (void)fpb; (void)f1_0; (void)f2_0;
            double fa = WS(W_F + 0, 0), fb = WS(W_F + 1, 0);
            for (int j = 0; j < P - 1; ++j) {
                const double l = WS(W_K + 1, j);
                const double mn1 = WS(W_G + 0, j), mn2 = WS(W_G + 1, j), mq1 = WS(W_G + 2, j), mq2 = WS(W_G + 3, j);
                const double ms1 = WS(W_H + 0, j), ms2 = WS(W_H + 1, j), mt1 = WS(W_H + 2, j), mt2 = WS(W_H + 3, j);
                const double fb1 = fma(-l, fa, fb);
                dg1 -= fma(ms1, fa, mt1 * fb1); dg2 -= fma(ms2, fa, mt2 * fb1);
                const double fna = WS(W_F + 0, j + 1) - fma(mn1, fa, mq1 * fb1), fnb = WS(W_F + 1, j + 1) - fma(mn2, fa, mq2 * fb1);
                WS(W_F + 0, j) = fa; WS(W_F + 1, j) = fb1;
                fa = fna; fb = fnb;
            }
            g1 = fa + gdown1<L>(dg1, lane); g2 = fb + gdown1<L>(dg2, lane);
            // separator forward solve with the stored multipliers (l, m1a, m1b, m2a, m2b)
#define SEP_FWD(M, m4, q1, q2) { const double q2_ = fma(-M.a, (q1), (q2)); g1 -= fma(M.b, (q1), M.d * q2_); g2 -= fma(M.c, (q1), (m4) * q2_); }
            for (int k = 1; k <= kmax; ++k) {
                const double q1 = gfrom<L>(g1, fsrc), q2 = gfrom<L>(g2, fsrc);
                if (fo == k) SEP_FWD(Mout, mo4, q1, q2)
            }
            {
                constexpr int la = r_root - 1, lb = r_root + 1;
                const double a1 = gfrom<L>(g1, la), a2 = gfrom<L>(g2, la), b1 = gfrom<L>(g1, lb), b2 = gfrom<L>(g2, lb);
                if (is_root) {
                    SEP_FWD(Mout, mo4, a1, a2)
                    SEP_FWD(Mout2, mo24, b1, b2)
                }
            }
#undef SEP_FWD
        }
        BACK_ALL();

        // =========================================================================================== pass 4: corrector direction
        double ap, ad;
        {
            const double dy1_right = gdown1<L>(WS(W_F + 0, 0), lane), dy2_right = gdown1<L>(WS(W_F + 1, 0), lane);
            double ip = 0.0, id = 0.0, xsp = xs_left, xep = xe_left;
            for (int j = 0; j < P; ++j) {
                if (!ACT(j)) continue;
                const bool has_s = HAS_S(j);
                Per q; load_per(q, w, P, j);
                Res r;
                residuals(q, WS(W_C, j), WS(W_B4, j), xsp, xep, Y1N(j), Y2N(j), b3, u, K, true, has_s, r);
                xsp = q.xs; xep = q.xe;
                const double rxg = WS(W_RX + 0, j), rxi = WS(W_RX + 1, j), rxo = WS(W_RX + 2, j), rxs = WS(W_RX + 3, j);
                const double rxe = WS(W_RX + 4, j), rxp = WS(W_RX + 5, j), rxq = WS(W_RX + 6, j);
                const double rsi = frcp(q.si), rso = frcp(q.so);
                const Scal sc = LSCAL(j);
                const double s11 = sc.s11, s22 = sc.s22, s12 = sc.s12, dsk = sc.dsk, dek = sc.dek;
                const double kap = sc.kap, tau = sc.tau, dii = sc.dii, iot = sc.iot, dO = sc.dO;
                const double dg = sc.dg, dq = sc.dq, dp = sc.dp, di = sc.di;
                const double ag = smu - WS(W_PR + 0, j), ai = smu - WS(W_PR + 1, j), ao = smu - WS(W_PR + 2, j), as_ = smu - WS(W_PR + 3, j);
                const double ae = smu - WS(W_PR + 4, j), app = smu - WS(W_PR + 5, j), aq = smu - WS(W_PR + 6, j);
                const double asi_ = smu - WS(W_PR + 7, j), aso_ = smu - WS(W_PR + 8, j);
                const double hg = r.rdg + q.zg - ag * rxg, he = r.rde + q.ze - ae * rxe, hp = r.rdp + q.zp - app * rxp, hq = r.rdq + q.zq - aq * rxq;
                const double hs = has_s ? r.rds + q.zs - as_ * rxs : 0.0;
                const double hi = r.rdi + q.zi - ai * rxi + (-q.wi * r.rui + asi_) * rsi - q.wi;
                const double ho = r.rdo + q.zo - ao * rxo + (-q.wo * r.ruo + aso_) * rso - q.wo;
                const double w3 = r.rp3 + dp * hp, w4 = r.rp4 + dg * hg + dq * hq;
                const double dy1 = WS(W_F + 0, j), dy2 = WS(W_F + 1, j);
                const double d1n = (j == P - 1) ? dy1_right : WS(W_F + 0, j + 1);
                const double d2n = (j == P - 1) ? dy2_right : WS(W_F + 1, j + 1);
                const double e1 = dy1 - d1n - hs, e2 = dy2 - d2n - he;
                const double v = a * dy1 + hf * dy2;
                const double dxs = has_s ? s11 * e1 - s12 * e2 + dsk * w3 : 0.0;
                const double dxe = s22 * e2 - s12 * e1 + dek * w3;
                const double dxi = -tau * (v + hi) + dii * w4;
                const double dxo = dO * (binv * dy1 - hf * dy2 - ho);
                const double dxg = dg * iot * (r.rp4 + di * (hi - hg + v) + dq * (hq - hg));
                const double dy3 = kap * w3 - dsk * e1 - dek * e2;
                const double dy4 = iot * w4 + dii * (hi + v);
                const double dxp = dp * (dy3 - hp), dxq = dq * (dy4 - hq);
                const double dzg = ag * rxg - q.zg - q.zg * dxg * rxg, dzi = ai * rxi - q.zi - q.zi * dxi * rxi;
                const double dzo = ao * rxo - q.zo - q.zo * dxo * rxo, dzs = has_s ? as_ * rxs - q.zs - q.zs * dxs * rxs : 0.0;
                const double dze = ae * rxe - q.ze - q.ze * dxe * rxe, dzp = app * rxp - q.zp - q.zp * dxp * rxp;
                const double dzq = aq * rxq - q.zq - q.zq * dxq * rxq;
                const double dsi = r.rui - dxi, dso = r.ruo - dxo;
                const double dwi = asi_ * rsi - q.wi - q.wi * dsi * rsi, dwo = aso_ * rso - q.wo - q.wo * dso * rso;
                ip = dmax(ip, dmax(dmax(dmax(-dxg * rxg, -dxi * rxi), dmax(-dxo * rxo, -dxs * rxs)),
                                   dmax(dmax(-dxe * rxe, -dxp * rxp), dmax(-dxq * rxq, dmax(-dsi * rsi, -dso * rso)))));
                id = dmax(id, dmax(dmax(dmax(-dzg * frcp(q.zg), -dzi * frcp(q.zi)), dmax(-dzo * frcp(q.zo), has_s ? -dzs * frcp(q.zs) : 0.0)),
                                   dmax(dmax(-dze * frcp(q.ze), -dzp * frcp(q.zp)),
                                        dmax(-dzq * frcp(q.zq), dmax(-dwi * frcp(q.wi), -dwo * frcp(q.wo))))));
                WS(W_SC + 0, j) = dxg; WS(W_SC + 1, j) = dxi; WS(W_SC + 2, j) = dxo; WS(W_SC + 3, j) = dxs; WS(W_SC + 4, j) = dxe;
                WS(W_SC + 5, j) = dxp; WS(W_SC + 6, j) = dxq; WS(W_SC + 7, j) = dy3; WS(W_SC + 8, j) = dy4;
            }
            ip = gmax<L>(ip); id = gmax<L>(id);
            ap = step_frac < ip ? step_frac / ip : 1.0;
            ad = step_frac < id ? step_frac / id : 1.0;
        }

        // =========================================================================================== pass 5: step
        for (int j = 0; j < P; ++j) {
            if (!ACT(j)) continue;
            const bool has_s = HAS_S(j);
            Per q; load_per(q, w, P, j);
            const double rxg = WS(W_RX + 0, j), rxi = WS(W_RX + 1, j), rxo = WS(W_RX + 2, j), rxs = WS(W_RX + 3, j);
            const double rxe = WS(W_RX + 4, j), rxp = WS(W_RX + 5, j), rxq = WS(W_RX + 6, j);
            const double rsi = frcp(q.si), rso = frcp(q.so);
            const double dxg = WS(W_SC + 0, j), dxi = WS(W_SC + 1, j), dxo = WS(W_SC + 2, j), dxs = WS(W_SC + 3, j);
            const double dxe = WS(W_SC + 4, j), dxp = WS(W_SC + 5, j), dxq = WS(W_SC + 6, j);
            const double dsi = (u - q.xi - q.si) - dxi, dso = (u - q.xo - q.so) - dxo;
            const double dzg = (smu - WS(W_PR + 0, j)) * rxg - q.zg - q.zg * dxg * rxg;
            const double dzi = (smu - WS(W_PR + 1, j)) * rxi - q.zi - q.zi * dxi * rxi;
            const double dzo = (smu - WS(W_PR + 2, j)) * rxo - q.zo - q.zo * dxo * rxo;
            const double dzs = (smu - WS(W_PR + 3, j)) * rxs - q.zs - q.zs * dxs * rxs;
            const double dze = (smu - WS(W_PR + 4, j)) * rxe - q.ze - q.ze * dxe * rxe;
            const double dzp = (smu - WS(W_PR + 5, j)) * rxp - q.zp - q.zp * dxp * rxp;
            const double dzq = (smu - WS(W_PR + 6, j)) * rxq - q.zq - q.zq * dxq * rxq;
            const double dwi = (smu - WS(W_PR + 7, j)) * rsi - q.wi - q.wi * dsi * rsi;
            const double dwo = (smu - WS(W_PR + 8, j)) * rso - q.wo - q.wo * dso * rso;
            q.xg += ap * dxg; q.xi += ap * dxi; q.xo += ap * dxo; q.xe += ap * dxe; q.xp += ap * dxp; q.xq += ap * dxq;
            q.zg += ad * dzg; q.zi += ad * dzi; q.zo += ad * dzo; q.ze += ad * dze; q.zp += ad * dzp; q.zq += ad * dzq;
            if (has_s) { q.xs += ap * dxs; q.zs += ad * dzs; }
            q.si += ap * dsi; q.so += ap * dso; q.wi += ad * dwi; q.wo += ad * dwo;
            q.y1 += ad * WS(W_F + 0, j); q.y2 += ad * WS(W_F + 1, j); q.y3 += ad * WS(W_SC + 7, j); q.y4 += ad * WS(W_SC + 8, j);
            store_per(q, w, P, j);
        }
    }
    // ---- results
    if (lane == 0) {
        Q.obj[p] = po_last * beta_b * beta_c + kconst;
        Q.status[p] = status;
        Q.iters[p] = it + it0;
    }
    if (Q.x_out) {
        double *xo_ = Q.x_out + p * (long long)Q.n;
        for (int j = 0; j < P; ++j) {
            const int t = t0 + j;
            if (t < T) {
                const int *ci_ = Q.col_idx + (long long)t * 7;
                for (int k = 0; k < 7; ++k)
                    if (ci_[k] >= 0) xo_[ci_[k]] = WS(W_X + k, j) * beta_b;
            }
        }
    }
    if (Q.y_out) {
        double *yo_ = Q.y_out + p * (long long)Q.m;
        for (int j = 0; j < P; ++j) {
            const int t = t0 + j;
            if (t < T) {
                const int *ri_ = Q.row_idx + (long long)t * 4;
                for (int k = 0; k < 4; ++k) yo_[ri_[k]] = WS(W_Y + k, j) * beta_c;
            }
        }
    }
    return status == DSP_OPTIMAL ? 0 : it + it0 + 1;
#undef WS
#undef LSCAL
#undef ACT
#undef HAS_S
#undef Y1N
#undef Y2N
#undef BACK_ALL
#undef SEP_SOLVE
}

// persistent warps: one LP at a time per warp, tickets from a global counter; second attempt as in the other kernels
__device__ void warp_body_long(const LongParams &LQ, int warp_global, int lane) {
    double *wsw = LQ.ws + (size_t)warp_global * NW * LQ.P * 32;
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(LQ.q.ticket, 1ULL);
        t = __shfl_sync(FULL, t, 0);
        if ((long long)t >= LQ.q.N) break;
        int it0 = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            // second attempt: shorter step and a 100x proximal term (the other kernels use 10x).  At T = 8736 the failures are LPs whose
            // normal matrix (cond > 1e15) lets the solve drift along near-null directions: dx = D (A' dy - h) with D = x / z ~ 1e9 turns a
            // 1e-9 error of A' dy into a step of order 1, which the proximal term converts into a dual residual stuck at 1e-7; 1e-6
            // damps that (on the emulator: the one LP in 64 of the full-year sweep that 10x leaves NUMERICAL converges, 43 + 55
            // iterations, objective 4e-12 from the band kernel's; 1000x stalls at MAX_ITER)
            const double sf = attempt ? 0.99 : LQ.q.step_frac, rg = attempt ? 100.0 * LQ.q.reg : LQ.q.reg;
            const int r = solve_long(LQ, wsw, (long long)t, lane, sf, rg, it0);
            if (r == 0) break;
            it0 = r - 1;
        }
    }
}

}  // namespace stage2long
