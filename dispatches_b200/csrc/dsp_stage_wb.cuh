// dsp_stage_wb.cuh -- stage-structured IPM kernel for the wind+battery price-taker LP, T <= 32 periods.
//
// Hot path of BASELINE configs C1/C2/C5: wind_battery_optimize with design_opt=False
// (wind_battery_LMP.py:172-267) in the reduced form of dispatches_b200/templates.py::wind_battery.
//
// Mapping: ONE WARP PER LP, ONE LANE PER PERIOD, STATE IN REGISTERS (no shared memory; ptxas spills ~0.4 KB per thread
// to local memory at the 168-register cap):
//   lane t holds the period's 7 columns  g (grid), i (charge), o (discharge), s (state of charge), e (throughput),
//   p (slack of the SoC bound), q (slack of the wind balance), their duals, the 4 row duals and the Newton data.
//   Neighbouring periods talk through warp shuffles (s[t-1], e[t-1], y1[t+1], y2[t+1]).
// Linear algebra per IPM iteration (numpy mirror: oracle/ipm_stage_numpy.py, MODE="twisted"):
//   * the normal matrix M = A D A' is reduced inside each lane by eliminating the two local rows (wind balance,
//     SoC bound) in the cancellation-free form  d - d^2/m = d (m - d)/m ;
//   * what remains is block tridiagonal in time with 2x2 blocks (dy1, dy2); it is factorised by a block LDL'
//     that eliminates from BOTH ends of the horizon towards the root period r = T/2 ("twisted" order: half the
//     sequential depth of a one-way sweep, same stability as Cholesky), 2 solves per iteration reuse the factor;
//   * Mehrotra predictor-corrector, same scaling / start / stopping rules as the generic kernel.
// HBM traffic per LP: 8T (LMP row) in, 16 B out (+ x, y on request).  FP64 throughout.
#pragma once
#include "dsp_nan_rows.cuh"

namespace stagewb {

struct StageParams {
    int T;
    double a, binv, hf, dl, dur, krev;      // charge eff., 1/discharge eff., 1/2, degradation, duration, cost scale
    int wcf_off, p_off;                     // rparams layout: wind_kw*cf_t at wcf_off+t, battery kW at p_off
    const int *col_idx;                     // [T*7] template column of (t, g/i/o/s/e/p/q) or -1
    const int *row_idx;                     // [T*4] template row of (t, r1..r4)
};

__device__ __forceinline__ double frcp(double x) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    double e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    return r;
}

// max without fmax's NaN bookkeeping (DSETP.MAX + quiet-NaN fix-up costs ~9 SASS instructions per call)
__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }

__device__ __forceinline__ double shfl_src(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ double up1(double v, int lane) {
    double r = __shfl_up_sync(0xffffffffu, v, 1);
    return lane == 0 ? 0.0 : r;
}
__device__ __forceinline__ double down1(double v, int lane) {
    double r = __shfl_down_sync(0xffffffffu, v, 1);
    return lane == 31 ? 0.0 : r;
}
__device__ __forceinline__ double wmax(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = dmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// max over the warp of NON-NEGATIVE doubles with two 32-bit hardware reductions (redux.sync) instead of five
// shuffle levels: for v >= 0 the IEEE bit pattern is monotone, so reduce the high words, then the low words of the
// lanes that hold the maximal high word
__device__ __forceinline__ double wmax_pos(double v) {
    v = v > 0.0 ? v : 0.0;          // negatives and -0.0 would win the unsigned comparison
    const unsigned hi = (unsigned)__double2hiint(v), lo = (unsigned)__double2loint(v);
    const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
    const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
    return __hiloint2double((int)mh, (int)ml);
}
__device__ __forceinline__ double wsum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct Sym2 { double a, b, c; };            // [[a, b], [b, c]]
struct Mat2 { double a, b, c, d; };         // [[a, b], [c, d]]

// inverse of an SPD 2x2 block: adjugate / determinant, one reciprocal (the determinant keeps its accuracy through the
// fused multiply-add; with the proximal regularisation the blocks are far from singular -- checked in the mirror)
__device__ __forceinline__ Sym2 inv_spd(const Sym2 &D) {
    const double i = frcp(fma(D.a, D.c, -(D.b * D.b)));
    Sym2 r;
    r.a = D.c * i;
    r.b = -D.b * i;
    r.c = D.a * i;
    return r;
}
__device__ __forceinline__ Mat2 mul_ss(const Sym2 &A, const Sym2 &B) {      // A * B
    Mat2 r;
    r.a = fma(A.a, B.a, A.b * B.b); r.b = fma(A.a, B.b, A.b * B.c);
    r.c = fma(A.b, B.a, A.c * B.b); r.d = fma(A.b, B.b, A.c * B.c);
    return r;
}
// D -= G * C   (C symmetric; the product is symmetric in exact arithmetic)
__device__ __forceinline__ void sub_gc(Sym2 &D, const Mat2 &G, const Sym2 &C) {
    D.a -= fma(G.a, C.a, G.b * C.b);
    D.b -= fma(G.a, C.b, G.b * C.c);
    D.c -= fma(G.c, C.b, G.d * C.c);
}

struct Factor {          // per-lane pieces of the twisted block LDL'
    Sym2 Dhinv;          // inverse of the eliminated diagonal block
    Mat2 G, G2;          // multipliers towards the outer neighbour(s) (G2: root only)
    Sym2 Cin;            // coupling to the inner neighbour (towards the root)
    int src, fo, bsrc, bo;
    bool is_root;
};

// backward half of the solve: on entry (g1, g2) is the forward-eliminated right-hand side, on exit the solution
__device__ __forceinline__ void tw_back(const Factor &F, double &g1, double &g2, int T, int lane) {
    const int r = T / 2, smax = max(r, T - 1 - r);
    double u1 = 0.0, u2 = 0.0;
    if (F.is_root) {
        u1 = fma(F.Dhinv.a, g1, F.Dhinv.b * g2);
        u2 = fma(F.Dhinv.b, g1, F.Dhinv.c * g2);
    }
#pragma unroll 1
    for (int s = 1; s <= smax; ++s) {
        const double r1 = shfl_src(u1, F.bsrc), r2 = shfl_src(u2, F.bsrc);
        if (F.bo == s) {
            const double t1 = g1 - fma(F.Cin.a, r1, F.Cin.b * r2);
            const double t2 = g2 - fma(F.Cin.b, r1, F.Cin.c * r2);
            u1 = fma(F.Dhinv.a, t1, F.Dhinv.b * t2);
            u2 = fma(F.Dhinv.b, t1, F.Dhinv.c * t2);
        }
    }
    g1 = u1; g2 = u2;
}

__device__ __forceinline__ void tw_solve(const Factor &F, double &g1, double &g2, int T, int lane) {
    const int r = T / 2, kmax = max(r - 1, T - 2 - r);
#pragma unroll 1
    for (int k = 1; k <= kmax; ++k) {
        const double r1 = shfl_src(g1, F.src), r2 = shfl_src(g2, F.src);
        if (F.fo == k) {
            g1 -= fma(F.G.a, r1, F.G.b * r2);
            g2 -= fma(F.G.c, r1, F.G.d * r2);
        }
    }
    {
        const double a1 = shfl_src(g1, max(r - 1, 0)), a2 = shfl_src(g2, max(r - 1, 0));
        const double b1 = shfl_src(g1, min(r + 1, 31)), b2 = shfl_src(g2, min(r + 1, 31));
        if (F.is_root) {
            if (r >= 1) { g1 -= fma(F.G.a, a1, F.G.b * a2); g2 -= fma(F.G.c, a1, F.G.d * a2); }
            if (r + 1 <= T - 1) { g1 -= fma(F.G2.a, b1, F.G2.b * b2); g2 -= fma(F.G2.c, b1, F.G2.d * b2); }
        }
    }
    tw_back(F, g1, g2, T, lane);
}

struct Out {
    double *obj, *x_out, *y_out;
    int *status, *iters;
    int n, m;
};

// solves LP number p; all 32 lanes of the warp participate.  The sweep loops are deliberately NOT unrolled and the horizon
// is a run-time value: the iteration body is ~3k instructions, and a T=24 instantiation with unrolled sweeps (7k) ran
// slower, limited by instruction-cache misses
__device__ int solve_one(const StageParams &S, const double *cp, const double *rpar, double kconst, long long p,
                          double tol, double feas_tol, double step_frac, double reg, int max_iter, const Out &O, int lane, int it0) {
    const int T = S.T;
    const bool act = lane < T, has_s = lane < T - 1;
    const double a = S.a, binv = S.binv, hf = S.hf, dl = S.dl;
    // ---- problem data of this period
    const double lam = act ? cp[lane] : 0.0;
    const double wcf = act ? rpar[S.wcf_off + lane] : 0.0;
    const double P = rpar[S.p_off];
    double c = S.krev * lam;
    double b3 = S.dur * P, b4 = wcf;
    const double b4max = wmax_pos(fabs(b4));
    double beta_b = dmax(dmax(fabs(b3), b4max), P);
    beta_b = beta_b > 0.0 ? beta_b : 1.0;
    if (P < -1e-9 * beta_b) {       // negative battery power bound beyond rounding: infeasible (the band kernel's rule)
        if (lane == 0) { O.obj[p] = __longlong_as_double(0x7ff8000000000000LL); O.status[p] = DSP_INFEASIBLE; O.iters[p] = it0; }
        dsp_nan_rows(O.x_out, O.n, O.y_out, O.m, p, lane, 32);
        return 0;
    }
    const double cmax = wmax_pos(fabs(c));
    const double beta_c = cmax > 0.0 ? cmax : 1.0;
    c = c / beta_c; b3 = b3 / beta_b; b4 = b4 / beta_b;
    const double u = dmax(P / beta_b, 1e-10);
    const double nrm_b = 1.0 + dmax(fabs(b3), b4max / beta_b), nrm_c = 1.0 + (cmax > 0.0 ? 1.0 : 0.0);
    const double ntot = (double)(9 * T - 1);
    // ---- start point
    double xg = 1.0, xi = fmin(1.0, 0.5 * u), xo = xi, xs = has_s ? 1.0 : 0.0, xe = 1.0, xp = 1.0, xq = 1.0;
    double zg = 1.0, zi = 1.0, zo = 1.0, zs = has_s ? 1.0 : 0.0, ze = 1.0, zp = 1.0, zq = 1.0;
    double si = u - xi, so = u - xo, wi = 1.0, wo = 1.0;
    double y1 = 0.0, y2 = 0.0, y3 = 0.0, y4 = 0.0;
    // ---- twisted elimination order
    Factor F;
    const int rt = T / 2, kmax = max(rt - 1, T - 2 - rt);
    F.is_root = (lane == rt);
    F.src = min(max(lane < rt ? lane - 1 : lane + 1, 0), 31);
    F.fo = (!act || F.is_root) ? 1 << 20 : (lane < rt ? lane : T - 1 - lane);
    F.bsrc = min(max(lane < rt ? lane + 1 : lane - 1, 0), 31);
    F.bo = (!act || F.is_root) ? 1 << 20 : abs(lane - rt);

    int status = DSP_MAX_ITER, it = 0;
    double pobj = 0.0;
    PH_INIT
    for (it = 0; it <= max_iter; ++it) {
        PH(15);
        // ---- residuals
        const double xs_p = up1(xs, lane), xe_p = up1(xe, lane);
        const double y1n = down1(y1, lane), y2n = down1(y2, lane);
        double rp1 = -(xs - xs_p - a * xi + binv * xo);
        double rp2 = -(xe - xe_p - hf * xi - hf * xo);
        double rp3 = b3 - (xs + dl * xe + xp);
        double rp4 = b4 - (xg + xi + xq);
        double rdg = c - y4 - zg;
        double rdi = a * y1 + hf * y2 - y4 - zi + wi;
        double rdo = c - binv * y1 + hf * y2 - zo + wo;
        double rds = has_s ? -(y1 - y1n + y3) - zs : 0.0;
        double rde = -(y2 - y2n + dl * y3) - ze;
        double rdp = -y3 - zp, rdq = -y4 - zq;
        double rui = u - xi - si, ruo = u - xo - so;
        double pm = 0.0, dm = 0.0, mus = 0.0, po = 0.0, dob = 0.0;
        if (act) {
            pm = dmax(dmax(dmax(fabs(rp1), fabs(rp2)), dmax(fabs(rp3), fabs(rp4))), dmax(fabs(rui), fabs(ruo)));
            dm = dmax(dmax(dmax(fabs(rdg), fabs(rdi)), dmax(fabs(rdo), fabs(rds))), dmax(dmax(fabs(rde), fabs(rdp)), fabs(rdq)));
            mus = xg * zg + xi * zi + xo * zo + xs * zs + xe * ze + xp * zp + xq * zq + si * wi + so * wo;
            po = c * (xg + xo);
            dob = b3 * y3 + b4 * y4 - u * (wi + wo);
        } else {
            rp1 = rp2 = rp3 = rp4 = rdg = rdi = rdo = rds = rde = rdp = rdq = rui = ruo = 0.0;
        }
        const double res = wmax_pos(dmax(pm / nrm_b, dm / nrm_c));
        mus = wsum(mus); po = wsum(po); dob = wsum(dob);
        pobj = po;
        const double mu = mus / ntot;
        const double den = dmax(kGapFloor, fabs(po));
        const double gap = fabs(po - dob) / den, cgap = ntot * mu / den;
        if (!(mu == mu) || !(po == po) || mu > 1e100) { status = DSP_NUMERICAL; break; }
        if (res < feas_tol && gap < tol) { status = DSP_OPTIMAL; break; }
        if (cgap < tol && res < 10.0 * feas_tol && gap < 10.0 * tol) { status = DSP_OPTIMAL; break; }
        if (cgap < 1e-3 * tol) {
            status = (res < 100.0 * feas_tol && gap < 1000.0 * tol) ? DSP_OPTIMAL : DSP_NUMERICAL;
            break;
        }
        if (it == max_iter) break;
        PH(8);
        // ---- scaling matrix D and reciprocals
        const double rxg = frcp(xg), rxi = frcp(xi), rxo = frcp(xo), rxe = frcp(xe), rxp = frcp(xp), rxq = frcp(xq);
        const double rxs = has_s ? frcp(xs) : 0.0;
        const double rsi = frcp(si), rso = frcp(so);
        const double rzg = frcp(zg), rze = frcp(ze), rzp = frcp(zp), rzq = frcp(zq), rzs = has_s ? frcp(zs) : 0.0;
        const double rzi = frcp(zi), rzo = frcp(zo), rwi = frcp(wi), rwo = frcp(wo);
        // d = 1 / (z/x [+ w/s] + reg / max(1, x^2)): the proximal term caps d for columns that never approach a bound;
        // dividing by x^2 for x > 1 keeps it scale invariant (the throughput column grows with the horizon)
        const double qg = xg > 1.0 ? reg * rxg * rxg : reg, qe = xe > 1.0 ? reg * rxe * rxe : reg;
        const double qp = xp > 1.0 ? reg * rxp * rxp : reg, qq = xq > 1.0 ? reg * rxq * rxq : reg;
        const double qs = xs > 1.0 ? reg * rxs * rxs : reg;
        const double dg = xg * frcp(fma(qg, xg, zg)), de = xe * frcp(fma(qe, xe, ze));
        const double dp = xp * frcp(fma(qp, xp, zp)), dq = xq * frcp(fma(qq, xq, zq));
        const double ds = has_s ? xs * frcp(fma(qs, xs, zs)) : 0.0;
        const double di = frcp(fma(zi, rxi, wi * rsi) + reg), dO = frcp(fma(zo, rxo, wo * rso) + reg);   // x_i, x_o <= u <= 1
        // ---- per-period blocks after eliminating the wind-balance and SoC-bound rows (cancellation-free)
        const double kap = frcp(ds + dl * dl * de + dp);
        const double s11 = ds * (dl * dl * de + dp) * kap;
        const double s22 = de * (ds + dp) * kap;
        const double s12 = dl * ds * de * kap;
        const double iot = frcp(dg + di + dq);
        const double tau = di * (dg + dq) * iot;
        const double s11p = up1(s11, lane), s22p = up1(s22, lane), s12p = up1(s12, lane);
        Sym2 D;
        D.a = s11 + s11p + a * a * tau + binv * binv * dO;
        D.c = s22 + s22p + hf * hf * (tau + dO);
        D.b = a * hf * tau - hf * binv * dO - s12 - s12p;
        Sym2 Bn, Bp;                       // coupling with t+1 (own) and with t-1 (the previous lane's)
        Bn.a = (lane < T - 1) ? -s11 : 0.0; Bn.c = (lane < T - 1) ? -s22 : 0.0; Bn.b = (lane < T - 1) ? s12 : 0.0;
        Bp.a = -s11p; Bp.c = -s22p; Bp.b = s12p;
        if (!act) { D.a = 1.0; D.b = 0.0; D.c = 1.0; }
        const Sym2 Cout = (lane < rt) ? Bp : Bn;
        F.Cin = (lane < rt) ? Bn : Bp;
        const double dsk = ds * kap, dek = dl * de * kap, dii = di * iot;
        // ---- Newton right-hand side for complementarity targets ax (x z -> ax), as (s w -> as)
        double dxg, dxi, dxo, dxs, dxe, dxp, dxq, dy1, dy2, dy3, dy4;
        double cg = 0, ci = 0, co = 0, cs = 0, ce = 0, cpp = 0, cq = 0, csi = 0, cso = 0;   // predictor products
        double smu = 0.0;
        double hg, hi, ho, hs, he, hp, hq, w3, w4;
        auto make_rhs = [&](bool corr, double &f1, double &f2) {
            hg = rdg + zg; hi = rdi + zi; ho = rdo + zo; hs = rds + zs; he = rde + ze; hp = rdp + zp; hq = rdq + zq;
            double asi = -wi * rui, aso = -wo * ruo;
            if (corr) {
                hg -= (smu - cg) * rxg; hi -= (smu - ci) * rxi; ho -= (smu - co) * rxo; hs -= (smu - cs) * rxs;
                he -= (smu - ce) * rxe; hp -= (smu - cpp) * rxp; hq -= (smu - cq) * rxq;
                asi += smu - csi; aso += smu - cso;
            }
            hi += asi * rsi - wi; ho += aso * rso - wo;
            if (!has_s) hs = 0.0;
            w3 = rp3 + dp * hp;
            const double ph1 = s11 * hs - s12 * he - dsk * w3;
            const double ph2 = s22 * he - s12 * hs - dek * w3;
            w4 = rp4 + dg * hg + dq * hq;
            const double psi = tau * hi - dii * w4;
            const double doh = dO * ho;
            f1 = rp1 + ph1 - up1(ph1, lane) - a * psi + binv * doh;
            f2 = rp2 + ph2 - up1(ph2, lane) - hf * psi - hf * doh;
            if (!act) { f1 = 0.0; f2 = 0.0; }
        };
        auto recover = [&](double u1, double u2) {
            dy1 = u1; dy2 = u2;
            const double e1 = dy1 - down1(dy1, lane) - hs, e2 = dy2 - down1(dy2, lane) - he;
            const double v = a * dy1 + hf * dy2;
            dxs = has_s ? s11 * e1 - s12 * e2 + dsk * w3 : 0.0;
            dxe = s22 * e2 - s12 * e1 + dek * w3;
            dxi = -tau * (v + hi) + dii * w4;
            dxo = dO * (binv * dy1 - hf * dy2 - ho);
            dxg = dg * iot * (rp4 + di * (hi - hg + v) + dq * (hq - hg));
            dy3 = kap * (w3 - ds * e1 - dl * de * e2);
            dy4 = iot * (w4 + di * (hi + v));
            dxp = dp * (dy3 - hp);
            dxq = dq * (dy4 - hq);
        };
        // ---- twisted block LDL'; the forward elimination of the PREDICTOR right-hand side rides along in the same
        // ---- sweep (its shuffles and FMAs fill the latency shadow of the 2x2 inversions)
        PH(9);
        double g1, g2;
        make_rhs(false, g1, g2);
        PH(10);
        Sym2 Dh = D;
        // deferred reciprocal: the lanes pass the eliminated block Dh itself; the receiver forms Cout adj(R) Cout' while
        // the reciprocal of det(R) is in flight, so the dependent chain per step is  shfl -> det -> rcp -> fma
        F.G.a = F.G.b = F.G.c = F.G.d = 0.0;
        F.G2 = F.G;
#pragma unroll 1
        for (int k = 1; k <= kmax; ++k) {
            Sym2 R;
            R.a = shfl_src(Dh.a, F.src); R.b = shfl_src(Dh.b, F.src); R.c = shfl_src(Dh.c, F.src);
            const double q1 = shfl_src(g1, F.src), q2 = shfl_src(g2, F.src);
            if (F.fo == k) {
                const double rd = frcp(fma(R.a, R.c, -(R.b * R.b)));
                Sym2 adj; adj.a = R.c; adj.b = -R.b; adj.c = R.a;
                const Mat2 X = mul_ss(Cout, adj);
                const double ya = fma(X.a, Cout.a, X.b * Cout.b), yb = fma(X.a, Cout.b, X.b * Cout.c), yc = fma(X.c, Cout.b, X.d * Cout.c);
                const double t1 = fma(X.a, q1, X.b * q2), t2 = fma(X.c, q1, X.d * q2);
                Dh.a = fma(-ya, rd, Dh.a); Dh.b = fma(-yb, rd, Dh.b); Dh.c = fma(-yc, rd, Dh.c);
                g1 = fma(-t1, rd, g1); g2 = fma(-t2, rd, g2);
                F.G.a = X.a * rd; F.G.b = X.b * rd; F.G.c = X.c * rd; F.G.d = X.d * rd;
            }
        }
        {
            Sym2 Ra, Rb;
            const int la = max(rt - 1, 0), lb = min(rt + 1, 31);
            Ra.a = shfl_src(Dh.a, la); Ra.b = shfl_src(Dh.b, la); Ra.c = shfl_src(Dh.c, la);
            Rb.a = shfl_src(Dh.a, lb); Rb.b = shfl_src(Dh.b, lb); Rb.c = shfl_src(Dh.c, lb);
            const double a1 = shfl_src(g1, la), a2 = shfl_src(g2, la), b1 = shfl_src(g1, lb), b2 = shfl_src(g2, lb);
            if (F.is_root) {
                if (rt >= 1) {
                    F.G = mul_ss(Bp, inv_spd(Ra)); sub_gc(Dh, F.G, Bp);
                    g1 -= fma(F.G.a, a1, F.G.b * a2); g2 -= fma(F.G.c, a1, F.G.d * a2);
                }
                if (rt + 1 <= T - 1) {
                    F.G2 = mul_ss(Bn, inv_spd(Rb)); sub_gc(Dh, F.G2, Bn);
                    g1 -= fma(F.G2.a, b1, F.G2.b * b2); g2 -= fma(F.G2.c, b1, F.G2.d * b2);
                }
            }
        }
        F.Dhinv = inv_spd(Dh);
        PH(11);
        // ---- affine predictor: backward sweep only
        tw_back(F, g1, g2, T, lane);
        PH(12);
        recover(g1, g2);
        // dz = ax/x - z - z dx / x ;  dw = as/s - w - w ds / s
        double dzg = -zg - zg * dxg * rxg, dzi = -zi - zi * dxi * rxi, dzo = -zo - zo * dxo * rxo;
        double dzs = has_s ? -zs - zs * dxs * rxs : 0.0, dze = -ze - ze * dxe * rxe, dzp = -zp - zp * dxp * rxp;
        double dzq = -zq - zq * dxq * rxq;
        double dsi = rui - dxi, dso = ruo - dxo;
        double dwi = -wi - wi * dsi * rsi, dwo = -wo - wo * dso * rso;
        double ip = 0.0, id = 0.0;             // 1/alpha
        if (act) {
            ip = dmax(dmax(dmax(-dxg * rxg, -dxi * rxi), dmax(-dxo * rxo, -dxs * rxs)), dmax(dmax(-dxe * rxe, -dxp * rxp), -dxq * rxq));
            ip = dmax(ip, dmax(-dsi * rsi, -dso * rso));
            id = dmax(dmax(dmax(-dzg * rzg, -dzi * rzi), dmax(-dzo * rzo, -dzs * rzs)), dmax(dmax(-dze * rze, -dzp * rzp), -dzq * rzq));
            id = dmax(id, dmax(-dwi * rwi, -dwo * rwo));
        }
        ip = wmax_pos(ip); id = wmax_pos(id);
        double ap = ip > 1.0 ? 1.0 / ip : 1.0, ad = id > 1.0 ? 1.0 / id : 1.0;
        double mua = 0.0;
        if (act) {
            mua = (xg + ap * dxg) * (zg + ad * dzg) + (xi + ap * dxi) * (zi + ad * dzi) + (xo + ap * dxo) * (zo + ad * dzo)
                + (xs + ap * dxs) * (zs + ad * dzs) + (xe + ap * dxe) * (ze + ad * dze) + (xp + ap * dxp) * (zp + ad * dzp)
                + (xq + ap * dxq) * (zq + ad * dzq) + (si + ap * dsi) * (wi + ad * dwi) + (so + ap * dso) * (wo + ad * dwo);
        }
        mua = wsum(mua) / ntot;
        cg = dxg * dzg; ci = dxi * dzi; co = dxo * dzo; cs = dxs * dzs; ce = dxe * dze; cpp = dxp * dzp; cq = dxq * dzq;
        csi = dsi * dwi; cso = dso * dwo;
        const double sg = mua / mu;
        smu = sg * sg * sg * mu;
        PH(13);
        // ---- corrector
        make_rhs(true, g1, g2);
        tw_solve(F, g1, g2, T, lane);
        PH(14);
        recover(g1, g2);
        dzg = (smu - cg) * rxg - zg - zg * dxg * rxg; dzi = (smu - ci) * rxi - zi - zi * dxi * rxi;
        dzo = (smu - co) * rxo - zo - zo * dxo * rxo; dzs = has_s ? (smu - cs) * rxs - zs - zs * dxs * rxs : 0.0;
        dze = (smu - ce) * rxe - ze - ze * dxe * rxe; dzp = (smu - cpp) * rxp - zp - zp * dxp * rxp;
        dzq = (smu - cq) * rxq - zq - zq * dxq * rxq;
        dsi = rui - dxi; dso = ruo - dxo;
        dwi = (smu - csi) * rsi - wi - wi * dsi * rsi; dwo = (smu - cso) * rso - wo - wo * dso * rso;
        ip = 0.0; id = 0.0;
        if (act) {
            ip = dmax(dmax(dmax(-dxg * rxg, -dxi * rxi), dmax(-dxo * rxo, -dxs * rxs)), dmax(dmax(-dxe * rxe, -dxp * rxp), -dxq * rxq));
            ip = dmax(ip, dmax(-dsi * rsi, -dso * rso));
            id = dmax(dmax(dmax(-dzg * rzg, -dzi * rzi), dmax(-dzo * rzo, -dzs * rzs)), dmax(dmax(-dze * rze, -dzp * rzp), -dzq * rzq));
            id = dmax(id, dmax(-dwi * rwi, -dwo * rwo));
        }
        ip = wmax_pos(ip); id = wmax_pos(id);
        ap = (step_frac * 1.0 < ip) ? step_frac / ip : 1.0;     // min(1, step_frac / ip)
        ad = (step_frac * 1.0 < id) ? step_frac / id : 1.0;
        if (act) {
            xg += ap * dxg; xi += ap * dxi; xo += ap * dxo; xe += ap * dxe; xp += ap * dxp; xq += ap * dxq;
            zg += ad * dzg; zi += ad * dzi; zo += ad * dzo; ze += ad * dze; zp += ad * dzp; zq += ad * dzq;
            if (has_s) { xs += ap * dxs; zs += ad * dzs; }
            si += ap * dsi; so += ap * dso; wi += ad * dwi; wo += ad * dwo;
            y1 += ad * dy1; y2 += ad * dy2; y3 += ad * dy3; y4 += ad * dy4;
        }
    }
    // ---- results
    if (lane == 0) {
        O.obj[p] = pobj * beta_b * beta_c + kconst;
        O.status[p] = status;
        O.iters[p] = it + it0;
    }
    if (O.x_out && act) {
        double *xo_ = O.x_out + p * (long long)O.n;
        const int *ci_ = S.col_idx + lane * 7;
        const double vals[7] = {xg, xi, xo, xs, xe, xp, xq};
#pragma unroll
        for (int k = 0; k < 7; ++k)
            if (ci_[k] >= 0) xo_[ci_[k]] = vals[k] * beta_b;
    }
    if (O.y_out && act) {
        double *yo_ = O.y_out + p * (long long)O.m;
        const int *ri_ = S.row_idx + lane * 4;
        yo_[ri_[0]] = y1 * beta_c; yo_[ri_[1]] = y2 * beta_c; yo_[ri_[2]] = y3 * beta_c; yo_[ri_[3]] = y4 * beta_c;
    }
    return status == DSP_OPTIMAL ? 0 : it + it0 + 1;
}

}  // namespace stagewb
