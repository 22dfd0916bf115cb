// dsp_band_split.cuh -- partitioned band LDL' of the split band kernel `dsp_ipm_band_split_kernel<W>` (DSP_KERNEL_BAND_SPLIT).
//
// One warp per LP, everything in a per-warp region of a global workspace laid out [array][slot][lane]: the template's rows, in band
// order, are cut into 32 contiguous chunks, chunk L (rows base*L + min(L, rem) ..., base = m / 32, rem = m % 32) owned by lane L, row
// slot s of lane L at index s * 32 + L of every row vector.  Every access of the warp to slot s is one coalesced line.
//
// Factorisation: a scalar LDL' of P M P' for a fixed permutation P -- a nested dissection of the band.  The last W rows of chunks
// 0..30 are separators S_0..S_30, the other rows interiors I_0..I_31.  Order: every interior (ascending), then S_0..S_14, then
// S_30..S_16, then S_15 (the separator chain eliminated from both ends, meeting in the middle).
//   * interiors: each lane eliminates I_L in Cholesky order with the band kernel's pivot rule (1/d = 0 for d <= 0, reciprocal by
//     frcpd).  Column i of L has its band entries (rows i+1..i+W of the chunk, S_L included) and a W-column spike G towards the
//     previous lane's separator S_{L-1} (rows of I_L only couple to S_{L-1} through the band for the first W rows of the chunk; the
//     elimination fills the rest).  The Schur update of S_{L-1}'s diagonal block is accumulated in E (lane L) and added after.
//   * separators: the 31 W x W diagonal blocks D_k (S_k rows' band entries inside S_k) and off-diagonal blocks C_k (rows S_k,
//     columns S_{k-1}: the spike of S_k's rows) form a block-tridiagonal system, eliminated with scalar pivots, 16 steps, the W x W
//     updates of a pivot spread over the 32 lanes.  No explicitly inverted pivot block (dsp_stage2_long.cuh: they lose convergence
//     at long horizons).
// Storage after the factorisation: band slot 0 holds 1/d, the other band slots, G and C hold UNSCALED entries L * d (dsp_band.cuh).
// The substitutions follow the same order: lanes in parallel on their interiors, the separator chain, the interiors again.
//
// Needs every chunk to hold at least 2W rows (m >= 64 W), so that two separators never touch.  Numpy mirror:
// oracle/ipm_band_split_numpy.py.  Plain C++ over warp builtins down to split_solve: tests/emu compiles it with g++ on the SIMT
// emulator.
#pragma once

namespace bsplit {

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define BSD __device__ __forceinline__
#else
#define BSD inline
#endif

BSD double frcp(double x) {          // band::frcpd
    double r;
#if defined(__CUDA_ARCH__)
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#else
    r = (double)(1.0f / (float)x);
    if (!(r == r) || r == 0.0 || r > 1e300 || r < -1e300) r = 1.0 / x;
#endif
    double e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    e = fma(-x, r, 1.0);
    return fma(r, e, r);
}

// workspace of the factor: band (W+1 arrays of Sr slots), spike (W arrays of Sr slots), E (W*W arrays of one slot), the meeting
// scratch X (W*W + W doubles, shared by the warp)
template <int W>
struct Factor {
    double *Mb, *G, *E, *X;
    int Sr, m;
    BSD double &mb(int k, int s, int L) const { return Mb[((size_t)k * Sr + s) * 32 + L]; }
    BSD double &g(int k, int s, int L) const { return G[((size_t)k * Sr + s) * 32 + L]; }
    BSD double &e(int a, int b, int L) const { return E[(a * W + b) * 32 + L]; }
    BSD int rows(int L) const { return (m >> 5) + (L < (m & 31) ? 1 : 0); }
    // separator block k: D(a, b) = M[S_k a][S_k b] (a >= b), C(a, b) = M[S_k a][S_{k-1} b]
    BSD double &D(int k, int a, int b) const { return mb(a - b, rows(k) - W + a, k); }
    BSD double &C(int k, int a, int b) const { return g(b, rows(k) - W + a, k); }
};
template <int W>
constexpr long long factor_doubles(int Sr) { return (long long)(2 * W + 1) * Sr * 32 + W * W * 32 + W * W + W; }

// M = P' L D L' P in place.  On entry F.Mb holds the band of M in split layout: mb(k, s, L) = M[i][i-k] for row i = slot s of lane
// L (entries with i-k < 0 zero).
template <int W>
BSD void split_factor(const Factor<W> &F, int lane) {
    const int cs = F.rows(lane);
    const int ni = lane < 31 ? cs - W : cs;
    // the band entries of the first W rows that reach into the previous chunk (S_{lane-1}) start the spike
    for (int s = 0; s < cs; ++s)
        for (int k = 0; k < W; ++k) F.g(k, s, lane) = (lane > 0 && s < W && k >= s) ? F.mb(s + W - k, s, lane) : 0.0;
    for (int a = 0; a < W * W; ++a) F.E[a * 32 + lane] = 0.0;
    for (int a = lane; a < W * W + W; a += 32) F.X[a] = 0.0;
    // ---- interiors, every lane on its own chunk
    for (int j = 0; j < ni; ++j) {
        const double piv = F.mb(0, j, lane);
        const double inv = piv > 0.0 ? frcp(piv) : 0.0;
        double l[W], gj[W];
#pragma unroll
        for (int r = 1; r <= W; ++r) l[r - 1] = j + r < cs ? F.mb(r, j + r, lane) : 0.0;
#pragma unroll
        for (int k = 0; k < W; ++k) gj[k] = F.g(k, j, lane);
#pragma unroll
        for (int r = 1; r <= W; ++r) {
            if (j + r >= cs) break;
            const double lr = l[r - 1];
#pragma unroll
            for (int q = 1; q <= r; ++q) F.mb(r - q, j + r, lane) -= lr * l[q - 1] * inv;
#pragma unroll
            for (int k = 0; k < W; ++k) F.g(k, j + r, lane) -= lr * gj[k] * inv;
        }
#pragma unroll
        for (int a = 0; a < W; ++a)
#pragma unroll
            for (int b = 0; b <= a; ++b) F.e(a, b, lane) -= gj[a] * gj[b] * inv;
        F.mb(0, j, lane) = inv;
    }
    __syncwarp();
    // S_k's diagonal block gets the Schur update of I_{k+1}
    if (lane < 31)
        for (int a = 0; a < W; ++a)
            for (int b = 0; b <= a; ++b) F.D(lane, a, b) += F.e(a, b, lane + 1);
    __syncwarp();
    // ---- separator chain: step t eliminates S_t (forward side) and S_{30-t} (backward side), pivot by pivot
    double *X = F.X;           // the backward side's update of D_15 at step 14 (the forward side writes D_15 in the same step)
    for (int t = 0; t < 15; ++t) {
        const int f = t, h = 30 - t;
        for (int p = 0; p < W; ++p) {
            const double pf = F.D(f, p, p), ph = F.D(h, p, p);
            const double invf = pf > 0.0 ? frcp(pf) : 0.0, invh = ph > 0.0 ? frcp(ph) : 0.0;
            for (int it = lane; it < 6 * W * W; it += 32) {
                const int grp = it / (W * W), a = (it / W) % W, b = it % W;
                switch (grp) {
                    case 0: if (b > p && a >= b) F.D(f, a, b) -= F.D(f, a, p) * F.D(f, b, p) * invf; break;
                    case 1: if (b > p) F.C(f + 1, a, b) -= F.C(f + 1, a, p) * F.D(f, b, p) * invf; break;
                    case 2: if (a >= b) F.D(f + 1, a, b) -= F.C(f + 1, a, p) * F.C(f + 1, b, p) * invf; break;
                    case 3: if (b > p && a >= b) F.D(h, a, b) -= F.D(h, a, p) * F.D(h, b, p) * invh; break;
                    case 4: if (a > p) F.C(h, a, b) -= F.D(h, a, p) * F.C(h, p, b) * invh; break;
                    default:
                        if (a >= b) {
                            const double u = F.C(h, p, a) * F.C(h, p, b) * invh;
                            if (h == 16) X[a * W + b] -= u; else F.D(h - 1, a, b) -= u;
                        }
                }
            }
            __syncwarp();
            if (lane == 0) { F.D(f, p, p) = invf; F.D(h, p, p) = invh; }
        }
    }
    __syncwarp();
    for (int it = lane; it < W * W; it += 32) {
        const int a = it / W, b = it % W;
        if (a >= b) F.D(15, a, b) += X[it];
    }
    __syncwarp();
    for (int p = 0; p < W; ++p) {              // the middle block
        const double pm = F.D(15, p, p);
        const double invm = pm > 0.0 ? frcp(pm) : 0.0;
        for (int it = lane; it < W * W; it += 32) {
            const int a = it / W, b = it % W;
            if (b > p && a >= b) F.D(15, a, b) -= F.D(15, a, p) * F.D(15, b, p) * invm;
        }
        __syncwarp();
        if (lane == 0) F.D(15, p, p) = invm;
    }
    __syncwarp();
}

// solve M v = r in place (v in split layout: v[s * 32 + L]) with the factor of split_factor
template <int W>
BSD void split_solve(const Factor<W> &F, double *v, int lane) {
    const int cs = F.rows(lane);
    const int ni = lane < 31 ? cs - W : cs;
    const int csp = lane > 0 ? F.rows(lane - 1) : 0;
#define VS(k, a) v[(F.rows(k) - W + (a)) * 32 + (k)]
    // ---- forward, interiors: the spike's contributions to S_{lane-1} collect in registers
    double acc[W];
#pragma unroll
    for (int k = 0; k < W; ++k) acc[k] = 0.0;
    for (int j = 0; j < ni; ++j) {
        const double t = v[j * 32 + lane] * F.mb(0, j, lane);
#pragma unroll
        for (int r = 1; r <= W; ++r)
            if (j + r < cs) v[(j + r) * 32 + lane] -= F.mb(r, j + r, lane) * t;
        if (lane > 0) {
#pragma unroll
            for (int k = 0; k < W; ++k) acc[k] -= F.g(k, j, lane) * t;
        }
    }
    __syncwarp();
    if (lane > 0) {
#pragma unroll
        for (int k = 0; k < W; ++k) v[(csp - W + k) * 32 + lane - 1] += acc[k];
    }
    double *xv = F.X + W * W;
    for (int k = lane; k < W; k += 32) xv[k] = 0.0;
    __syncwarp();
    // ---- forward, separator chain
    for (int t = 0; t < 15; ++t) {
        const int f = t, h = 30 - t;
        for (int p = 0; p < W; ++p) {
            const double tf = VS(f, p) * F.D(f, p, p), th = VS(h, p) * F.D(h, p, p);
            for (int it = lane; it < 4 * W; it += 32) {
                const int grp = it / W, a = it % W;
                switch (grp) {
                    case 0: if (a > p) VS(f, a) -= F.D(f, a, p) * tf; break;
                    case 1: VS(f + 1, a) -= F.C(f + 1, a, p) * tf; break;
                    case 2: if (a > p) VS(h, a) -= F.D(h, a, p) * th; break;
                    default: {
                        const double u = F.C(h, p, a) * th;
                        if (h == 16) xv[a] -= u; else VS(h - 1, a) -= u;
                    }
                }
            }
            __syncwarp();
        }
    }
    for (int a = lane; a < W; a += 32) VS(15, a) += xv[a];
    __syncwarp();
    for (int p = 0; p < W; ++p) {
        const double tm = VS(15, p) * F.D(15, p, p);
        for (int a = p + 1 + lane; a < W; a += 32) VS(15, a) -= F.D(15, a, p) * tm;
        __syncwarp();
    }
    // ---- diagonal
    for (int s = 0; s < cs; ++s) v[s * 32 + lane] *= F.mb(0, s, lane);
    __syncwarp();
    // ---- backward, separator chain: the middle block, then S_{15-j} and S_{15+j} outwards
    for (int a = W - 1; a > 0; --a) {
        const double va = VS(15, a);
        for (int p = lane; p < a; p += 32) VS(15, p) -= F.D(15, p, p) * F.D(15, a, p) * va;
        __syncwarp();
    }
    for (int j = 1; j <= 15; ++j) {
        const int f = 15 - j, h = 15 + j;
        for (int it = lane; it < 2 * W; it += 32) {       // the already solved neighbour block
            const int p = it % W;
            double s = 0.0;
            if (it < W) {
                for (int a = 0; a < W; ++a) s += F.C(f + 1, a, p) * VS(f + 1, a);
                VS(f, p) -= F.D(f, p, p) * s;
            } else {
                for (int b = 0; b < W; ++b) s += F.C(h, p, b) * VS(h - 1, b);
                VS(h, p) -= F.D(h, p, p) * s;
            }
        }
        __syncwarp();
        for (int a = W - 1; a > 0; --a) {
            const double vf = VS(f, a), vh = VS(h, a);
            for (int it = lane; it < 2 * a; it += 32) {
                if (it < a) VS(f, it) -= F.D(f, it, it) * F.D(f, a, it) * vf;
                else VS(h, it - a) -= F.D(h, it - a, it - a) * F.D(h, a, it - a) * vh;
            }
            __syncwarp();
        }
    }
    // ---- backward, interiors
    double sp[W];
#pragma unroll
    for (int k = 0; k < W; ++k) sp[k] = lane > 0 ? v[(csp - W + k) * 32 + lane - 1] : 0.0;
    for (int j = ni - 1; j >= 0; --j) {
        double s = 0.0;
#pragma unroll
        for (int r = 1; r <= W; ++r)
            if (j + r < cs) s += F.mb(r, j + r, lane) * v[(j + r) * 32 + lane];
        if (lane > 0) {
#pragma unroll
            for (int k = 0; k < W; ++k) s += F.g(k, j, lane) * sp[k];
        }
        v[j * 32 + lane] -= F.mb(0, j, lane) * s;
    }
    __syncwarp();
#undef VS
}

#undef BSD
}  // namespace bsplit

#if defined(__CUDACC__)
// ======================================================================================================================================
// The kernel (included by dsp_lp.cu after the band kernel: KParams, warp reductions, frcpd).  One attempt on LP p runs the band
// kernel's solve_one -- same scaling, start point, proximal term, stopping rule, INFEASIBLE bound rule and results -- over a copy of the
// template renumbered to the split layout: row slot s of lane L is split row s * 32 + L; a column goes to the lane that owns the first
// row it appears in (ascending template order within a lane), column slot s of lane L is split column s * 32 + L.  So an element-wise
// pass is every lane walking its own slots in step, and a CSR product reads another lane's entries only at chunk edges.
// ======================================================================================================================================
struct SplitParams {
    int Sr, Sc;                                  // row / column slots per lane
    const int *ccnt;                             // columns of every lane [32]
    const int *cnat;                             // template column of split column j (-1: padding)
    const int *A_ptr, *A_idx, *At_ptr, *At_idx, *asm_ptr, *asm_col;     // split-layout CSR, CSC and band assembly list
    const double *A_val, *At_val, *asm_val;
    double *ws;                                  // per-warp regions of warp_doubles
    long long warp_doubles;
};

// per-warp region: 14 column arrays of Sc * 32, 4 row arrays of Sr * 32, then the factor (bsplit::factor_doubles)
struct SWork {
    double *x, *z, *c, *rd, *d, *dx, *cor, *rx, *s, *wv, *u, *ru, *cors, *rs;   // columns (bound arrays used on bounded columns)
    double *y, *b, *rp, *dy;                                                    // rows
};
inline __host__ __device__ long long split_vec_doubles(int Sr, int Sc) { return 14LL * Sc * 32 + 4LL * Sr * 32; }

#define SCOLS for (int s_ = 0; s_ < cc; ++s_) if (const int j = s_ * 32 + lane; true)
#define SROWS for (int s_ = 0; s_ < cs; ++s_) if (const int i = s_ * 32 + lane; true)

template <bool CORR, int BW>
__device__ __forceinline__ void split_newton(const SWork &W, const bsplit::Factor<BW> &F, const SplitParams &S, const int *cnat, int nb,
                                             int cc, int cs, double smu, int lane) {
    SCOLS {
        double h = W.rd[j] + W.z[j];
        if (cnat[j] < nb) {
            const double wj = W.wv[j];
            double as = -wj * W.ru[j];
            if (CORR) { h -= (smu - W.cor[j]) * W.rx[j]; as += smu - W.cors[j]; }
            h += as * W.rs[j] - wj;
        } else if (CORR) {
            h -= (smu - W.cor[j]) * W.rx[j];
        }
        W.dx[j] = W.d[j] * h;
    }
    __syncwarp();
    SROWS {
        double acc = W.rp[i];
        for (int q = S.A_ptr[i]; q < S.A_ptr[i + 1]; ++q) acc += S.A_val[q] * W.dx[S.A_idx[q]];
        W.dy[i] = acc;
    }
    __syncwarp();
    bsplit::split_solve<BW>(F, W.dy, lane);
    SCOLS {
        double acc = 0.0;
        for (int q = S.At_ptr[j]; q < S.At_ptr[j + 1]; ++q) acc += S.At_val[q] * W.dy[S.At_idx[q]];
        W.dx[j] = W.d[j] * acc - W.dx[j];
    }
    __syncwarp();
}

template <bool CORR>
__device__ __forceinline__ void split_step_pass(const SWork &W, const int *cnat, int nb, int cc, double smu, int lane, double &ip,
                                                double &id) {
    SCOLS {
        const double zj = W.z[j], rxj = W.rx[j], dxj = W.dx[j];
        double dzj = -zj - zj * dxj * rxj;
        if (CORR) dzj += (smu - W.cor[j]) * rxj;
        if (cnat[j] < nb) {
            const double wj = W.wv[j], rsj = W.rs[j];
            const double dsj = W.ru[j] - dxj;
            double dwj = -wj - wj * dsj * rsj;
            if (CORR) dwj += (smu - W.cors[j]) * rsj;
            ip = dmaxd(ip, dmaxd(-dxj * rxj, -dsj * rsj));
            id = dmaxd(id, dmaxd(-dzj * frcpd(zj), -dwj * frcpd(wj)));
        } else {
            ip = dmaxd(ip, -dxj * rxj);
            id = dmaxd(id, -dzj * frcpd(zj));
        }
    }
}

template <int BW>
__device__ void split_solve_one(const SWork &W, const bsplit::Factor<BW> &F, const KParams &P, const SplitParams &S, long long p, int lane,
                                double step_frac, double reg, int it0, int *status_out, int *iters_out) {
    const int n = P.n, nb = P.nb, m = P.m;
    const int cc = S.ccnt[lane], cs = F.rows(lane);
    const int r0 = lane * (m >> 5) + min(lane, m & 31);        // template row of this lane's slot 0
    const int *cnat = S.cnat;
    const double *cp = P.cparams + p * (long long)P.Pc;
    const double *rp_ = P.rparams + p * P.rstride;
    // ---- instantiate c, b, u, objective constant from the parameter maps
    double cmax = 0.0, bmax = 0.0, kconst = 0.0;
    SCOLS {
        const int jn = cnat[j];
        double acc = P.c0[jn];
        for (int q = P.cm_ptr[jn]; q < P.cm_ptr[jn + 1]; ++q) acc += P.cm_val[q] * cp[P.cm_idx[q]];
        W.c[j] = acc;
        cmax = dmaxd(cmax, fabs(acc));
        if (jn < nb) {
            double ua = P.u0[jn];
            for (int q = P.um_ptr[jn]; q < P.um_ptr[jn + 1]; ++q) ua += P.um_val[q] * rp_[P.um_idx[q]];
            W.u[j] = ua;
            bmax = dmaxd(bmax, ua);
        }
    }
    SROWS {
        const int rn = r0 + s_;
        double acc = P.b0[rn];
        for (int q = P.bm_ptr[rn]; q < P.bm_ptr[rn + 1]; ++q) acc += P.bm_val[q] * rp_[P.bm_idx[q]];
        W.b[i] = acc;
        bmax = dmaxd(bmax, fabs(acc));
    }
    for (int r = lane; r < P.Pr; r += 32) kconst += P.omap[r] * rp_[r];
    for (int r = lane; r < P.Pc; r += 32) kconst += P.ocmap[r] * cp[r];
    kconst = warp_sum(kconst) + P.o0;
    cmax = warp_max(cmax);
    bmax = warp_max(bmax);
    const double beta_b = bmax > 0.0 ? bmax : 1.0;
    const double beta_c = cmax > 0.0 ? cmax : 1.0;
    // ---- scale, start point
    double bsmax = 0.0;
    bool bad_u = false;             // a negative upper bound: the LP is infeasible, not "u = 1e-10"
    SROWS {
        const double v = W.b[i] / beta_b;
        W.b[i] = v;
        W.y[i] = 0.0;
        bsmax = dmaxd(bsmax, fabs(v));
    }
    SCOLS {
        W.c[j] = W.c[j] / beta_c;
        double xj = 1.0;
        if (cnat[j] < nb) {
            bad_u |= W.u[j] < -1e-9 * beta_b;
            const double uj = dmaxd(W.u[j] / beta_b, 1e-10);
            W.u[j] = uj;
            xj = fmin(1.0, 0.5 * uj);
            W.s[j] = uj - xj;
            W.wv[j] = 1.0;
        }
        W.x[j] = xj;
        W.z[j] = 1.0;
    }
    bsmax = warp_max(bsmax);
    const double nrm_b = 1.0 + bsmax, nrm_c = 1.0 + (cmax > 0.0 ? 1.0 : 0.0);
    const double ntot = (double)(n + nb);
    __syncwarp();
    if (__any_sync(0xffffffffu, bad_u)) {
        if (lane == 0) { P.obj[p] = __longlong_as_double(0x7ff8000000000000LL); P.status[p] = DSP_INFEASIBLE; P.iters[p] = it0; }
        dsp_nan_rows(P.x_out, n, P.y_out, m, p, lane, 32);
        *status_out = DSP_OPTIMAL;          // no second attempt
        *iters_out = it0;
        return;
    }

    int status = DSP_MAX_ITER, it = 0;
    double pobj = 0.0;
    for (it = 0; it <= P.max_iter; ++it) {
        // ---- residuals, complementarity, objectives, scaling matrix
        double pmax = 0.0, dmax = 0.0, musum = 0.0, po = 0.0, dobj = 0.0;
        SROWS {
            double acc = W.b[i];
            for (int q = S.A_ptr[i]; q < S.A_ptr[i + 1]; ++q) acc -= S.A_val[q] * W.x[S.A_idx[q]];
            W.rp[i] = acc;
            pmax = dmaxd(pmax, fabs(acc));
            dobj += W.b[i] * W.y[i];
        }
        SCOLS {
            const double xj = W.x[j], zj = W.z[j];
            double acc = W.c[j] - zj;
            for (int q = S.At_ptr[j]; q < S.At_ptr[j + 1]; ++q) acc -= S.At_val[q] * W.y[S.At_idx[q]];
            const double rxj = frcpd(xj);
            double t = zj * rxj + (xj > 1.0 ? reg * rxj * rxj : reg);      // proximal term, scale invariant for x > 1
            if (cnat[j] < nb) {
                const double sj = W.s[j], wj = W.wv[j], uj = W.u[j];
                acc += wj;
                const double r = uj - xj - sj;
                const double rsj = frcpd(sj);
                W.ru[j] = r;
                W.rs[j] = rsj;
                pmax = dmaxd(pmax, fabs(r));
                musum += sj * wj;
                dobj -= uj * wj;
                t += wj * rsj;
            }
            W.rx[j] = rxj;
            W.rd[j] = acc;
            W.d[j] = frcpd(t);
            dmax = dmaxd(dmax, fabs(acc));
            musum += xj * zj;
            po += W.c[j] * xj;
        }
        pmax = warp_max(pmax);
        dmax = warp_max(dmax);
        musum = warp_sum(musum);
        po = warp_sum(po);
        dobj = warp_sum(dobj);
        pobj = po;
        const double mu = musum / ntot;
        const double gap = fabs(po - dobj) / dmaxd(kGapFloor, fabs(po));
        if (!(mu == mu) || !(po == po) || mu > 1e100) { status = DSP_NUMERICAL; break; }
        const double res = dmaxd(pmax / nrm_b, dmax / nrm_c);
        const double cgap = ntot * mu / dmaxd(kGapFloor, fabs(po));
        if (res < P.feas_tol && gap < P.tol) { status = DSP_OPTIMAL; break; }
        if (cgap < P.tol && res < 10.0 * P.feas_tol && gap < 10.0 * P.tol) { status = DSP_OPTIMAL; break; }
        if (cgap < 1e-3 * P.tol) {
            status = (res < 100.0 * P.feas_tol && gap < 1000.0 * P.tol) ? DSP_OPTIMAL : DSP_NUMERICAL;
            break;
        }
        if (it == P.max_iter) break;
        __syncwarp();
        // ---- assemble the band of M = A D A' (split layout), factorise
        for (int s_ = 0; s_ < cs; ++s_) {
#pragma unroll
            for (int k = 0; k <= BW; ++k) {
                const int e = (k * S.Sr + s_) * 32 + lane;
                double acc = 0.0;
                for (int q = S.asm_ptr[e]; q < S.asm_ptr[e + 1]; ++q) acc += S.asm_val[q] * W.d[S.asm_col[q]];
                F.Mb[e] = acc;
            }
        }
        __syncwarp();
        bsplit::split_factor<BW>(F, lane);
        // ---- affine predictor
        split_newton<false, BW>(W, F, S, cnat, nb, cc, cs, 0.0, lane);
        double ip = 0.0, id = 0.0;
        split_step_pass<false>(W, cnat, nb, cc, 0.0, lane, ip, id);
        ip = warp_max(ip); id = warp_max(id);
        double ap = ip > 1.0 ? 1.0 / ip : 1.0, ad = id > 1.0 ? 1.0 / id : 1.0;
        double mua = 0.0;
        SCOLS {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j];
            const double dzj = -zj - zj * dxj * W.rx[j];
            mua += (xj + ap * dxj) * (zj + ad * dzj);
            W.cor[j] = dxj * dzj;
            if (cnat[j] < nb) {
                const double sj = W.s[j], wj = W.wv[j];
                const double dsj = W.ru[j] - dxj;
                const double dwj = -wj - wj * dsj * W.rs[j];
                mua += (sj + ap * dsj) * (wj + ad * dwj);
                W.cors[j] = dsj * dwj;
            }
        }
        mua = warp_sum(mua) / ntot;
        const double sg = mua / mu;
        const double smu = sg * sg * sg * mu;
        __syncwarp();
        // ---- centring corrector
        split_newton<true, BW>(W, F, S, cnat, nb, cc, cs, smu, lane);
        ip = 0.0; id = 0.0;
        split_step_pass<true>(W, cnat, nb, cc, smu, lane, ip, id);
        ip = warp_max(ip); id = warp_max(id);
        ap = step_frac < ip ? step_frac / ip : 1.0;
        ad = step_frac < id ? step_frac / id : 1.0;
        SCOLS {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j], rxj = W.rx[j];
            const double dzj = (smu - W.cor[j]) * rxj - zj - zj * dxj * rxj;
            if (cnat[j] < nb) {
                const double sj = W.s[j], wj = W.wv[j], rsj = W.rs[j];
                const double dsj = W.ru[j] - dxj;
                const double dwj = (smu - W.cors[j]) * rsj - wj - wj * dsj * rsj;
                W.s[j] = sj + ap * dsj;
                W.wv[j] = wj + ad * dwj;
            }
            W.x[j] = xj + ap * dxj;
            W.z[j] = zj + ad * dzj;
        }
        SROWS W.y[i] += ad * W.dy[i];
        __syncwarp();
    }
    // ---- results, in the template's (or, dsp_lp_template_create_csr, the caller's) order
    if (lane == 0) {
        P.obj[p] = pobj * beta_b * beta_c + kconst;
        P.status[p] = status;
        P.iters[p] = it + it0;
    }
    if (P.x_out) {
        double *xo = P.x_out + p * (long long)n;
        SCOLS { const int jn = cnat[j]; xo[P.xperm ? P.xperm[jn] : jn] = W.x[j] * beta_b; }
    }
    if (P.y_out) {
        double *yo = P.y_out + p * (long long)m;
        SROWS { const int rn = r0 + s_; yo[P.yperm ? P.yperm[rn] : rn] = W.y[i] * beta_c; }
    }
    __syncwarp();
    *status_out = status;
    *iters_out = it + it0;
}
#undef SCOLS
#undef SROWS

constexpr int kSplitWarps = 4;      // warps per CTA of the split kernel

template <int BW>
__global__ void __launch_bounds__(kSplitWarps * 32) dsp_ipm_band_split_kernel(const KParams P, const SplitParams S) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *base = S.ws + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (size_t)S.warp_doubles;
    const size_t cs = (size_t)S.Sc * 32, rs = (size_t)S.Sr * 32;
    SWork W;
    W.x = base; W.z = W.x + cs; W.c = W.z + cs; W.rd = W.c + cs; W.d = W.rd + cs; W.dx = W.d + cs; W.cor = W.dx + cs; W.rx = W.cor + cs;
    W.s = W.rx + cs; W.wv = W.s + cs; W.u = W.wv + cs; W.ru = W.u + cs; W.cors = W.ru + cs; W.rs = W.cors + cs;
    W.y = W.rs + cs; W.b = W.y + rs; W.rp = W.b + rs; W.dy = W.rp + rs;
    bsplit::Factor<BW> F;
    F.Mb = W.dy + rs; F.G = F.Mb + (BW + 1) * rs; F.E = F.G + BW * rs; F.X = F.E + BW * BW * 32;
    F.Sr = S.Sr; F.m = P.m;
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1ULL);
        t = __shfl_sync(0xffffffffu, t, 0);
        if ((long long)t >= P.N) break;
        int st, it0 = 0;
        // second attempt: shorter step and a 100x proximal term (the long-horizon kernel's: 10x is not enough at cond 1e15)
        split_solve_one<BW>(W, F, P, S, (long long)t, lane, P.step_frac, P.reg, 0, &st, &it0);
#ifdef DSP_PHASES       // instrumentation build: LPs whose first attempt / both attempts end non-optimal (tools/gpu_band_phases_long.py)
        if (lane == 0 && st != DSP_OPTIMAL) atomicAdd(&g_phase[14], 1ULL);
#endif
        if (st != DSP_OPTIMAL) split_solve_one<BW>(W, F, P, S, (long long)t, lane, 0.99, 100.0 * P.reg, it0, &st, &it0);
#ifdef DSP_PHASES
        if (lane == 0 && st != DSP_OPTIMAL) atomicAdd(&g_phase[15], 1ULL);
#endif
    }
}
#endif
