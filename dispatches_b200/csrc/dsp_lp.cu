// dsp_lp.cu -- batched primal-dual interior-point LP solver for sm_90a (H100).  C ABI: include/dsp_lp.h
//
// Replaces the per-scenario  SolverFactory("cbc").solve(m)  loop of the reference's price-taker sweeps
// (wind_battery_LMP.py:266-267, wind_battery_PEM_LMP.py:296-298, price_taker_analysis.py:365-403) by one
// launch that solves the whole scenario batch.
//
// Kernel `dsp_ipm_band_kernel`  (generic path, any template whose A*A' is banded):
//   * one CTA per SM, persistent; one WARP per LP, problems handed out by an atomic ticket (iteration counts
//     differ per LP, SURVEY.md §7.3-4);
//   * the shared template (A in CSR and CSC, band assembly list) is staged once per CTA into shared memory with
//     a TMA bulk copy (cp.async.bulk + mbarrier) when it fits, otherwise read through L2;
//   * every per-problem vector and the band of M = A D A' live in shared memory for the whole solve;
//     HBM traffic per LP is the parameter row in and (obj, status, iters [, x, y]) out;
//   * FP64 throughout (cond(M) reaches 1e15 near convergence, SURVEY.md §0.6);
//   * Mehrotra predictor-corrector; M is factorised once per iteration by a band LDL' (half bandwidth w),
//     two band solves per iteration.  The numpy mirror of exactly this algorithm is oracle/ipm_numpy.py.
//
// Kernel `dsp_ipm_dense_kernel` (any bandwidth, m <= 1024; dsp_lp_template_create_dense or DSP_KERNEL_DENSE): the same iteration,
// one CTA per LP, M = A D A' dense in a workspace, blocked LDL' with FP64 tensor-core trailing updates (dsp_dense.cuh).
#include "dsp_lp.h"

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "dsp_band.cuh"
#include "dsp_nan_rows.cuh"

#define DSP_VERSION "dsp_lp 0.2 (sm_90a band-IPM + stage kernels)"

namespace {

#ifdef DSP_PHASES            // developer instrumentation: per-phase cycle counters (warp 0 of block 0 accumulates)
__device__ unsigned long long g_phase[16];
__device__ int g_pass2_twice;    // stage 2 runs pass 2 of every round twice (DSP_STAGE2_PASS2_TWICE, tools/gpu_stage2_phases.py)
#define PH_INIT long long ph_t0 = clock64();
#define PH(k) do { long long ph_t1 = clock64(); if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&g_phase[k], (unsigned long long)(ph_t1 - ph_t0)); ph_t0 = clock64(); } while (0)
#else
#define PH_INIT
#define PH(k)
#endif

constexpr int kMaxWarps = 16;
constexpr double kGapFloor = 1e-4;         // scaled-objective floor of the relative gap test

struct KParams {
    // template
    int m, n, nb, w, Pc, Pr, nnz, nasm;
    const unsigned char *hot_g;   // hot blob in global memory
    int hot_bytes;                // multiple of 16
    int hot_in_smem;
    const double *c0, *b0, *u0, *omap, *ocmap;
    const int *cm_ptr, *cm_idx, *bm_ptr, *bm_idx, *um_ptr, *um_idx;
    const double *cm_val, *bm_val, *um_val;
    double o0;
    // batch
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    double tol, feas_tol, step_frac, reg;
    int max_iter;
    double *obj, *x_out, *y_out;
    int *status, *iters;
    unsigned long long *ticket;
    double *ws;                   // non-null: per-warp work regions live in this global-memory workspace (long horizons)
    int prob_doubles;             // per-warp work-region doubles
    int prob_off;                 // byte offset of the first per-warp region
    int band_doubles;             // doubles of the (dy, Mb) tail of a work region: what the LDL' / substitution sweeps touch
    int hybrid;                   // workspace mode with the (dy, Mb) tail in shared memory (sweeps at shared-memory latency)
    const int *xperm, *yperm;     // non-null: x_out / y_out index of internal column j / row i (dsp_lp_template_create_csr)
    // per-problem matrix coefficients (dsp_lp_template_set_matrix_params):  A_val[q] = A0[q] + sum coef * rparams[param]
    int n_amap;                   // 0: the matrix is shared by the batch
    const int *amap_q, *amap_param;       // CSR position / rparams index of every term
    const double *amap_coef;
    const int *at_from;           // CSC position -> CSR position (A' values follow A's)
    const int *asm_qa, *asm_qb;   // band assembly: the two CSR positions whose product is asm_val[p]
    int retry_only;               // second pass behind a stage kernel: solve only the LPs whose status is MAX_ITER / NUMERICAL
};

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- TMA bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP + SYNCS)
__device__ __forceinline__ void tma_stage(void *dst, const void *src, int bytes, uint64_t *bar) {
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
        // bulk copies are limited in size per instruction; issue in chunks
        int off = 0;
        while (off < bytes) {
            int chunk = min(bytes - off, 32768);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32((char *)dst + off)), "l"((const char *)src + off), "r"(chunk), "r"(smem_u32(bar))
                         : "memory");
            off += chunk;
        }
    }
    // every thread waits for phase 0 to complete
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(0)
        : "memory");
}

struct Hot {   // views into the hot blob (shared or global)
    const double *A_val, *At_val, *asm_val;
    const int *A_ptr, *A_idx, *At_ptr, *At_idx, *asm_ptr, *asm_col;
};

__device__ __forceinline__ Hot hot_views(const unsigned char *base, const KParams &P) {
    Hot h;
    h.A_val = (const double *)base;
    h.At_val = h.A_val + P.nnz;
    h.asm_val = h.At_val + P.nnz;
    h.A_ptr = (const int *)(h.asm_val + P.nasm);
    h.A_idx = h.A_ptr + (P.m + 1);
    h.At_ptr = h.A_idx + P.nnz;
    h.At_idx = h.At_ptr + (P.n + 1);
    h.asm_ptr = h.At_idx + P.nnz;
    h.asm_col = h.asm_ptr + (P.m * (P.w + 1) + 1);
    return h;
}

// band LDL' / substitution sweeps (dsp_band.cuh)
using band::dmaxd;
using band::frcpd;
using band::band_factor;
using band::band_solve;

struct Work {   // per-warp shared-memory vectors
    double *x, *z, *c, *rd, *d, *dx, *cor, *rx;     // n
    double *s, *wv, *u, *ru, *cors, *rs;            // nb
    double *y, *b, *rp;                             // m
    double *dy;                                     // m + 2W (padded)
    double *Mb;                                     // (m + 2W) * (W+1) (padded)
};

// Newton direction for the complementarity targets  x z -> ax,  s w -> as  (ax = as = 0: affine predictor;
// ax_j = smu - cor_j: centring corrector).  On exit W.dx = dx, W.dy = dy.
template <bool CORR, int BW>
__device__ __forceinline__ void newton(const Work &W, const Hot &H, const KParams &P, double smu, int lane) {
    const int n = P.n, nb = P.nb, m = P.m;
    for (int j = lane; j < nb; j += 32) {           // bounded columns
        const double wj = W.wv[j];
        double h = W.rd[j] + W.z[j], as = -wj * W.ru[j];
        if (CORR) { h -= (smu - W.cor[j]) * W.rx[j]; as += smu - W.cors[j]; }
        h += as * W.rs[j] - wj;
        W.dx[j] = W.d[j] * h;
    }
    for (int j = nb + lane; j < n; j += 32) {       // the rest
        double h = W.rd[j] + W.z[j];
        if (CORR) h -= (smu - W.cor[j]) * W.rx[j];
        W.dx[j] = W.d[j] * h;
    }
    __syncwarp();
    for (int i = lane; i < m; i += 32) {
        double acc = W.rp[i];
        for (int q = H.A_ptr[i]; q < H.A_ptr[i + 1]; ++q) acc += H.A_val[q] * W.dx[H.A_idx[q]];
        W.dy[i] = acc;
    }
    __syncwarp();
    band_solve<BW>(W.Mb, W.dy, m, lane);
    for (int j = lane; j < n; j += 32) {
        double acc = 0.0;
        for (int q = H.At_ptr[j]; q < H.At_ptr[j + 1]; ++q) acc += H.At_val[q] * W.dy[H.At_idx[q]];
        W.dx[j] = W.d[j] * acc - W.dx[j];
    }
    __syncwarp();
}

// step-length pass shared by predictor and corrector: 1/alpha_p, 1/alpha_d candidates of this lane
template <bool CORR>
__device__ __forceinline__ void step_pass(const Work &W, const KParams &P, double smu, int lane, double &ip, double &id) {
    const int n = P.n, nb = P.nb;
    for (int j = lane; j < nb; j += 32) {
        const double zj = W.z[j], wj = W.wv[j], rxj = W.rx[j], rsj = W.rs[j], dxj = W.dx[j];
        double dzj = -zj - zj * dxj * rxj;
        const double dsj = W.ru[j] - dxj;
        double dwj = -wj - wj * dsj * rsj;
        if (CORR) { dzj += (smu - W.cor[j]) * rxj; dwj += (smu - W.cors[j]) * rsj; }
        ip = dmaxd(ip, dmaxd(-dxj * rxj, -dsj * rsj));
        id = dmaxd(id, dmaxd(-dzj * frcpd(zj), -dwj * frcpd(wj)));
    }
    for (int j = nb + lane; j < n; j += 32) {
        const double zj = W.z[j], rxj = W.rx[j], dxj = W.dx[j];
        double dzj = -zj - zj * dxj * rxj;
        if (CORR) dzj += (smu - W.cor[j]) * rxj;
        ip = dmaxd(ip, -dxj * rxj);
        id = dmaxd(id, -dzj * frcpd(zj));
    }
}

template <int BW>
__device__ void solve_one(const Work &W, const Hot &H0, const KParams &P, long long p, int lane, double step_frac,
                          double reg, int it0, int *status_out, int *iters_out) {
    const int n = P.n, nb = P.nb, m = P.m;
    constexpr int W1 = BW + 1;
    const double *cp = P.cparams + p * (long long)P.Pc;
    const double *rp_ = P.rparams + p * P.rstride;
    Hot H = H0;
    if (P.n_amap > 0) {
        // this LP's own matrix values (free design columns multiplied by per-scenario capacity factors, wind_power.py:120-122):
        // CSR values, CSC values and the band-assembly products live in the warp's work region behind the band
        double *Av = W.Mb + (m + BW) * W1, *Atv = Av + P.nnz, *asv = Atv + P.nnz;
        for (int q = lane; q < P.nnz; q += 32) Av[q] = H0.A_val[q];
        __syncwarp();
        if (lane == 0)
            for (int k = 0; k < P.n_amap; ++k) Av[P.amap_q[k]] += P.amap_coef[k] * rp_[P.amap_param[k]];
        __syncwarp();
        for (int q = lane; q < P.nnz; q += 32) Atv[q] = Av[P.at_from[q]];
        for (int q = lane; q < P.nasm; q += 32) asv[q] = Av[P.asm_qa[q]] * Av[P.asm_qb[q]];
        __syncwarp();
        H.A_val = Av; H.At_val = Atv; H.asm_val = asv;
    }
    // ---- instantiate c, b, u, objective constant from the parameter maps
    double cmax = 0.0, bmax = 0.0, kconst = 0.0;
    for (int j = lane; j < n; j += 32) {
        double acc = P.c0[j];
        for (int q = P.cm_ptr[j]; q < P.cm_ptr[j + 1]; ++q) acc += P.cm_val[q] * cp[P.cm_idx[q]];
        W.c[j] = acc;
        cmax = dmaxd(cmax, fabs(acc));
    }
    for (int i = lane; i < m; i += 32) {
        double acc = P.b0[i];
        for (int q = P.bm_ptr[i]; q < P.bm_ptr[i + 1]; ++q) acc += P.bm_val[q] * rp_[P.bm_idx[q]];
        W.b[i] = acc;
        bmax = dmaxd(bmax, fabs(acc));
    }
    for (int j = lane; j < nb; j += 32) {
        double acc = P.u0[j];
        for (int q = P.um_ptr[j]; q < P.um_ptr[j + 1]; ++q) acc += P.um_val[q] * rp_[P.um_idx[q]];
        W.u[j] = acc;
        bmax = dmaxd(bmax, acc);
    }
    for (int r = lane; r < P.Pr; r += 32) kconst += P.omap[r] * rp_[r];
    for (int r = lane; r < P.Pc; r += 32) kconst += P.ocmap[r] * cp[r];
    kconst = warp_sum(kconst) + P.o0;
    cmax = warp_max(cmax);
    bmax = warp_max(bmax);
    const double beta_b = bmax > 0.0 ? bmax : 1.0;
    const double beta_c = cmax > 0.0 ? cmax : 1.0;
    // ---- scale, start point, zero the paddings
    double bsmax = 0.0;
    bool bad_u = false;             // a negative upper bound (Umap / rparams): the LP is infeasible, not "u = 1e-10"
    for (int i = lane; i < m; i += 32) {
        const double v = W.b[i] / beta_b;
        W.b[i] = v;
        W.y[i] = 0.0;
        bsmax = dmaxd(bsmax, fabs(v));
    }
    for (int j = lane; j < n; j += 32) {
        W.c[j] = W.c[j] / beta_c;
        double xj = 1.0;
        if (j < nb) {
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
    for (int k = lane; k < BW * W1; k += 32) { W.Mb[-(k + 1)] = 0.0; W.Mb[m * W1 + k] = 0.0; }
    for (int k = lane; k < BW; k += 32) { W.dy[-(k + 1)] = 0.0; W.dy[m + k] = 0.0; }
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
    PH_INIT
    for (it = 0; it <= P.max_iter; ++it) {
        PH(7);
        // ---- residuals, complementarity, objectives, scaling matrix (reciprocals kept for the whole iteration)
        double pmax = 0.0, dmax = 0.0, musum = 0.0, po = 0.0, dobj = 0.0;
        for (int i = lane; i < m; i += 32) {
            double acc = W.b[i];
            for (int q = H.A_ptr[i]; q < H.A_ptr[i + 1]; ++q) acc -= H.A_val[q] * W.x[H.A_idx[q]];
            W.rp[i] = acc;
            pmax = dmaxd(pmax, fabs(acc));
            dobj += W.b[i] * W.y[i];
        }
        for (int j = lane; j < n; j += 32) {
            const double xj = W.x[j], zj = W.z[j];
            double acc = W.c[j] - zj;
            for (int q = H.At_ptr[j]; q < H.At_ptr[j + 1]; ++q) acc -= H.At_val[q] * W.y[H.At_idx[q]];
            const double rxj = frcpd(xj);
            double t = zj * rxj + (xj > 1.0 ? reg * rxj * rxj : reg);      // proximal term, scale invariant for x > 1
            if (j < nb) {
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
        const double cgap = ntot * mu / dmaxd(kGapFloor, fabs(po));   // what further iterations can still reduce
        if (res < P.feas_tol && gap < P.tol) { status = DSP_OPTIMAL; break; }
        // complementarity has converged but residuals / objective gap sit at the rounding floor of the
        // ill-conditioned normal equations: iterating further only loses accuracy -> accept what is there
        if (cgap < P.tol && res < 10.0 * P.feas_tol && gap < 10.0 * P.tol) { status = DSP_OPTIMAL; break; }
        if (cgap < 1e-3 * P.tol) {
            status = (res < 100.0 * P.feas_tol && gap < 1000.0 * P.tol) ? DSP_OPTIMAL : DSP_NUMERICAL;
            break;
        }
        if (it == P.max_iter) break;
        __syncwarp();
        PH(0);
        // ---- assemble the band of M = A D A'
        const int nent = m * W1;
        for (int e = lane; e < nent; e += 32) {
            double acc = 0.0;
            for (int q = H.asm_ptr[e]; q < H.asm_ptr[e + 1]; ++q) acc += H.asm_val[q] * W.d[H.asm_col[q]];
            W.Mb[e] = acc;
        }
        __syncwarp();
        PH(1);
        band_factor<BW>(W.Mb, m, lane);
        PH(2);
        // ---- affine predictor
        newton<false, BW>(W, H, P, 0.0, lane);
        PH(3);
        double ip = 0.0, id = 0.0;
        step_pass<false>(W, P, 0.0, lane, ip, id);
        ip = warp_max(ip); id = warp_max(id);
        double ap = ip > 1.0 ? 1.0 / ip : 1.0, ad = id > 1.0 ? 1.0 / id : 1.0;
        double mua = 0.0;
        for (int j = lane; j < n; j += 32) {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j];
            const double dzj = -zj - zj * dxj * W.rx[j];
            mua += (xj + ap * dxj) * (zj + ad * dzj);
            W.cor[j] = dxj * dzj;
            if (j < nb) {
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
        PH(4);
        // ---- centring corrector
        newton<true, BW>(W, H, P, smu, lane);
        PH(5);
        ip = 0.0; id = 0.0;
        step_pass<true>(W, P, smu, lane, ip, id);
        ip = warp_max(ip); id = warp_max(id);
        ap = step_frac < ip ? step_frac / ip : 1.0;
        ad = step_frac < id ? step_frac / id : 1.0;
        for (int j = lane; j < n; j += 32) {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j], rxj = W.rx[j];
            const double dzj = (smu - W.cor[j]) * rxj - zj - zj * dxj * rxj;
            if (j < nb) {
                const double sj = W.s[j], wj = W.wv[j], rsj = W.rs[j];
                const double dsj = W.ru[j] - dxj;
                const double dwj = (smu - W.cors[j]) * rsj - wj - wj * dsj * rsj;
                W.s[j] = sj + ap * dsj;
                W.wv[j] = wj + ad * dwj;
            }
            W.x[j] = xj + ap * dxj;
            W.z[j] = zj + ad * dzj;
        }
        for (int i = lane; i < m; i += 32) W.y[i] += ad * W.dy[i];
        __syncwarp();
        PH(6);
    }
    // ---- results
    if (lane == 0) {
        P.obj[p] = pobj * beta_b * beta_c + kconst;
        P.status[p] = status;
        P.iters[p] = it + it0;
    }
    if (P.x_out) {
        double *xo = P.x_out + p * (long long)n;
        if (P.xperm) { for (int j = lane; j < n; j += 32) xo[P.xperm[j]] = W.x[j] * beta_b; }
        else { for (int j = lane; j < n; j += 32) xo[j] = W.x[j] * beta_b; }
    }
    if (P.y_out) {
        double *yo = P.y_out + p * (long long)m;
        if (P.yperm) { for (int i = lane; i < m; i += 32) yo[P.yperm[i]] = W.y[i] * beta_c; }
        else { for (int i = lane; i < m; i += 32) yo[i] = W.y[i] * beta_c; }
    }
    __syncwarp();
    *status_out = status;
    *iters_out = it + it0;
}

// WS = true: per-warp work regions in the global workspace P.ws (long horizons); false: in shared memory (the compiler
// then keeps every W.* access an LDS/STS instead of a generic load)
// HS = true: the template blob is staged into shared memory (its accesses become LDS too)
template <int BW, bool WS, bool HS>
__global__ void __launch_bounds__(kMaxWarps * 32, 1) dsp_ipm_band_kernel(const KParams P) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Hot H;
    if (HS) {
        tma_stage(smem + 16, P.hot_g, P.hot_bytes, (uint64_t *)smem);
        H = hot_views(smem + 16, P);
    } else {
        H = hot_views(P.hot_g, P);
    }
    double *base;
    if (WS) base = P.ws + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (size_t)P.prob_doubles;
    else base = (double *)(smem + P.prob_off) + (size_t)warp * P.prob_doubles;
    Work W;
    const int n = P.n, nb = P.nb, m = P.m;
    W.x = base; W.z = W.x + n; W.c = W.z + n; W.rd = W.c + n; W.d = W.rd + n; W.dx = W.d + n; W.cor = W.dx + n; W.rx = W.cor + n;
    W.s = W.rx + n; W.wv = W.s + nb; W.u = W.wv + nb; W.ru = W.u + nb; W.cors = W.ru + nb; W.rs = W.cors + nb;
    W.y = W.rs + nb; W.b = W.y + m; W.rp = W.b + m;
    double *band0 = W.rp + m;
    if (WS && P.hybrid) band0 = (double *)(smem + P.prob_off) + (size_t)warp * P.band_doubles;
    W.dy = band0 + BW;
    W.Mb = W.dy + m + BW + BW * (BW + 1);
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1ULL);
        t = __shfl_sync(0xffffffffu, t, 0);
        if ((long long)t >= P.N) break;
        if (P.retry_only && (P.status[t] == DSP_OPTIMAL || P.status[t] == DSP_INFEASIBLE)) continue;
        int st, it0 = 0;
        // second attempt (shorter step, stronger proximal term) for the rare LP whose first attempt ends non-optimal
        solve_one<BW>(W, H, P, (long long)t, lane, P.step_frac, P.reg, 0, &st, &it0);
        if (st != DSP_OPTIMAL) solve_one<BW>(W, H, P, (long long)t, lane, 0.99, 10.0 * P.reg, it0, &st, &it0);
    }
}

}  // namespace

#include "dsp_dense.cuh"

namespace {
// =====================================================================================================
// Dense kernel `dsp_ipm_dense_kernel` (any bandwidth, m <= 1024): one persistent CTA of kDenseWarps warps per LP, the same
// Mehrotra iteration as the band kernel's solve_one with its element-wise and CSR passes spread over the CTA; M = A D A' dense,
// factored by the blocked LDL' of dsp_dense.cuh in a per-CTA workspace region.  Numpy mirror: oracle/ipm_dense_numpy.py.
// =====================================================================================================
constexpr int kDenseWarps = 8;
constexpr int kDenseThreads = kDenseWarps * 32;
constexpr int kDenseMaxM = 1024;

struct DParams {
    int m, n, nb, Pc, Pr, nt;
    const double *c0, *b0, *u0, *omap, *ocmap;
    const int *cm_ptr, *cm_idx, *bm_ptr, *bm_idx, *um_ptr, *um_idx;
    const double *cm_val, *bm_val, *um_val;
    double o0;
    const int *A_ptr, *A_idx, *At_ptr, *At_idx;
    const double *A_val, *At_val;
    int nent;                          // entries of the lower pattern of A A', tile-major
    const int *asm_pos, *asm_ptr, *asm_col;   // workspace offset of entry e; its products asm_val[asm_ptr[e] ..] * d[asm_col[..]]
    const double *asm_val;
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    double tol, feas_tol, step_frac, reg;
    int max_iter;
    double *obj, *x_out, *y_out;
    int *status, *iters;
    unsigned long long *ticket;
    const int *xperm, *yperm;
    double *ws;                        // per-CTA regions: the lower tiles of M, then (vec_in_smem == 0) the per-LP vectors
    long long cta_doubles;
    int vec_in_smem;
};

// doubles of the per-LP vectors: x z c rd d dx cor rx (n), s wv u ru cors rs (nb), y b rp (m), dy dinv (mp)
inline long long dense_vec_doubles(int m, int n, int nb, int nt) { return 8LL * n + 6LL * nb + 3LL * m + 2LL * nt * dense::TS; }
// shared memory ahead of the vectors: reduction slots and the ticket, the two staged-tile buffers
constexpr size_t kDenseSmemFixed = (size_t)(2 * kDenseWarps + 2 * dense::TS * dense::LDS) * 8;

struct DWork {
    double *x, *z, *c, *rd, *d, *dx, *cor, *rx;
    double *s, *wv, *u, *ru, *cors, *rs;
    double *y, *b, *rp;
    double *dy, *dinv;                 // mp
    double *G;                         // lower tiles of M
    double *SA, *SB, *red;
};

__device__ __forceinline__ double cta_max(double v, double *red) {
    v = warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = red[0];
#pragma unroll
    for (int w = 1; w < kDenseWarps; ++w) r = fmax(r, red[w]);
    return r;
}
__device__ __forceinline__ double cta_sum(double v, double *red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = red[0];
#pragma unroll
    for (int w = 1; w < kDenseWarps; ++w) r += red[w];
    return r;
}

template <bool CORR>
__device__ void dense_newton(const DWork &W, const DParams &P, double smu, int tid) {
    const int n = P.n, nb = P.nb, m = P.m, mp = P.nt * dense::TS;
    for (int j = tid; j < nb; j += kDenseThreads) {
        const double wj = W.wv[j];
        double h = W.rd[j] + W.z[j], as = -wj * W.ru[j];
        if (CORR) { h -= (smu - W.cor[j]) * W.rx[j]; as += smu - W.cors[j]; }
        h += as * W.rs[j] - wj;
        W.dx[j] = W.d[j] * h;
    }
    for (int j = nb + tid; j < n; j += kDenseThreads) {
        double h = W.rd[j] + W.z[j];
        if (CORR) h -= (smu - W.cor[j]) * W.rx[j];
        W.dx[j] = W.d[j] * h;
    }
    __syncthreads();
    for (int i = tid; i < mp; i += kDenseThreads) {
        double acc = 0.0;
        if (i < m) {
            acc = W.rp[i];
            for (int q = P.A_ptr[i]; q < P.A_ptr[i + 1]; ++q) acc += P.A_val[q] * W.dx[P.A_idx[q]];
        }
        W.dy[i] = acc;
    }
    __syncthreads();
    dense::solve(W.G, P.nt, W.dinv, W.dy, tid >> 5, kDenseWarps, tid & 31);
    for (int j = tid; j < n; j += kDenseThreads) {
        double acc = 0.0;
        for (int q = P.At_ptr[j]; q < P.At_ptr[j + 1]; ++q) acc += P.At_val[q] * W.dy[P.At_idx[q]];
        W.dx[j] = W.d[j] * acc - W.dx[j];
    }
    __syncthreads();
}

template <bool CORR>
__device__ __forceinline__ void dense_step_pass(const DWork &W, const DParams &P, double smu, int tid, double &ip, double &id) {
    const int n = P.n, nb = P.nb;
    for (int j = tid; j < nb; j += kDenseThreads) {
        const double zj = W.z[j], wj = W.wv[j], rxj = W.rx[j], rsj = W.rs[j], dxj = W.dx[j];
        double dzj = -zj - zj * dxj * rxj;
        const double dsj = W.ru[j] - dxj;
        double dwj = -wj - wj * dsj * rsj;
        if (CORR) { dzj += (smu - W.cor[j]) * rxj; dwj += (smu - W.cors[j]) * rsj; }
        ip = dmaxd(ip, dmaxd(-dxj * rxj, -dsj * rsj));
        id = dmaxd(id, dmaxd(-dzj * frcpd(zj), -dwj * frcpd(wj)));
    }
    for (int j = nb + tid; j < n; j += kDenseThreads) {
        const double zj = W.z[j], rxj = W.rx[j], dxj = W.dx[j];
        double dzj = -zj - zj * dxj * rxj;
        if (CORR) dzj += (smu - W.cor[j]) * rxj;
        ip = dmaxd(ip, -dxj * rxj);
        id = dmaxd(id, -dzj * frcpd(zj));
    }
}

// one attempt on LP p: the band kernel's solve_one (same scaling, start point, proximal term, stopping rule, results rules)
__device__ void dense_solve_one(const DWork &W, const DParams &P, long long p, double step_frac, double reg, int it0, int *status_out,
                                int *iters_out) {
    const int n = P.n, nb = P.nb, m = P.m, nt = P.nt, mp = nt * dense::TS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const double *cp = P.cparams + p * (long long)P.Pc;
    const double *rp_ = P.rparams + p * P.rstride;
    double cmax = 0.0, bmax = 0.0, kconst = 0.0;
    for (int j = tid; j < n; j += kDenseThreads) {
        double acc = P.c0[j];
        for (int q = P.cm_ptr[j]; q < P.cm_ptr[j + 1]; ++q) acc += P.cm_val[q] * cp[P.cm_idx[q]];
        W.c[j] = acc;
        cmax = dmaxd(cmax, fabs(acc));
    }
    for (int i = tid; i < m; i += kDenseThreads) {
        double acc = P.b0[i];
        for (int q = P.bm_ptr[i]; q < P.bm_ptr[i + 1]; ++q) acc += P.bm_val[q] * rp_[P.bm_idx[q]];
        W.b[i] = acc;
        bmax = dmaxd(bmax, fabs(acc));
    }
    for (int j = tid; j < nb; j += kDenseThreads) {
        double acc = P.u0[j];
        for (int q = P.um_ptr[j]; q < P.um_ptr[j + 1]; ++q) acc += P.um_val[q] * rp_[P.um_idx[q]];
        W.u[j] = acc;
        bmax = dmaxd(bmax, acc);
    }
    for (int r = tid; r < P.Pr; r += kDenseThreads) kconst += P.omap[r] * rp_[r];
    for (int r = tid; r < P.Pc; r += kDenseThreads) kconst += P.ocmap[r] * cp[r];
    kconst = cta_sum(kconst, W.red) + P.o0;
    cmax = cta_max(cmax, W.red);
    bmax = cta_max(bmax, W.red);
    const double beta_b = bmax > 0.0 ? bmax : 1.0;
    const double beta_c = cmax > 0.0 ? cmax : 1.0;
    double bsmax = 0.0;
    int bad_u = 0;
    for (int i = tid; i < m; i += kDenseThreads) {
        const double v = W.b[i] / beta_b;
        W.b[i] = v;
        W.y[i] = 0.0;
        bsmax = dmaxd(bsmax, fabs(v));
    }
    for (int j = tid; j < n; j += kDenseThreads) {
        W.c[j] = W.c[j] / beta_c;
        double xj = 1.0;
        if (j < nb) {
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
    bsmax = cta_max(bsmax, W.red);
    const double nrm_b = 1.0 + bsmax, nrm_c = 1.0 + (cmax > 0.0 ? 1.0 : 0.0);
    const double ntot = (double)(n + nb);
    if (__syncthreads_or(bad_u)) {
        if (tid == 0) { P.obj[p] = __longlong_as_double(0x7ff8000000000000LL); P.status[p] = DSP_INFEASIBLE; P.iters[p] = it0; }
        dsp_nan_rows(P.x_out, n, P.y_out, m, p, tid, kDenseThreads);
        *status_out = DSP_OPTIMAL;          // no second attempt
        *iters_out = it0;
        return;
    }
    const long long ntd = dense::tiles_doubles(nt);
    int status = DSP_MAX_ITER, it = 0;
    double pobj = 0.0;
    for (it = 0; it <= P.max_iter; ++it) {
        double pmax = 0.0, dmax = 0.0, musum = 0.0, po = 0.0, dobj = 0.0;
        for (int i = tid; i < m; i += kDenseThreads) {
            double acc = W.b[i];
            for (int q = P.A_ptr[i]; q < P.A_ptr[i + 1]; ++q) acc -= P.A_val[q] * W.x[P.A_idx[q]];
            W.rp[i] = acc;
            pmax = dmaxd(pmax, fabs(acc));
            dobj += W.b[i] * W.y[i];
        }
        for (int j = tid; j < n; j += kDenseThreads) {
            const double xj = W.x[j], zj = W.z[j];
            double acc = W.c[j] - zj;
            for (int q = P.At_ptr[j]; q < P.At_ptr[j + 1]; ++q) acc -= P.At_val[q] * W.y[P.At_idx[q]];
            const double rxj = frcpd(xj);
            double t = zj * rxj + (xj > 1.0 ? reg * rxj * rxj : reg);
            if (j < nb) {
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
        pmax = cta_max(pmax, W.red);
        dmax = cta_max(dmax, W.red);
        musum = cta_sum(musum, W.red);
        po = cta_sum(po, W.red);
        dobj = cta_sum(dobj, W.red);
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
        // ---- assemble the lower tiles of M = A D A' (padding rows: decoupled unit rows) and factor them
        for (long long e = tid; e < ntd; e += kDenseThreads) W.G[e] = 0.0;
        __syncthreads();
        for (int e = tid; e < P.nent; e += kDenseThreads) {
            double acc = 0.0;
            for (int q = P.asm_ptr[e]; q < P.asm_ptr[e + 1]; ++q) acc += P.asm_val[q] * W.d[P.asm_col[q]];
            W.G[P.asm_pos[e]] = acc;
        }
        for (int i = m + tid; i < mp; i += kDenseThreads)
            W.G[(long long)dense::tile_index(i / dense::TS, i / dense::TS) * dense::TILE + (i % dense::TS) * (dense::TS + 1)] = 1.0;
        dense::factor(W.G, nt, W.SA, W.SB, W.dinv, warp, kDenseWarps, lane);
        // ---- affine predictor
        dense_newton<false>(W, P, 0.0, tid);
        double ip = 0.0, id = 0.0;
        dense_step_pass<false>(W, P, 0.0, tid, ip, id);
        ip = cta_max(ip, W.red); id = cta_max(id, W.red);
        double ap = ip > 1.0 ? 1.0 / ip : 1.0, ad = id > 1.0 ? 1.0 / id : 1.0;
        double mua = 0.0;
        for (int j = tid; j < n; j += kDenseThreads) {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j];
            const double dzj = -zj - zj * dxj * W.rx[j];
            mua += (xj + ap * dxj) * (zj + ad * dzj);
            W.cor[j] = dxj * dzj;
            if (j < nb) {
                const double sj = W.s[j], wj = W.wv[j];
                const double dsj = W.ru[j] - dxj;
                const double dwj = -wj - wj * dsj * W.rs[j];
                mua += (sj + ap * dsj) * (wj + ad * dwj);
                W.cors[j] = dsj * dwj;
            }
        }
        mua = cta_sum(mua, W.red) / ntot;
        const double sg = mua / mu;
        const double smu = sg * sg * sg * mu;
        // ---- centring corrector
        dense_newton<true>(W, P, smu, tid);
        ip = 0.0; id = 0.0;
        dense_step_pass<true>(W, P, smu, tid, ip, id);
        ip = cta_max(ip, W.red); id = cta_max(id, W.red);
        ap = step_frac < ip ? step_frac / ip : 1.0;
        ad = step_frac < id ? step_frac / id : 1.0;
        for (int j = tid; j < n; j += kDenseThreads) {
            const double xj = W.x[j], zj = W.z[j], dxj = W.dx[j], rxj = W.rx[j];
            const double dzj = (smu - W.cor[j]) * rxj - zj - zj * dxj * rxj;
            if (j < nb) {
                const double sj = W.s[j], wj = W.wv[j], rsj = W.rs[j];
                const double dsj = W.ru[j] - dxj;
                const double dwj = (smu - W.cors[j]) * rsj - wj - wj * dsj * rsj;
                W.s[j] = sj + ap * dsj;
                W.wv[j] = wj + ad * dwj;
            }
            W.x[j] = xj + ap * dxj;
            W.z[j] = zj + ad * dzj;
        }
        for (int i = tid; i < m; i += kDenseThreads) W.y[i] += ad * W.dy[i];
        __syncthreads();
    }
    // ---- results
    if (tid == 0) {
        P.obj[p] = pobj * beta_b * beta_c + kconst;
        P.status[p] = status;
        P.iters[p] = it + it0;
    }
    if (P.x_out) {
        double *xo = P.x_out + p * (long long)n;
        if (P.xperm) { for (int j = tid; j < n; j += kDenseThreads) xo[P.xperm[j]] = W.x[j] * beta_b; }
        else { for (int j = tid; j < n; j += kDenseThreads) xo[j] = W.x[j] * beta_b; }
    }
    if (P.y_out) {
        double *yo = P.y_out + p * (long long)m;
        if (P.yperm) { for (int i = tid; i < m; i += kDenseThreads) yo[P.yperm[i]] = W.y[i] * beta_c; }
        else { for (int i = tid; i < m; i += kDenseThreads) yo[i] = W.y[i] * beta_c; }
    }
    __syncthreads();
    *status_out = status;
    *iters_out = it + it0;
}

__global__ void __launch_bounds__(kDenseThreads, 1) dsp_ipm_dense_kernel(const DParams P) {
    extern __shared__ __align__(16) double dsm[];
    unsigned long long &ticket = *(unsigned long long *)(dsm + kDenseWarps);     // behind the reduction slots
    DWork W;
    W.red = dsm;
    W.SA = dsm + 2 * kDenseWarps;
    W.SB = W.SA + dense::TS * dense::LDS;
    const int n = P.n, nb = P.nb, m = P.m, mp = P.nt * dense::TS;
    W.G = P.ws + (long long)blockIdx.x * P.cta_doubles;
    double *base = P.vec_in_smem ? W.SB + dense::TS * dense::LDS : W.G + dense::tiles_doubles(P.nt);
    W.x = base; W.z = W.x + n; W.c = W.z + n; W.rd = W.c + n; W.d = W.rd + n; W.dx = W.d + n; W.cor = W.dx + n; W.rx = W.cor + n;
    W.s = W.rx + n; W.wv = W.s + nb; W.u = W.wv + nb; W.ru = W.u + nb; W.cors = W.ru + nb; W.rs = W.cors + nb;
    W.y = W.rs + nb; W.b = W.y + m; W.rp = W.b + m;
    W.dy = W.rp + m; W.dinv = W.dy + mp;
    for (;;) {
        if (threadIdx.x == 0) ticket = atomicAdd(P.ticket, 1ULL);
        __syncthreads();
        const unsigned long long t = ticket;
        __syncthreads();
        if ((long long)t >= P.N) break;
        int st, it0 = 0;
        // second attempt (shorter step, stronger proximal term) for the rare LP whose first attempt ends non-optimal
        dense_solve_one(W, P, (long long)t, P.step_frac, P.reg, 0, &st, &it0);
        if (st != DSP_OPTIMAL) dense_solve_one(W, P, (long long)t, 0.99, 10.0 * P.reg, it0, &st, &it0);
    }
}

}  // namespace

namespace {
#include "dsp_stage_wb.cuh"

// stage kernel: one warp per LP, one lane per period, all state in registers (see dsp_stage_wb.cuh)
constexpr int kStageWarps = 4;          // warps per CTA
constexpr int kStageMinBlocks = 3;      // CTAs per SM the register allocation must allow
__global__ void __launch_bounds__(32 * kStageWarps, kStageMinBlocks) dsp_ipm_stage_wb_kernel(const KParams P, const stagewb::StageParams S) {
    const int lane = threadIdx.x & 31;
    stagewb::Out O;
    O.obj = P.obj; O.x_out = P.x_out; O.y_out = P.y_out; O.status = P.status; O.iters = P.iters; O.n = P.n; O.m = P.m;
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1ULL);
        t = __shfl_sync(0xffffffffu, t, 0);
        if ((long long)t >= P.N) break;
        const double *cp = P.cparams + (long long)t * P.Pc;
        const double *rp = P.rparams + (long long)t * P.rstride;
        double kconst = 0.0;
        for (int r = lane; r < P.Pr; r += 32) kconst += P.omap[r] * rp[r];
        for (int r = lane; r < P.Pc; r += 32) kconst += P.ocmap[r] * cp[r];
        kconst = stagewb::wsum(kconst) + P.o0;
        // second attempt with a shorter step and a stronger proximal term for the (1 in 1e5) LPs whose first attempt ends
        // non-optimal: the rounding floor of the last iterations differs from LP to LP
        int it0 = 0;
        for (int attempt = 0; attempt < 2; ++attempt) {
            const double sf = attempt ? 0.99 : P.step_frac, rg = attempt ? 10.0 * P.reg : P.reg;
            const int r = stagewb::solve_one(S, cp, rp, kconst, (long long)t, P.tol, P.feas_tol, sf, rg, P.max_iter, O, lane, it0);
            if (r == 0) break;
            it0 = r - 1;
        }
    }
}

}  // namespace

#include "dsp_stage2.cuh"

namespace {
// stage kernel, generation 2: 32/L LPs per warp, P periods per lane, one warp per CTA (see dsp_stage2.cuh).  The register
// budget is the full 255 (65536 / (7 CTAs x 32 threads) = 292): occupancy is set by the 31 KB of shared memory per warp.
constexpr int kStage2Warps = 8;     // warps per CTA = per SM: 8 x 27.9 KB of shared memory, 8 x 32 x 255 registers.  (A ninth
                                    // warp does not fit the register file, which is per scheduler: a third warp on one of the
                                    // four caps every thread at 168 registers -- 2 KB of spills)
// warps per CTA (= per SM) of the chain kernel: what shared memory allows at 168 registers per thread (three warps on a scheduler).
// NF = 2 (19.5 KB per warp): 11 warps -- 2 904 group slots at L = 16 on the 132 SMs of an H100, so the 5 000 LPs of C3 are two
// waves instead of the three they are at 8 warps / 219 registers; NF = 3 (24.8 KB per warp): 8
constexpr int chain1_warps(int NF) { return NF == 2 ? 11 : 8; }
template <int L, int P>
__global__ void __launch_bounds__(32 * kStage2Warps, 1) dsp_ipm_stage2_wb_kernel(const stage2::Params Q) {
    extern __shared__ __align__(16) double s2_smem[];
    stage2::warp_body<L, P>(Q, s2_smem + (threadIdx.x >> 5) * stage2::SmemDoubles<P>::value, threadIdx.x & 31);
}

}  // namespace

#include "dsp_stage_chain1.cuh"
#include "dsp_stage2_long.cuh"

namespace {
// descriptor-driven stage kernel of the single-storage-chain family (dsp_stage_chain1.cuh): same CTA shape as stage2
template <int L, int P, int NF>
__global__ void __launch_bounds__(32 * chain1_warps(NF), 1) dsp_ipm_stage_chain1_kernel(const chain1::Params Q) {
    extern __shared__ __align__(16) double s2_smem[];
    chain1::warp_body<L, P, NF>(Q, s2_smem + (threadIdx.x >> 5) * chain1::Smem<NF, P>::doubles_per_warp, threadIdx.x & 31);
}
inline int chain1_lanes(int T) { return T <= 12 ? 4 : T <= 24 ? 8 : T <= 48 ? 16 : 32; }
constexpr int kChain1MaxT = 96;

// long horizons (T > 96) of the wind+battery structure: one warp per LP, state in a global workspace (dsp_stage2_long.cuh)
constexpr int kLongWarps = 4;
__global__ void __launch_bounds__(32 * kLongWarps) dsp_ipm_stage2_long_kernel(const stage2long::LongParams LQ) {
    stage2long::warp_body_long(LQ, blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), threadIdx.x & 31);
}

struct Stage2Geom { int L, P; };
inline Stage2Geom stage2_geometry(int T) {
    if (T <= 6) return {2, 3};
    if (T <= 12) return {4, 3};
    if (T <= 24) return {8, 3};
    if (T <= 32) return {16, 2};
    if (T <= 48) return {16, 3};
    return {32, 3};                  // T <= 96
}
constexpr int kStage2MaxT = 96;

// FP64 FMA micro-benchmark: the measured denominator of the FP64 roofline fraction bench.py reports.  8 independent DFMA
// chains per thread.
__global__ void __launch_bounds__(256) dsp_fp64_peak_kernel(double *out, int iters, double a, double b) {
    double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
    for (int i = 0; i < iters; ++i) {
        x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b);
        x4 = fma(x4, a, b); x5 = fma(x5, a, b); x6 = fma(x6, a, b); x7 = fma(x7, a, b);
    }
    const double r = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
    if (r == 123.456) out[0] = r;      // never true: keeps the chains alive
}

// =====================================================================================================
// host side
// =====================================================================================================
thread_local std::string g_err;
std::mutex g_mu;
int64_t g_launches = 0;
int g_last_grid = 0, g_last_block = 0, g_last_smem = 0, g_last_ppc = 0;

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess) {                                                              \
            g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                       \
            return DSP_E_CUDA;                                                                \
        }                                                                                     \
    } while (0)

template <class T>
int upload(const std::vector<T> &h, T **d) {
    *d = nullptr;
    size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(T);
    CK(cudaMalloc((void **)d, bytes));
    if (!h.empty()) {
        cudaError_t e_ = cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
        if (e_ != cudaSuccess) { cudaFree(*d); *d = nullptr; g_err = std::string("cudaMemcpy: ") + cudaGetErrorString(e_); return DSP_E_CUDA; }
    }
    return 0;
}

}  // namespace

struct dsp_template {
    KParams kp;
    bool has_stage;
    mutable double *ws;            // global workspace for templates whose work region exceeds shared memory
    mutable size_t ws_bytes;
    stagewb::StageParams sp;
    int stage_blocks_per_sm;
    bool has_chain1;               // descriptor-driven single-storage-chain stage kernel registered
    int c1_T, c1_NF;
    const int *c1_col_idx, *c1_row_idx;
    const double *c1_coef, *c1_coef_next;
    int device;
    int sm_count;
    int smem_optin;
    size_t ws_cap;                 // largest global workspace a launch may allocate: a quarter of device memory
    std::vector<void *> dev_allocs;
    std::vector<int> col_perm, row_perm;     // dsp_lp_template_create_csr: caller index of internal column / row
    std::vector<int> csr_ptr, csr_idx, asm_qa, asm_qb;   // permuted CSR pattern + assembly factor positions (kept for matrix parameters)
    unsigned long long *ticket;
    // host-call staging (pinned) and device buffers, grown on demand
    int64_t cap_N;
    double *h_cp, *h_rp, *h_obj, *h_x, *h_y;
    int32_t *h_status, *h_iters;
    double *d_cp, *d_rp, *d_obj, *d_x, *d_y;
    int32_t *d_status, *d_iters;
    bool cap_x, cap_y;
    int64_t cap_rp_rows;
    cudaStream_t stream, stream2;
    std::atomic<int> busy;         // a host call is in flight on this handle (staging buffers, streams and ticket are per handle)
    bool dense_only;               // made by dsp_lp_template_create_dense: no band data, only the dense kernel runs
    struct Dense {                 // the dense kernel's data (dense templates; band templates: built at the first DSP_KERNEL_DENSE call)
        bool ready;
        int nt, nent;
        const int *A_ptr, *A_idx, *At_ptr, *At_idx, *asm_pos, *asm_ptr, *asm_col;
        const double *A_val, *At_val, *asm_val;
    };
    mutable Dense dn;
};

namespace {
// The kernel instantiation of each family for a geometry.  Launches and cudaFuncSetAttribute calls both look it up here.
using BandKernel = void (*)(KParams);
using Stage2Kernel = void (*)(stage2::Params);
using Chain1Kernel = void (*)(chain1::Params);

// band kernel for half bandwidth W and a placement: work regions in the global workspace (ws) or in shared memory, with the
// template staged into shared memory (hot_in_smem) or read through L2
template <int W>
BandKernel band_kernel_w(bool ws, bool hot_in_smem) {
    return ws ? dsp_ipm_band_kernel<W, true, false> : hot_in_smem ? dsp_ipm_band_kernel<W, false, true> : dsp_ipm_band_kernel<W, false, false>;
}
BandKernel band_kernel(int w, bool ws, bool hot_in_smem) {
    switch (w) {
        case 1: return band_kernel_w<1>(ws, hot_in_smem);
        case 2: return band_kernel_w<2>(ws, hot_in_smem);
        case 4: return band_kernel_w<4>(ws, hot_in_smem);
        case 8: return band_kernel_w<8>(ws, hot_in_smem);
        case 16: return band_kernel_w<16>(ws, hot_in_smem);
        default: return band_kernel_w<32>(ws, hot_in_smem);
    }
}

Stage2Kernel stage2_kernel(const Stage2Geom &g) {
    if (g.L == 2) return dsp_ipm_stage2_wb_kernel<2, 3>;
    if (g.L == 4) return dsp_ipm_stage2_wb_kernel<4, 3>;
    if (g.L == 8) return dsp_ipm_stage2_wb_kernel<8, 3>;
    if (g.L == 16) return g.P == 2 ? dsp_ipm_stage2_wb_kernel<16, 2> : dsp_ipm_stage2_wb_kernel<16, 3>;
    return dsp_ipm_stage2_wb_kernel<32, 3>;
}
size_t stage2_smem_bytes(const Stage2Geom &g) {
    return (size_t)(g.P == 2 ? stage2::smem_doubles_per_warp<2>() : stage2::smem_doubles_per_warp<3>()) * 8;
}

template <int NF>
Chain1Kernel chain1_kernel_nf(int L) {
    return L == 4 ? dsp_ipm_stage_chain1_kernel<4, 3, NF> : L == 8 ? dsp_ipm_stage_chain1_kernel<8, 3, NF>
         : L == 16 ? dsp_ipm_stage_chain1_kernel<16, 3, NF> : dsp_ipm_stage_chain1_kernel<32, 3, NF>;
}
Chain1Kernel chain1_kernel(int L, int NF) { return NF == 2 ? chain1_kernel_nf<2>(L) : chain1_kernel_nf<3>(L); }
size_t chain1_smem_bytes(int NF) {
    return (size_t)(NF == 2 ? chain1::Smem<2, 3>::doubles_per_warp : chain1::Smem<3, 3>::doubles_per_warp) * 8;
}

// lets a stage kernel use `bytes` of dynamic shared memory, with the largest carveout
template <class F>
int allow_smem(F fn, size_t bytes) {
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    return 0;
}

int check_maps(const dsp_template_desc *D) {
    for (int q = 0; q < D->cmap.ptr[D->n]; ++q)
        if (D->cmap.idx[q] < 0 || D->cmap.idx[q] >= D->Pc) { g_err = "cmap.idx out of range"; return DSP_E_ARG; }
    for (int q = 0; q < D->bmap.ptr[D->m]; ++q)
        if (D->bmap.idx[q] < 0 || D->bmap.idx[q] >= D->Pr) { g_err = "bmap.idx out of range"; return DSP_E_ARG; }
    for (int q = 0; q < D->umap.ptr[D->nb]; ++q)
        if (D->umap.idx[q] < 0 || D->umap.idx[q] >= D->Pr) { g_err = "umap.idx out of range"; return DSP_E_ARG; }
    return 0;
}

// what every template carries whatever its kernels: the device and its limits, the streams, the ticket counter and the
// parameter maps of c, b, u and the objective constant (D's matrix and assembly fields are not read)
int template_init(dsp_template *T, const dsp_template_desc *D) {
    const int m = D->m, n = D->n, nb = D->nb;
    memset(&T->kp, 0, sizeof(KParams));
    T->cap_N = 0; T->cap_x = T->cap_y = false; T->cap_rp_rows = 0;
    T->has_stage = false; T->has_chain1 = false; T->stage_blocks_per_sm = 0; T->ws = nullptr; T->ws_bytes = 0;
    T->h_cp = T->h_rp = T->h_obj = T->h_x = T->h_y = nullptr; T->h_status = T->h_iters = nullptr;
    T->d_cp = T->d_rp = T->d_obj = T->d_x = T->d_y = nullptr; T->d_status = T->d_iters = nullptr;
    T->stream = nullptr; T->stream2 = nullptr; T->busy.store(0);
    T->dense_only = false;
    memset(&T->dn, 0, sizeof(T->dn));
    CK(cudaGetDevice(&T->device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, T->device));
    T->sm_count = prop.multiProcessorCount;
    T->smem_optin = (int)prop.sharedMemPerBlockOptin;
    T->ws_cap = prop.totalGlobalMem / 4;
    KParams &K = T->kp;
    K.m = m; K.n = n; K.nb = nb; K.Pc = D->Pc; K.Pr = D->Pr;
    K.o0 = D->o0;
    auto up_d = [&](const double *src, size_t cnt, const double **dst) -> int {
        std::vector<double> v(src, src + cnt);
        double *d;
        int rc = upload(v, &d);
        if (rc) return rc;
        T->dev_allocs.push_back(d);
        *dst = d;
        return 0;
    };
    auto up_i = [&](const int32_t *src, size_t cnt, const int **dst) -> int {
        std::vector<int> v(src, src + cnt);
        int *d;
        int rc = upload(v, &d);
        if (rc) return rc;
        T->dev_allocs.push_back(d);
        *dst = d;
        return 0;
    };
    int rc = 0;
    rc |= up_d(D->c0, n, &K.c0);
    rc |= up_d(D->b0, m, &K.b0);
    rc |= up_d(D->u0, nb, &K.u0);
    rc |= up_d(D->omap, D->Pr, &K.omap);
    rc |= up_d(D->ocmap, D->Pc, &K.ocmap);
    rc |= up_i(D->cmap.ptr, n + 1, &K.cm_ptr);
    rc |= up_i(D->cmap.idx, D->cmap.ptr[n], &K.cm_idx);
    rc |= up_d(D->cmap.val, D->cmap.ptr[n], &K.cm_val);
    rc |= up_i(D->bmap.ptr, m + 1, &K.bm_ptr);
    rc |= up_i(D->bmap.idx, D->bmap.ptr[m], &K.bm_idx);
    rc |= up_d(D->bmap.val, D->bmap.ptr[m], &K.bm_val);
    rc |= up_i(D->umap.ptr, nb + 1, &K.um_ptr);
    rc |= up_i(D->umap.idx, D->umap.ptr[nb], &K.um_idx);
    rc |= up_d(D->umap.val, D->umap.ptr[nb], &K.um_val);
    if (rc) return DSP_E_CUDA;
    CK(cudaMalloc((void **)&T->ticket, 16 * sizeof(unsigned long long)));
    T->dev_allocs.push_back(T->ticket);
    CK(cudaStreamCreateWithFlags(&T->stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&T->stream2, cudaStreamNonBlocking));
    return 0;
}

// The dense kernel's data for a template whose internal-order CSR is (A_ptr, A_idx, A_val): the CSC, and the assembly list of the
// lower pattern of A A' in tile-major workspace order -- entry e of M sits at asm_pos[e] and is the sum of
// asm_val[q] * d[asm_col[q]] over q in [asm_ptr[e], asm_ptr[e+1]).  Host-only analysis, then one upload.
constexpr long long kDenseMaxTerms = 1LL << 26;
int dense_build(dsp_template *T, const std::vector<int> &A_ptr, const std::vector<int> &A_idx, const std::vector<double> &A_val) {
    const int m = T->kp.m, n = T->kp.n, nnz = A_ptr[m];
    const int TS = dense::TS;
    std::vector<int> At_ptr(n + 1, 0), At_idx(nnz);
    std::vector<double> At_val(nnz);
    for (int q = 0; q < nnz; ++q) At_ptr[A_idx[q] + 1]++;
    for (int j = 0; j < n; ++j) At_ptr[j + 1] += At_ptr[j];
    {
        std::vector<int> fill(At_ptr.begin(), At_ptr.end() - 1);
        for (int i = 0; i < m; ++i)
            for (int q = A_ptr[i]; q < A_ptr[i + 1]; ++q) { const int dst = fill[A_idx[q]]++; At_idx[dst] = i; At_val[dst] = A_val[q]; }
    }
    long long nterms = 0;
    for (int j = 0; j < n; ++j) { const long long c = At_ptr[j + 1] - At_ptr[j]; nterms += c * (c + 1) / 2; }
    if (nterms > kDenseMaxTerms) { g_err = "dense kernel: the assembly list of A A' has more than 2^26 products"; return DSP_E_ARG; }
    // entries of the lower pattern (a >= b), first seen order; then sorted by workspace position
    std::vector<int> slot((size_t)m * m, -1), cnt;
    std::vector<long long> pos;
    for (int j = 0; j < n; ++j)
        for (int qa = At_ptr[j]; qa < At_ptr[j + 1]; ++qa)
            for (int qb = At_ptr[j]; qb <= qa; ++qb) {
                const int a = At_idx[qa], b = At_idx[qb];      // rows ascending within a column: a >= b
                int &e = slot[(size_t)a * m + b];
                if (e < 0) {
                    e = (int)pos.size();
                    pos.push_back((long long)dense::tile_index(a / TS, b / TS) * dense::TILE + (a % TS) * TS + (b % TS));
                    cnt.push_back(0);
                }
                cnt[e]++;
            }
    const int nent = (int)pos.size();
    std::vector<int> order(nent), rank(nent);
    for (int e = 0; e < nent; ++e) order[e] = e;
    std::sort(order.begin(), order.end(), [&](int x, int y) { return pos[x] < pos[y]; });
    for (int r = 0; r < nent; ++r) rank[order[r]] = r;
    std::vector<int> asm_pos(nent), asm_ptr(nent + 1, 0), asm_col((size_t)nterms);
    std::vector<double> asm_val((size_t)nterms);
    for (int r = 0; r < nent; ++r) { asm_pos[r] = (int)pos[order[r]]; asm_ptr[r + 1] = asm_ptr[r] + cnt[order[r]]; }
    std::vector<int> fill(asm_ptr.begin(), asm_ptr.end() - 1);
    for (int j = 0; j < n; ++j)
        for (int qa = At_ptr[j]; qa < At_ptr[j + 1]; ++qa)
            for (int qb = At_ptr[j]; qb <= qa; ++qb) {
                const int r = rank[slot[(size_t)At_idx[qa] * m + At_idx[qb]]];
                asm_col[fill[r]] = j;
                asm_val[fill[r]++] = At_val[qa] * At_val[qb];
            }
    dsp_template::Dense &D = T->dn;
    int *pi; double *pd;
    auto ui = [&](const std::vector<int> &v, const int **dst) { int rc = upload(v, &pi); if (!rc) { T->dev_allocs.push_back(pi); *dst = pi; } return rc; };
    auto ud = [&](const std::vector<double> &v, const double **dst) { int rc = upload(v, &pd); if (!rc) { T->dev_allocs.push_back(pd); *dst = pd; } return rc; };
    int rc = 0;
    rc = rc ? rc : ui(A_ptr, &D.A_ptr);
    rc = rc ? rc : ui(A_idx, &D.A_idx);
    rc = rc ? rc : ud(A_val, &D.A_val);
    rc = rc ? rc : ui(At_ptr, &D.At_ptr);
    rc = rc ? rc : ui(At_idx, &D.At_idx);
    rc = rc ? rc : ud(At_val, &D.At_val);
    rc = rc ? rc : ui(asm_pos, &D.asm_pos);
    rc = rc ? rc : ui(asm_ptr, &D.asm_ptr);
    rc = rc ? rc : ui(asm_col, &D.asm_col);
    rc = rc ? rc : ud(asm_val, &D.asm_val);
    if (rc) return rc;
    CK(cudaFuncSetAttribute(dsp_ipm_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T->smem_optin));
    D.nt = (m + TS - 1) / TS;
    D.nent = nent;
    D.ready = true;
    return 0;
}
}  // namespace

extern "C" {

static void free_staging(dsp_template *T);

const char *dsp_lp_version(void) { return DSP_VERSION; }

double dsp_lp_fp64_peak_tflops(void) {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1.0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    double *d = nullptr;
    if (cudaMalloc((void **)&d, 8) != cudaSuccess) return -1.0;
    const int iters = 8192, blocks = sms * 8, threads = 256;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    dsp_fp64_peak_kernel<<<blocks, threads>>>(d, 64, 0.999999, 1e-9);       // warm-up
    float best = 1e30f;
    for (int rep = 0; rep < 5; ++rep) {
        cudaEventRecord(e0);
        dsp_fp64_peak_kernel<<<blocks, threads>>>(d, iters, 0.999999, 1e-9);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        best = ms < best ? ms : best;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
    if (cudaGetLastError() != cudaSuccess) return -1.0;
    const double flops = 2.0 * 8.0 * (double)iters * (double)blocks * (double)threads;
    return flops / (best * 1e-3) / 1e12;
}
#ifdef DSP_PHASES
int dsp_lp_phases(unsigned long long *out16, int reset) {
    cudaMemcpyFromSymbol(out16, g_phase, sizeof(unsigned long long) * 16);
    if (reset) { unsigned long long z[16] = {0}; cudaMemcpyToSymbol(g_phase, z, sizeof(z)); }
    return 0;
}
#endif
const char *dsp_lp_last_error(void) { return g_err.c_str(); }
int64_t dsp_lp_launch_count(void) { return g_launches; }
int dsp_lp_last_launch(int32_t *grid, int32_t *block, int32_t *smem_bytes, int32_t *ppc) {
    if (grid) *grid = g_last_grid;
    if (block) *block = g_last_block;
    if (smem_bytes) *smem_bytes = g_last_smem;
    if (ppc) *ppc = g_last_ppc;
    return 0;
}

void dsp_lp_default_opts(dsp_opts *o) {
    o->tol = 1e-9;
    o->feas_tol = 1e-9;
    o->max_iter = 60;
    o->step_frac = 0.9995;
    o->device = -1;
    o->reg_primal = 1e-8;
    o->kernel = DSP_KERNEL_AUTO;
}

int dsp_lp_template_create(const dsp_template_desc *D, dsp_template **out) {
    if (!D || !out || D->m <= 0 || D->n <= 0 || D->nb < 0 || D->nb > D->n || D->w < 0 || D->w >= D->m + 1) {
        g_err = "dsp_lp_template_create: bad dimensions";
        return DSP_E_ARG;
    }
    const int m = D->m, n = D->n, nb = D->nb, w = D->w;
    const int nnz = D->A_ptr[m];
    // the kernels are instantiated for half bandwidths 1, 2, 4, 8, 16, 32: pad the band storage to the next one
    int wt = 1;
    while (wt < w) wt *= 2;
    if (wt > 32) { g_err = "dsp_lp_template_create: half bandwidth of A*A' above 32 is not supported"; return DSP_E_ARG; }
    const int nent = m * (wt + 1);
    const int nasm = D->asm_ptr[m * (w + 1)];
    std::vector<int> asm_ptr_pad(nent + 1, 0);
    for (int i = 0; i < m; ++i)
        for (int k = 0; k <= wt; ++k) {
            const int cnt = (k <= w) ? D->asm_ptr[i * (w + 1) + k + 1] - D->asm_ptr[i * (w + 1) + k] : 0;
            asm_ptr_pad[i * (wt + 1) + k + 1] = asm_ptr_pad[i * (wt + 1) + k] + cnt;
        }
    for (int q = 0; q < nasm; ++q)
        if (D->asm_col[q] < 0 || D->asm_col[q] >= n) { g_err = "asm_col out of range"; return DSP_E_ARG; }
    if (int rc = check_maps(D)) return rc;
    // CSC of A
    std::vector<int> At_ptr(n + 1, 0), At_idx(nnz);
    std::vector<double> At_val(nnz);
    for (int q = 0; q < nnz; ++q) {
        if (D->A_idx[q] < 0 || D->A_idx[q] >= n) { g_err = "A_idx out of range"; return DSP_E_ARG; }
        At_ptr[D->A_idx[q] + 1]++;
    }
    for (int j = 0; j < n; ++j) At_ptr[j + 1] += At_ptr[j];
    {
        std::vector<int> fill(At_ptr.begin(), At_ptr.end() - 1);
        for (int i = 0; i < m; ++i)
            for (int q = D->A_ptr[i]; q < D->A_ptr[i + 1]; ++q) {
                int dst = fill[D->A_idx[q]]++;
                At_idx[dst] = i;
                At_val[dst] = D->A_val[q];
            }
    }
    // hot blob
    size_t dbl = (size_t)nnz * 2 + nasm;
    size_t ints = (size_t)(m + 1) + nnz + (n + 1) + nnz + (nent + 1) + nasm;
    size_t hot_bytes = dbl * 8 + ints * 4;
    hot_bytes = (hot_bytes + 15) / 16 * 16;
    std::vector<unsigned char> hot(hot_bytes, 0);
    {
        double *pd = (double *)hot.data();
        memcpy(pd, D->A_val, (size_t)nnz * 8); pd += nnz;
        memcpy(pd, At_val.data(), (size_t)nnz * 8); pd += nnz;
        memcpy(pd, D->asm_val, (size_t)nasm * 8); pd += nasm;
        int *pi = (int *)pd;
        memcpy(pi, D->A_ptr, (size_t)(m + 1) * 4); pi += m + 1;
        memcpy(pi, D->A_idx, (size_t)nnz * 4); pi += nnz;
        memcpy(pi, At_ptr.data(), (size_t)(n + 1) * 4); pi += n + 1;
        memcpy(pi, At_idx.data(), (size_t)nnz * 4); pi += nnz;
        memcpy(pi, asm_ptr_pad.data(), (size_t)(nent + 1) * 4); pi += nent + 1;
        memcpy(pi, D->asm_col, (size_t)nasm * 4);
    }
    dsp_template *T = new dsp_template();
    struct Guard {      // every error return below releases the handle and its device allocations
        dsp_template *t;
        ~Guard() { if (t) dsp_lp_template_destroy(t); }
    } guard{T};
    if (int rc = template_init(T, D)) return rc;
    KParams &K = T->kp;
    K.w = wt; K.nnz = nnz; K.nasm = nasm;
    K.hot_bytes = (int)hot_bytes;
    {
        unsigned char *d;
        int rc = upload(hot, &d);
        if (rc) return rc;
        T->dev_allocs.push_back(d);
        K.hot_g = d;
    }
    K.band_doubles = (m + 2 * wt) + (m + 2 * wt) * (wt + 1);
    K.prob_doubles = 8 * n + 6 * nb + 3 * m + K.band_doubles;
    K.hybrid = 0;
    for (int bw = 1; bw <= 32; bw *= 2)
        for (int placement = 0; placement < 3; ++placement)       // workspace, shared memory + staged template, shared memory
            CK(cudaFuncSetAttribute(band_kernel(bw, placement == 0, placement == 1), cudaFuncAttributeMaxDynamicSharedMemorySize, T->smem_optin));
    guard.t = nullptr;
    *out = T;
    return 0;
}

int dsp_lp_template_set_stage_wb(dsp_template *T, const dsp_stage_wb_desc *d) {
    if (!T || !d || d->T < 1) { g_err = "dsp_lp_template_set_stage_wb: need T >= 1"; return DSP_E_ARG; }
    if (T->kp.Pc < d->T || T->kp.Pr <= std::max(d->wcf_off + d->T - 1, d->p_off)) {
        g_err = "dsp_lp_template_set_stage_wb: parameter layout does not fit the template";
        return DSP_E_ARG;
    }
    stagewb::StageParams &S = T->sp;
    S.T = d->T; S.a = d->a; S.binv = d->binv; S.hf = d->half; S.dl = d->delta; S.dur = d->dur; S.krev = d->k_rev;
    S.wcf_off = d->wcf_off; S.p_off = d->p_off;
    std::vector<int> ci(d->col_idx, d->col_idx + 7 * d->T), ri(d->row_idx, d->row_idx + 4 * d->T);
    for (int v : ci) if (v < -1 || v >= T->kp.n) { g_err = "col_idx out of range"; return DSP_E_ARG; }
    for (int v : ri) if (v < 0 || v >= T->kp.m) { g_err = "row_idx out of range"; return DSP_E_ARG; }
    int *dci, *dri;
    int rc = upload(ci, &dci); if (rc) return rc;
    rc = upload(ri, &dri); if (rc) return rc;
    T->dev_allocs.push_back(dci); T->dev_allocs.push_back(dri);
    S.col_idx = dci; S.row_idx = dri;
    int nb = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, dsp_ipm_stage_wb_kernel, 32 * kStageWarps, 0));
    T->stage_blocks_per_sm = std::max(nb, 1);
    if (d->T <= kStage2MaxT) {
        const Stage2Geom g = stage2_geometry(d->T);
        rc = allow_smem(stage2_kernel(g), stage2_smem_bytes(g) * kStage2Warps);
        if (rc) return rc;
    }
    T->has_stage = true;
    return 0;
}

int dsp_lp_template_set_stage_chain1(dsp_template *T, const dsp_stage_chain1_desc *d) {
    if (!T || !d || d->T < 1 || d->T > kChain1MaxT || d->NF < 2 || d->NF > 3) {
        g_err = "dsp_lp_template_set_stage_chain1: need 1 <= T <= 96 and NF = 2 or 3 (pad absent flows with col_idx = -1)";
        return DSP_E_ARG;
    }
    if (d->T != T->kp.m) { g_err = "dsp_lp_template_set_stage_chain1: one row per period expected (T == m)"; return DSP_E_ARG; }
    const int NC = d->NF + 1;
    std::vector<int> ci(d->col_idx, d->col_idx + (size_t)d->T * NC), ri(d->row_idx, d->row_idx + d->T);
    std::vector<char> seen(T->kp.n, 0);
    for (int v : ci) {
        if (v < -1 || v >= T->kp.n) { g_err = "chain1: col_idx out of range"; return DSP_E_ARG; }
        if (v >= 0) { if (seen[v]) { g_err = "chain1: a column is listed twice"; return DSP_E_ARG; } seen[v] = 1; }
    }
    for (int j = 0; j < T->kp.n; ++j) if (!seen[j]) { g_err = "chain1: every template column must be listed"; return DSP_E_ARG; }
    for (int v : ri) if (v < 0 || v >= T->kp.m) { g_err = "chain1: row_idx out of range"; return DSP_E_ARG; }
    // internal (kernel) indices: templates created from plain CSR carry a caller->internal permutation
    std::vector<int> cpos(T->kp.n), rpos(T->kp.m);
    for (int k = 0; k < T->kp.n; ++k) cpos[T->col_perm.empty() ? k : T->col_perm[k]] = k;
    for (int k = 0; k < T->kp.m; ++k) rpos[T->row_perm.empty() ? k : T->row_perm[k]] = k;
    for (int &v : ci) if (v >= 0) v = cpos[v];
    for (int &v : ri) v = rpos[v];
    std::vector<double> cf(d->coef, d->coef + (size_t)d->T * NC), cn(d->coef_next, d->coef_next + d->T);
    int *dci, *dri; double *dcf, *dcn;
    int rc = upload(ci, &dci); if (rc) return rc; T->dev_allocs.push_back(dci);
    rc = upload(ri, &dri); if (rc) return rc; T->dev_allocs.push_back(dri);
    rc = upload(cf, &dcf); if (rc) return rc; T->dev_allocs.push_back(dcf);
    rc = upload(cn, &dcn); if (rc) return rc; T->dev_allocs.push_back(dcn);
    T->c1_T = d->T; T->c1_NF = d->NF;
    T->c1_col_idx = dci; T->c1_row_idx = dri; T->c1_coef = dcf; T->c1_coef_next = dcn;
    rc = allow_smem(chain1_kernel(chain1_lanes(d->T), d->NF), chain1_smem_bytes(d->NF) * chain1_warps(d->NF));
    if (rc) return rc;
    T->has_chain1 = true;
    return 0;
}

void dsp_lp_template_destroy(dsp_template *T) {
    if (!T) return;
    for (void *p : T->dev_allocs) cudaFree(p);
    cudaFree(T->ws);
    free_staging(T);
    if (T->stream) cudaStreamDestroy(T->stream);
    if (T->stream2) cudaStreamDestroy(T->stream2);
    delete T;
}

// Geometry of a band-kernel launch: one persistent CTA per SM, `warps` LPs in flight per CTA, and one of three
// placements of the per-LP work region:
//   smem    everything in shared memory: fastest warp, but only as many LPs per SM as regions fit;
//   hybrid  the (dy, Mb) tail -- all that the LDL' / substitution sweeps touch -- in shared memory, the element-wise
//           vectors in a global workspace (coalesced streaming through L2): a slower warp, but more LPs per SM;
//   ws      everything in the global workspace, kMaxWarps LPs per SM: slower still per warp (L2 latency in the sweeps);
//           the only choice for long horizons (T = 8736).
struct BandGeom { long long warps; int hot_in_smem; size_t off; bool ws; int hybrid; };

BandGeom band_geometry(const dsp_template *T, const KParams &K) {
    const size_t prob_bytes = (size_t)K.prob_doubles * 8;
    const size_t band_bytes = (size_t)K.band_doubles * 8;
    const size_t budget = (size_t)T->smem_optin;
    BandGeom g{0, 1, 16 + (size_t)K.hot_bytes, false, 0};
    long long smem_warps = budget > g.off ? (long long)((budget - g.off) / prob_bytes) : 0;
    if (smem_warps < 4) {   // template too large to stage next to the work regions: read it through L2
        g.hot_in_smem = 0;
        g.off = 16;
        smem_warps = (long long)((budget - g.off) / prob_bytes);
    }
    const long long hybrid_warps = band_bytes + 16 <= budget ? std::min<long long>(kMaxWarps, (long long)((budget - 16) / band_bytes)) : 0;
    enum { M_SMEM, M_HYBRID, M_WS } mode = smem_warps >= 7 ? M_SMEM : hybrid_warps >= 6 ? M_HYBRID : smem_warps >= 4 ? M_SMEM : M_WS;
#ifdef DSP_PHASES
    // instrumentation build only: tools/gpu_band_modes.py forces a placement (DSP_BAND_MODE = smem | hybrid | ws) where it fits
    if (const char *e = getenv("DSP_BAND_MODE")) {
        if (!strcmp(e, "ws")) mode = M_WS;
        else if (!strcmp(e, "hybrid") && hybrid_warps >= 1) mode = M_HYBRID;
        else if (!strcmp(e, "smem") && smem_warps >= 1) mode = M_SMEM;
    }
#endif
    if (mode == M_SMEM) {
        g.warps = smem_warps;
    } else {
        g.ws = true; g.hot_in_smem = 0; g.off = 16;
        g.hybrid = mode == M_HYBRID;
        g.warps = g.hybrid ? hybrid_warps : kMaxWarps;
        while (g.warps > 1 && (size_t)T->sm_count * (size_t)g.warps * prob_bytes > T->ws_cap) g.warps /= 2;
    }
    g.warps = std::min<long long>(g.warps, kMaxWarps);
    return g;
}

// grows the handle's global workspace to at least `need` bytes, once the kernels already queued on the stream are done with it
static int grow_ws(const dsp_template *T, size_t need, cudaStream_t st) {
    if (need <= T->ws_bytes) return 0;
    CK(cudaStreamSynchronize(st));
    cudaFree(T->ws);
    T->ws = nullptr; T->ws_bytes = 0;
    CK(cudaMalloc((void **)&T->ws, need));
    T->ws_bytes = need;
    return 0;
}

// checks the launch just issued and records its geometry for dsp_lp_launch_count / dsp_lp_last_launch
static int launched(long long grid, long long block, size_t smem, long long ppc) {
    CK(cudaGetLastError());
    std::lock_guard<std::mutex> lk(g_mu);
    g_launches++;
    g_last_grid = (int)grid; g_last_block = (int)block; g_last_smem = (int)smem; g_last_ppc = (int)ppc;
    return 0;
}

// parameters of the stage-2 kernels (short and long horizon): the batch in K, the stage structure of the template
static stage2::Params stage2_params(const dsp_template *T, const KParams &K) {
    stage2::Params Q;
    Q.N = K.N; Q.cparams = K.cparams; Q.rparams = K.rparams; Q.rstride = K.rstride; Q.Pc = K.Pc; Q.Pr = K.Pr;
    Q.omap = K.omap; Q.ocmap = K.ocmap; Q.o0 = K.o0;
    Q.tol = K.tol; Q.feas_tol = K.feas_tol; Q.step_frac = K.step_frac; Q.reg = K.reg; Q.max_iter = K.max_iter;
    Q.obj = K.obj; Q.x_out = K.x_out; Q.y_out = K.y_out; Q.status = K.status; Q.iters = K.iters; Q.n = K.n; Q.m = K.m; Q.ticket = K.ticket;
    const stagewb::StageParams &S = T->sp;
    Q.T = S.T; Q.a = S.a; Q.binv = S.binv; Q.hf = S.hf; Q.dl = S.dl; Q.dur = S.dur; Q.krev = S.krev;
    Q.wcf_off = S.wcf_off; Q.p_off = S.p_off; Q.col_idx = S.col_idx; Q.row_idx = S.row_idx;
    Q.ahead = 0;
    return Q;
}

// long horizon (T > 96): one warp per LP, everything in a global workspace owned by the handle
static int launch_stage2_long(const dsp_template *T, const KParams &K, cudaStream_t st) {
    const int P = (T->sp.T + 31) / 32;
    const size_t per_warp = (size_t)stage2long::NW * P * 32 * sizeof(double);
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dsp_ipm_stage2_long_kernel, 32 * kLongWarps, 0));
    long long warps = std::min<long long>(K.N, (long long)T->sm_count * std::max(occ, 1) * kLongWarps);
    while (warps > 1 && (size_t)warps * per_warp > T->ws_cap) warps /= 2;
    // spread the warps over the SMs: one warp per CTA while there are fewer LPs than SMs x kLongWarps
    const int wpb = (int)std::min<long long>(kLongWarps, std::max<long long>(1, warps / T->sm_count));
    const long long blocks = (warps + wpb - 1) / wpb;
    const int rc = grow_ws(T, (size_t)blocks * wpb * per_warp, st);
    if (rc) return rc;
    stage2long::LongParams LQ;
    LQ.q = stage2_params(T, K);
    LQ.ws = T->ws; LQ.P = P;
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    dsp_ipm_stage2_long_kernel<<<(unsigned)blocks, 32 * wpb, 0, st>>>(LQ);
    return launched(blocks, 32 * wpb, 0, wpb);
}

// generation-2 stage kernel: 32/L LPs per warp, persistent CTAs, LP groups refill from the ticket counter
static int launch_stage2(const dsp_template *T, const KParams &K, cudaStream_t st) {
    const Stage2Geom g = stage2_geometry(T->sp.T);
    const int per_warp = 32 / g.L;
    // one persistent CTA per SM; its warps (up to kStage2Warps) run the phases of an IPM round in step
    int wmax = kStage2Warps;
#ifdef DSP_PHASES
    // instrumentation build only: tools/gpu_stage2_phases.py compares fewer warps per CTA (DSP_STAGE2_WARPS)
    if (const char *e = getenv("DSP_STAGE2_WARPS")) wmax = std::min(kStage2Warps, std::max(1, atoi(e)));
    {   // ... and times a second copy of pass 2 in every round (DSP_STAGE2_PASS2_TWICE=1)
        const char *e = getenv("DSP_STAGE2_PASS2_TWICE");
        const int twice = e && atoi(e) ? 1 : 0;
        CK(cudaMemcpyToSymbolAsync(g_pass2_twice, &twice, sizeof(int), 0, cudaMemcpyHostToDevice, st));
    }
#endif
    const long long warps_needed = (K.N + per_warp - 1) / per_warp;
    const long long blocks = std::max<long long>(1, std::min<long long>(T->sm_count, warps_needed));
    const int wpb = (int)std::min<long long>(wmax, (warps_needed + blocks - 1) / blocks);
    const size_t smem = stage2_smem_bytes(g) * wpb;
    stage2::Params Q = stage2_params(T, K);
    Q.ahead = (int)(blocks * wpb * per_warp);
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    stage2_kernel(g)<<<(unsigned)blocks, 32 * wpb, smem, st>>>(Q);
    return launched(blocks, 32 * wpb, smem, per_warp * wpb);
}

// generation-1 stage kernel (lane per period): no shared memory; persistent warps, one LP per warp at a time
static int launch_stage_v1(const dsp_template *T, const KParams &K, cudaStream_t st) {
    if (T->sp.T > 32) { g_err = "dsp_lp_solve_batch: the lane-per-period stage kernel needs T <= 32"; return DSP_E_ARG; }
    const long long blocks = std::min<long long>((long long)T->sm_count * T->stage_blocks_per_sm, (K.N + kStageWarps - 1) / kStageWarps);
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    dsp_ipm_stage_wb_kernel<<<(unsigned)blocks, kStageWarps * 32, 0, st>>>(K, T->sp);
    return launched(blocks, kStageWarps * 32, 0, kStageWarps);
}

// descriptor-driven single-storage-chain stage kernel: the CTA shape of stage 2, chain1_warps(NF) warps at most
static int launch_chain1(const dsp_template *T, const KParams &K, cudaStream_t st) {
    const int L = chain1_lanes(T->c1_T), per_warp = 32 / L, NF = T->c1_NF;
    const long long warps_needed = (K.N + per_warp - 1) / per_warp;
    const long long blocks = std::max<long long>(1, std::min<long long>(T->sm_count, warps_needed));
    const int wpb = (int)std::min<long long>(chain1_warps(NF), (warps_needed + blocks - 1) / blocks);
    const size_t smem = chain1_smem_bytes(NF) * wpb;
    chain1::Params Q;
    Q.N = K.N; Q.cparams = K.cparams; Q.rparams = K.rparams; Q.rstride = K.rstride; Q.Pc = K.Pc; Q.Pr = K.Pr;
    Q.omap = K.omap; Q.ocmap = K.ocmap; Q.o0 = K.o0;
    Q.tol = K.tol; Q.feas_tol = K.feas_tol; Q.step_frac = K.step_frac; Q.reg = K.reg; Q.max_iter = K.max_iter;
    Q.obj = K.obj; Q.x_out = K.x_out; Q.y_out = K.y_out; Q.status = K.status; Q.iters = K.iters; Q.n = K.n; Q.m = K.m; Q.nb = K.nb; Q.ticket = K.ticket;
    Q.c0 = K.c0; Q.b0 = K.b0; Q.u0 = K.u0; Q.cm_ptr = K.cm_ptr; Q.cm_idx = K.cm_idx; Q.cm_val = K.cm_val;
    Q.bm_ptr = K.bm_ptr; Q.bm_idx = K.bm_idx; Q.bm_val = K.bm_val; Q.um_ptr = K.um_ptr; Q.um_idx = K.um_idx; Q.um_val = K.um_val;
    Q.T = T->c1_T; Q.col_idx = T->c1_col_idx; Q.row_idx = T->c1_row_idx; Q.coef = T->c1_coef; Q.coef_next = T->c1_coef_next;
    Q.x_perm = K.xperm; Q.y_perm = K.yperm;
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    chain1_kernel(L, NF)<<<(unsigned)blocks, 32 * wpb, smem, st>>>(Q);
    return launched(blocks, 32 * wpb, smem, per_warp * wpb);
}

// generic band kernel, in the placement band_geometry picks
static int launch_band(const dsp_template *T, KParams K, cudaStream_t st) {
    const size_t prob_bytes = (size_t)K.prob_doubles * 8;
    const BandGeom geom = band_geometry(T, K);
    long long warps = geom.warps;
    long long ctas = std::min<long long>(T->sm_count, (K.N + warps - 1) / warps);
    // spread a small batch over all SMs
    if (ctas < T->sm_count && K.N > ctas) {
        ctas = std::min<long long>(T->sm_count, K.N);
        warps = std::min<long long>(warps, (K.N + ctas - 1) / ctas);
    }
    K.hot_in_smem = geom.hot_in_smem;
    K.prob_off = (int)geom.off;
    K.ws = nullptr;
    K.hybrid = geom.hybrid;
    size_t smem = geom.off + (size_t)warps * prob_bytes;
    if (geom.ws) {
        const int rc = grow_ws(T, (size_t)ctas * (size_t)warps * prob_bytes, st);
        if (rc) return rc;
        K.ws = T->ws;
        smem = geom.hybrid ? geom.off + (size_t)warps * K.band_doubles * 8 : 16;
    }
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    band_kernel(K.w, geom.ws, geom.hot_in_smem)<<<(unsigned)ctas, (unsigned)(warps * 32), smem, st>>>(K);
    return launched(ctas, warps * 32, smem, warps);
}

// the dense kernel's data of a band template, built from its device copy of A at the first DSP_KERNEL_DENSE call
static int ensure_dense(const dsp_template *T) {
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    const KParams &K = T->kp;
    if (K.n_amap > 0) { g_err = "dsp_lp_solve_batch: DSP_KERNEL_DENSE does not take per-problem matrix coefficients"; return DSP_E_ARG; }
    if (T->dn.ready) return 0;
    if (K.m > kDenseMaxM) { g_err = "dsp_lp_solve_batch: DSP_KERNEL_DENSE needs m <= 1024 (m = " + std::to_string(K.m) + ")"; return DSP_E_ARG; }
    std::vector<unsigned char> hot(K.hot_bytes);
    CK(cudaMemcpy(hot.data(), K.hot_g, hot.size(), cudaMemcpyDeviceToHost));
    const double *val = (const double *)hot.data();
    const int *ptr = (const int *)(val + 2 * (size_t)K.nnz + K.nasm), *idx = ptr + K.m + 1;
    return dense_build(const_cast<dsp_template *>(T), std::vector<int>(ptr, ptr + K.m + 1), std::vector<int>(idx, idx + K.nnz),
                       std::vector<double>(val, val + K.nnz));
}

// dense kernel: one persistent CTA per LP in flight, as many CTAs per SM as fit; the lower tiles of M of every CTA in the handle's
// workspace, the per-LP vectors in shared memory when they fit next to the two staged-tile buffers (else behind the tiles)
static int launch_dense(const dsp_template *T, const KParams &K, cudaStream_t st) {
    const dsp_template::Dense &D = T->dn;
    DParams Q;
    memset(&Q, 0, sizeof(Q));
    Q.m = K.m; Q.n = K.n; Q.nb = K.nb; Q.Pc = K.Pc; Q.Pr = K.Pr; Q.nt = D.nt;
    Q.c0 = K.c0; Q.b0 = K.b0; Q.u0 = K.u0; Q.omap = K.omap; Q.ocmap = K.ocmap;
    Q.cm_ptr = K.cm_ptr; Q.cm_idx = K.cm_idx; Q.cm_val = K.cm_val; Q.bm_ptr = K.bm_ptr; Q.bm_idx = K.bm_idx; Q.bm_val = K.bm_val;
    Q.um_ptr = K.um_ptr; Q.um_idx = K.um_idx; Q.um_val = K.um_val; Q.o0 = K.o0;
    Q.A_ptr = D.A_ptr; Q.A_idx = D.A_idx; Q.A_val = D.A_val; Q.At_ptr = D.At_ptr; Q.At_idx = D.At_idx; Q.At_val = D.At_val;
    Q.nent = D.nent; Q.asm_pos = D.asm_pos; Q.asm_ptr = D.asm_ptr; Q.asm_col = D.asm_col; Q.asm_val = D.asm_val;
    Q.N = K.N; Q.cparams = K.cparams; Q.rparams = K.rparams; Q.rstride = K.rstride;
    Q.tol = K.tol; Q.feas_tol = K.feas_tol; Q.step_frac = K.step_frac; Q.reg = K.reg; Q.max_iter = K.max_iter;
    Q.obj = K.obj; Q.x_out = K.x_out; Q.y_out = K.y_out; Q.status = K.status; Q.iters = K.iters; Q.ticket = K.ticket;
    Q.xperm = K.xperm; Q.yperm = K.yperm;
    const long long vec = dense_vec_doubles(K.m, K.n, K.nb, D.nt);
    Q.vec_in_smem = kDenseSmemFixed + (size_t)vec * 8 <= (size_t)T->smem_optin;
    const size_t smem = kDenseSmemFixed + (Q.vec_in_smem ? (size_t)vec * 8 : 0);
    Q.cta_doubles = dense::tiles_doubles(D.nt) + (Q.vec_in_smem ? 0 : vec);
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dsp_ipm_dense_kernel, kDenseThreads, smem));
    long long ctas = std::min<long long>(K.N, (long long)T->sm_count * std::max(occ, 1));
    while (ctas > 1 && (size_t)ctas * Q.cta_doubles * 8 > T->ws_cap) ctas /= 2;
    const int rc = grow_ws(T, (size_t)ctas * Q.cta_doubles * 8, st);
    if (rc) return rc;
    Q.ws = T->ws;
    CK(cudaMemsetAsync(K.ticket, 0, sizeof(unsigned long long), st));
    dsp_ipm_dense_kernel<<<(unsigned)ctas, kDenseThreads, smem, st>>>(Q);
    return launched(ctas, kDenseThreads, smem, 1);
}

static int launch_batch(const dsp_template *T, int64_t N, const double *cparams, const double *rparams,
                        int64_t rparams_stride, const dsp_opts *opts, double *obj, int32_t *status, int32_t *iters,
                        double *x, double *y, void *cuda_stream, unsigned long long *ticket) {
    if (!T || N < 0 || !obj || !status || !iters || (T->kp.Pc > 0 && !cparams) || (T->kp.Pr > 0 && !rparams)) {
        g_err = "dsp_lp_solve_batch: bad arguments";
        return DSP_E_ARG;
    }
    if (N == 0) return 0;
    dsp_opts o;
    dsp_lp_default_opts(&o);
    if (opts) o = *opts;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    KParams K = T->kp;
    K.N = N; K.cparams = cparams; K.rparams = rparams; K.rstride = rparams_stride;
    K.tol = o.tol; K.feas_tol = o.feas_tol; K.step_frac = o.step_frac; K.reg = o.reg_primal; K.max_iter = o.max_iter;
    K.obj = obj; K.status = status; K.iters = iters; K.x_out = x; K.y_out = y;
    K.ticket = ticket;
    K.retry_only = 0;
    if (T->dense_only && o.kernel != DSP_KERNEL_AUTO && o.kernel != DSP_KERNEL_DENSE) {
        g_err = "dsp_lp_solve_batch: a template made by dsp_lp_template_create_dense runs only the dense kernel (DSP_KERNEL_AUTO or DSP_KERNEL_DENSE)";
        return DSP_E_ARG;
    }
    if (T->dense_only || o.kernel == DSP_KERNEL_DENSE) {
        const int rc = ensure_dense(T);
        if (rc) return rc;
        return launch_dense(T, K, st);
    }
    const bool stage = o.kernel == DSP_KERNEL_AUTO || o.kernel == DSP_KERNEL_STAGE;
    if (T->has_stage && T->sp.T > kStage2MaxT && stage) {
        const int rc = launch_stage2_long(T, K, st);
        if (rc) return rc;
        // At T = 8736 cond(M) reaches 1e15 and the partitioned elimination order rounds differently from the band kernel's
        // sequential one: about 1 LP in 60 of the reference's full-year sweep stalls in the long kernel and converges in the
        // band kernel.  The band kernel therefore follows on the same stream and re-solves ONLY the LPs the long kernel left
        // with MAX_ITER / NUMERICAL (its warps skip every other ticket: a few microseconds when there is none).
        K.retry_only = 1;
        return launch_band(T, K, st);
    }
    if (T->has_stage && stage) return launch_stage2(T, K, st);
    if (T->has_stage && o.kernel == DSP_KERNEL_STAGE_V1) return launch_stage_v1(T, K, st);
    if (T->has_chain1 && stage) return launch_chain1(T, K, st);
    if (o.kernel == DSP_KERNEL_STAGE || o.kernel == DSP_KERNEL_STAGE_V1) {
        g_err = "dsp_lp_solve_batch: the template has no stage descriptor";
        return DSP_E_ARG;
    }
    return launch_band(T, K, st);
}

int dsp_lp_solve_batch(const dsp_template *T, int64_t N, const double *cparams, const double *rparams,
                       int64_t rparams_stride, const dsp_opts *opts, double *obj, int32_t *status, int32_t *iters,
                       double *x, double *y, void *cuda_stream) {
    return launch_batch(T, N, cparams, rparams, rparams_stride, opts, obj, status, iters, x, y, cuda_stream,
                        T ? T->ticket : nullptr);
}

static void free_staging(dsp_template *T) {
    cudaFree(T->d_cp); cudaFree(T->d_rp); cudaFree(T->d_obj); cudaFree(T->d_x); cudaFree(T->d_y);
    cudaFree(T->d_status); cudaFree(T->d_iters);
    cudaFreeHost(T->h_cp); cudaFreeHost(T->h_rp); cudaFreeHost(T->h_obj); cudaFreeHost(T->h_x); cudaFreeHost(T->h_y);
    cudaFreeHost(T->h_status); cudaFreeHost(T->h_iters);
    T->d_cp = T->d_rp = T->d_obj = T->d_x = T->d_y = nullptr; T->d_status = T->d_iters = nullptr;
    T->h_cp = T->h_rp = T->h_obj = T->h_x = T->h_y = nullptr; T->h_status = T->h_iters = nullptr;
    T->cap_N = 0; T->cap_rp_rows = 0; T->cap_x = T->cap_y = false;
}

// Grows the device buffers (and, unless the caller's buffers are page-locked, the pinned staging buffers) of the host call.
// On any allocation failure everything is released and the capacities are reset to 0, so a later call starts clean.
static int ensure_capacity(dsp_template *T, int64_t N, int64_t rp_rows, bool want_x, bool want_y, bool stage_in, bool stage_out) {
    const KParams &K = T->kp;
    const bool need_hin = stage_in && !T->h_cp, need_hout = stage_out && (!T->h_obj || (want_x && !T->h_x) || (want_y && !T->h_y));
    if (N > T->cap_N || rp_rows > T->cap_rp_rows || (want_x && !T->cap_x) || (want_y && !T->cap_y) || need_hin || need_hout) {
        const int64_t cap = std::max<int64_t>(N, T->cap_N);
        const int64_t rcap = std::max<int64_t>(rp_rows, T->cap_rp_rows);
        const bool cx = want_x || T->cap_x, cy = want_y || T->cap_y;
        const bool hin = stage_in || T->h_cp, hout = stage_out || T->h_obj;
        free_staging(T);
        const size_t ncp = (size_t)std::max<int64_t>(1, cap * K.Pc), nrp = (size_t)std::max<int64_t>(1, rcap * K.Pr);
        cudaError_t e = cudaSuccess;
        auto dev = [&](void **p, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(p, bytes); };
        auto host = [&](void **p, size_t bytes) { if (e == cudaSuccess) e = cudaMallocHost(p, bytes); };
        dev((void **)&T->d_cp, ncp * 8); dev((void **)&T->d_rp, nrp * 8);
        dev((void **)&T->d_obj, cap * 8); dev((void **)&T->d_status, cap * 4); dev((void **)&T->d_iters, cap * 4);
        if (cx) dev((void **)&T->d_x, (size_t)cap * K.n * 8);
        if (cy) dev((void **)&T->d_y, (size_t)cap * K.m * 8);
        // the small shared-rparams row is always staged through h_rp
        host((void **)&T->h_rp, (hin ? nrp : (size_t)std::max(1, K.Pr)) * 8);
        if (hin) host((void **)&T->h_cp, ncp * 8);
        if (hout) {
            host((void **)&T->h_obj, cap * 8); host((void **)&T->h_status, cap * 4); host((void **)&T->h_iters, cap * 4);
            if (cx) host((void **)&T->h_x, (size_t)cap * K.n * 8);
            if (cy) host((void **)&T->h_y, (size_t)cap * K.m * 8);
        }
        if (e != cudaSuccess) {
            free_staging(T);
            cudaGetLastError();
            g_err = std::string("dsp_lp_solve_batch_host: buffer allocation failed: ") + cudaGetErrorString(e);
            return DSP_E_CUDA;
        }
        T->cap_N = cap; T->cap_rp_rows = rcap; T->cap_x = cx; T->cap_y = cy;
    }
    return 0;
}

static int solve_batch_host_locked(dsp_template *T, int64_t N, const double *cparams, const double *rparams,
                                   int64_t rparams_stride, const dsp_opts *opts, double *obj, int32_t *status,
                                   int32_t *iters, double *x, double *y);

int dsp_lp_solve_batch_host(dsp_template *T, int64_t N, const double *cparams, const double *rparams,
                            int64_t rparams_stride, const dsp_opts *opts, double *obj, int32_t *status,
                            int32_t *iters, double *x, double *y) {
    if (!T || N < 0) { g_err = "dsp_lp_solve_batch_host: bad arguments"; return DSP_E_ARG; }
    int expected = 0;
    if (!T->busy.compare_exchange_strong(expected, 1)) {       // not re-entrant per handle: enforced, not just documented
        g_err = "dsp_lp_solve_batch_host: another host call is in flight on this template handle (use one handle per host thread)";
        return DSP_E_BUSY;
    }
    const int rc = solve_batch_host_locked(T, N, cparams, rparams, rparams_stride, opts, obj, status, iters, x, y);
    T->busy.store(0);
    return rc;
}

static int solve_batch_host_locked(dsp_template *T, int64_t N, const double *cparams, const double *rparams,
                                   int64_t rparams_stride, const dsp_opts *opts, double *obj, int32_t *status,
                                   int32_t *iters, double *x, double *y) {
    if (!T || N < 0) { g_err = "dsp_lp_solve_batch_host: bad arguments"; return DSP_E_ARG; }
    if (N == 0) return 0;
    const KParams &K = T->kp;
    const int64_t rp_rows = (rparams_stride == 0) ? 1 : N;
    if (!obj || !status || !iters || (K.Pc > 0 && !cparams) || (K.Pr > 0 && !rparams)) {
        g_err = "dsp_lp_solve_batch_host: bad arguments";
        return DSP_E_ARG;
    }
    if (K.Pr > 0 && rparams_stride != 0 && rparams_stride < K.Pr) { g_err = "dsp_lp_solve_batch_host: rparams_stride < Pr"; return DSP_E_ARG; }
    // chunked pipeline over two streams: the pinned-staging memcpy + H2D of chunk k+1 and the D2H of chunk k-1 overlap
    // the kernel of chunk k.  Caller buffers that are already page-locked (cudaHostAlloc / cudaHostRegister / a pinned
    // torch tensor) are used directly, without the staging copy (and without allocating staging buffers at all).
    auto pinned = [](const void *p) {
        if (!p) return false;
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return at.type == cudaMemoryTypeHost;
    };
    const bool in_pinned = pinned(cparams) && (K.Pr == 0 || pinned(rparams)) && (rparams_stride == 0 || rparams_stride == K.Pr);
    const bool out_pinned = pinned(obj) && pinned(status) && pinned(iters) && (!x || pinned(x)) && (!y || pinned(y));
    int rc = ensure_capacity(T, N, rp_rows, x != nullptr, y != nullptr, !in_pinned, !out_pinned);
    if (rc) return rc;
    cudaStream_t sts[2] = {T->stream, T->stream2};
    int64_t dstride = 0;
    // templates that run in global-workspace mode share ONE workspace: no concurrent chunk kernels for them
    const bool dense = T->dense_only || (opts && opts->kernel == DSP_KERNEL_DENSE);            // the dense kernel always uses the workspace
    const bool ws_template = dense || band_geometry(T, K).ws || (T->has_stage && T->sp.T > kStage2MaxT);    // (the long stage kernel's workspace too)
    // Chunks pay when there is something to overlap: the staging memcpy of pageable input (always), or the H2D copy of a batch whose
    // kernel runs for many waves.  A page-locked batch of a few waves goes in ONE piece: the persistent stage kernels fill every SM
    // with one CTA, so two chunk kernels cannot share the chip and each chunk ends in its own thinning tail.
    const int nchunk = ws_template ? 1
                     : in_pinned   ? (int)std::min<int64_t>(4, std::max<int64_t>(1, N / 65536))
                                   : (int)std::min<int64_t>(8, std::max<int64_t>(1, N / 2048));
    const bool shared_rp = (K.Pr > 0 && rparams_stride == 0);
    if (shared_rp) {
        memcpy(T->h_rp, rparams, (size_t)K.Pr * 8);
        CK(cudaMemcpyAsync(T->d_rp, T->h_rp, (size_t)K.Pr * 8, cudaMemcpyHostToDevice, sts[0]));
        if (nchunk > 1) CK(cudaStreamSynchronize(sts[0]));          // 0.2 KB, makes the row visible to both streams (one chunk: stream order suffices)
    } else if (K.Pr > 0) {
        dstride = K.Pr;
    }
    const int64_t per = (N + nchunk - 1) / nchunk;
    for (int c = 0; c < nchunk; ++c) {
        const int64_t lo = c * per, cnt = std::min<int64_t>(per, N - lo);
        if (cnt <= 0) break;
        cudaStream_t st = sts[c & 1];
        if (K.Pc > 0) {
            const double *src = cparams + lo * K.Pc;
            if (!in_pinned) { memcpy(T->h_cp + lo * K.Pc, src, (size_t)cnt * K.Pc * 8); src = T->h_cp + lo * K.Pc; }
            CK(cudaMemcpyAsync(T->d_cp + lo * K.Pc, src, (size_t)cnt * K.Pc * 8, cudaMemcpyHostToDevice, st));
        }
        if (K.Pr > 0 && !shared_rp) {
            const double *src = rparams + lo * K.Pr;
            if (!in_pinned) {
                if (rparams_stride != K.Pr) {   // compact strided rows
                    for (int64_t r = 0; r < cnt; ++r) memcpy(T->h_rp + (lo + r) * K.Pr, rparams + (lo + r) * rparams_stride, (size_t)K.Pr * 8);
                } else {
                    memcpy(T->h_rp + lo * K.Pr, src, (size_t)cnt * K.Pr * 8);
                }
                src = T->h_rp + lo * K.Pr;
            }
            CK(cudaMemcpyAsync(T->d_rp + lo * K.Pr, src, (size_t)cnt * K.Pr * 8, cudaMemcpyHostToDevice, st));
        }
        rc = launch_batch(T, cnt, T->d_cp + lo * K.Pc, shared_rp ? T->d_rp : T->d_rp + lo * K.Pr, dstride, opts,
                          T->d_obj + lo, T->d_status + lo, T->d_iters + lo, x ? T->d_x + lo * K.n : nullptr,
                          y ? T->d_y + lo * K.m : nullptr, st, T->ticket + c);
        if (rc) return rc;
        double *o_obj = out_pinned ? obj : T->h_obj; int32_t *o_st = out_pinned ? status : T->h_status;
        int32_t *o_it = out_pinned ? iters : T->h_iters; double *o_x = out_pinned ? x : T->h_x; double *o_y = out_pinned ? y : T->h_y;
        CK(cudaMemcpyAsync(o_obj + lo, T->d_obj + lo, (size_t)cnt * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(o_st + lo, T->d_status + lo, (size_t)cnt * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(o_it + lo, T->d_iters + lo, (size_t)cnt * 4, cudaMemcpyDeviceToHost, st));
        if (x) CK(cudaMemcpyAsync(o_x + lo * K.n, T->d_x + lo * K.n, (size_t)cnt * K.n * 8, cudaMemcpyDeviceToHost, st));
        if (y) CK(cudaMemcpyAsync(o_y + lo * K.m, T->d_y + lo * K.m, (size_t)cnt * K.m * 8, cudaMemcpyDeviceToHost, st));
    }
    cudaStream_t st = sts[0];
    CK(cudaStreamSynchronize(sts[1]));
    CK(cudaStreamSynchronize(st));
    if (!out_pinned) {
        memcpy(obj, T->h_obj, (size_t)N * 8);
        memcpy(status, T->h_status, (size_t)N * 4);
        memcpy(iters, T->h_iters, (size_t)N * 4);
        if (x) memcpy(x, T->h_x, (size_t)N * K.n * 8);
        if (y) memcpy(y, T->h_y, (size_t)N * K.m * 8);
    }
    return 0;
}


// ---------------------------------------------------------------------------------------------------------------------
// Template from plain CSR: everything dsp_lp_template_create expects from its caller -- bounded columns first, a
// bandwidth-reducing row order for A A', the assembly list of the band of A D A' -- is derived here, so that a C caller
// (or the Pyomo walker) hands over nothing but the standard-form LP.  Host-only analysis: no CUDA call before the upload.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct CsrAnalysis {
    std::vector<int> col_perm, row_perm;      // internal -> caller
    int nb = 0, w = 0, w_natural = 0, w_rcm = 0;
    std::vector<int> A_ptr, A_idx;            // permuted CSR
    std::vector<double> A_val;
    std::vector<int> asm_ptr, asm_col;
    std::vector<double> asm_val;
    std::vector<int> asm_qa, asm_qb;          // CSR positions of the two factors of every assembly term
};

int bandwidth_of(const std::vector<std::vector<int>> &adj, const std::vector<int> &pos) {
    int w = 0;
    for (size_t i = 0; i < adj.size(); ++i)
        for (int j : adj[i]) w = std::max(w, std::abs(pos[i] - pos[j]));
    return w;
}

// reverse Cuthill-McKee on the row graph of A A' (start of every component: a pseudo-peripheral node of minimum degree)
std::vector<int> rcm_order(const std::vector<std::vector<int>> &adj) {
    const int m = (int)adj.size();
    std::vector<int> order; order.reserve(m);
    std::vector<char> seen(m, 0);
    std::vector<int> by_deg(m);
    for (int i = 0; i < m; ++i) by_deg[i] = i;
    std::stable_sort(by_deg.begin(), by_deg.end(), [&](int a, int b) { return adj[a].size() < adj[b].size(); });
    auto bfs = [&](int start, std::vector<int> &out, std::vector<char> &mark) {
        out.clear(); out.push_back(start); mark[start] = 1;
        for (size_t h = 0; h < out.size(); ++h) {
            std::vector<int> nb;
            for (int v : adj[out[h]]) if (!mark[v]) { mark[v] = 1; nb.push_back(v); }
            std::stable_sort(nb.begin(), nb.end(), [&](int a, int b) { return adj[a].size() < adj[b].size(); });
            out.insert(out.end(), nb.begin(), nb.end());
        }
    };
    for (int s0 : by_deg) {
        if (seen[s0]) continue;
        int start = s0;
        std::vector<int> comp;
        for (int pass = 0; pass < 3; ++pass) {         // walk towards a pseudo-peripheral node
            std::vector<char> mark(seen);
            bfs(start, comp, mark);
            int last = comp.back();
            if (last == start) break;
            start = last;
        }
        std::vector<int> comp2;
        bfs(start, comp2, seen);
        order.insert(order.end(), comp2.begin(), comp2.end());
    }
    std::reverse(order.begin(), order.end());
    return order;
}

int analyze_csr(const dsp_lp_desc *D, CsrAnalysis &R) {
    if (!D || D->m <= 0 || D->n <= 0 || !D->A_ptr || !D->A_idx || !D->A_val || !D->u0) { g_err = "dsp_lp_analyze: bad descriptor"; return DSP_E_ARG; }
    const int m = D->m, n = D->n;
    const int nnz = D->A_ptr[m];
    for (int q = 0; q < nnz; ++q)
        if (D->A_idx[q] < 0 || D->A_idx[q] >= n) { g_err = "dsp_lp_analyze: A_idx out of range"; return DSP_E_ARG; }
    // 1. bounded columns first (stable)
    R.col_perm.clear();
    for (int j = 0; j < n; ++j) if (D->u0[j] < 1e300) R.col_perm.push_back(j);
    R.nb = (int)R.col_perm.size();
    for (int j = 0; j < n; ++j) if (!(D->u0[j] < 1e300)) R.col_perm.push_back(j);
    std::vector<int> col_pos(n);
    for (int k = 0; k < n; ++k) col_pos[R.col_perm[k]] = k;
    // 2. row graph of A A'
    std::vector<std::vector<int>> rows_of_col(n);
    for (int i = 0; i < m; ++i)
        for (int q = D->A_ptr[i]; q < D->A_ptr[i + 1]; ++q) rows_of_col[D->A_idx[q]].push_back(i);
    std::vector<std::vector<int>> adj(m);
    for (int j = 0; j < n; ++j)
        for (int a : rows_of_col[j])
            for (int b : rows_of_col[j])
                if (a != b) adj[a].push_back(b);
    for (auto &v : adj) { std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end()); }
    std::vector<int> nat(m), pos(m);
    for (int i = 0; i < m; ++i) nat[i] = pos[i] = i;
    R.w_natural = bandwidth_of(adj, pos);
    std::vector<int> rcm = rcm_order(adj);
    for (int k = 0; k < m; ++k) pos[rcm[k]] = k;
    R.w_rcm = bandwidth_of(adj, pos);
    R.row_perm = (R.w_natural <= R.w_rcm) ? nat : rcm;
    R.w = std::min(R.w_natural, R.w_rcm);
    std::vector<int> row_pos(m);
    for (int k = 0; k < m; ++k) row_pos[R.row_perm[k]] = k;
    // 3. permuted CSR with sorted column indices
    R.A_ptr.assign(m + 1, 0); R.A_idx.resize(nnz); R.A_val.resize(nnz);
    for (int k = 0; k < m; ++k) R.A_ptr[k + 1] = R.A_ptr[k] + (D->A_ptr[R.row_perm[k] + 1] - D->A_ptr[R.row_perm[k]]);
    for (int k = 0; k < m; ++k) {
        const int i = R.row_perm[k];
        std::vector<std::pair<int, double>> ent;
        for (int q = D->A_ptr[i]; q < D->A_ptr[i + 1]; ++q) ent.emplace_back(col_pos[D->A_idx[q]], D->A_val[q]);
        std::sort(ent.begin(), ent.end());
        for (size_t e = 0; e < ent.size(); ++e) { R.A_idx[R.A_ptr[k] + e] = ent[e].first; R.A_val[R.A_ptr[k] + e] = ent[e].second; }
    }
    // 4. assembly list of the lower band of M = A D A':  M[i][i-k] = sum coef * d[col]   (coef = A[i][col] * A[i-k][col])
    const int w = R.w;
    struct Term { int col, qa, qb; double v; };
    std::vector<std::vector<Term>> ent((size_t)m * (w + 1));
    struct RowEnt { int row, q; double v; };
    std::vector<std::vector<RowEnt>> col_rows(n);       // (new row, CSR position, value) per new column
    for (int k = 0; k < m; ++k)
        for (int q = R.A_ptr[k]; q < R.A_ptr[k + 1]; ++q) col_rows[R.A_idx[q]].push_back({k, q, R.A_val[q]});
    for (int j = 0; j < n; ++j)
        for (auto &ra : col_rows[j])
            for (auto &rb : col_rows[j])
                if (rb.row <= ra.row) ent[(size_t)ra.row * (w + 1) + (ra.row - rb.row)].push_back({j, ra.q, rb.q, ra.v * rb.v});
    R.asm_ptr.assign((size_t)m * (w + 1) + 1, 0);
    R.asm_col.clear(); R.asm_val.clear(); R.asm_qa.clear(); R.asm_qb.clear();
    for (size_t e = 0; e < ent.size(); ++e) {
        R.asm_ptr[e + 1] = R.asm_ptr[e] + (int)ent[e].size();
        for (auto &t : ent[e]) { R.asm_col.push_back(t.col); R.asm_val.push_back(t.v); R.asm_qa.push_back(t.qa); R.asm_qb.push_back(t.qb); }
    }
    return 0;
}

// rows of a dsp_param_map re-ordered: out row k = in row perm[k]
void permute_map(const dsp_param_map &in, const std::vector<int> &perm, int nrows_out, std::vector<int> &ptr, std::vector<int> &idx, std::vector<double> &val) {
    ptr.assign(nrows_out + 1, 0); idx.clear(); val.clear();
    for (int k = 0; k < nrows_out; ++k) {
        const int r = perm[k];
        if (in.ptr) for (int q = in.ptr[r]; q < in.ptr[r + 1]; ++q) { idx.push_back(in.idx[q]); val.push_back(in.val[q]); }
        ptr[k + 1] = (int)idx.size();
    }
}
}  // namespace

int dsp_lp_analyze_csr(const dsp_lp_desc *D, int32_t *nb, int32_t *w, int32_t *w_natural, int32_t *w_rcm, int32_t *col_perm, int32_t *row_perm) {
    CsrAnalysis R;
    int rc = analyze_csr(D, R);
    if (rc) return rc;
    if (nb) *nb = R.nb;
    if (w) *w = R.w;
    if (w_natural) *w_natural = R.w_natural;
    if (w_rcm) *w_rcm = R.w_rcm;
    if (col_perm) std::copy(R.col_perm.begin(), R.col_perm.end(), col_perm);
    if (row_perm) std::copy(R.row_perm.begin(), R.row_perm.end(), row_perm);
    return 0;
}

int dsp_lp_template_create_csr(const dsp_lp_desc *D, dsp_template **out) {
    if (!out) { g_err = "dsp_lp_template_create_csr: out is NULL"; return DSP_E_ARG; }
    CsrAnalysis R;
    int rc = analyze_csr(D, R);
    if (rc) return rc;
    const int m = D->m, n = D->n, nb = R.nb;
    std::vector<double> c0(n), u0(std::max(nb, 1)), b0(m);
    for (int k = 0; k < n; ++k) c0[k] = D->c0 ? D->c0[R.col_perm[k]] : 0.0;
    for (int k = 0; k < nb; ++k) u0[k] = D->u0[R.col_perm[k]];
    for (int k = 0; k < m; ++k) b0[k] = D->b0 ? D->b0[R.row_perm[k]] : 0.0;
    std::vector<int> cp, ci, bp, bi, up, ui;
    std::vector<double> cv, bv, uv;
    permute_map(D->cmap, R.col_perm, n, cp, ci, cv);
    permute_map(D->bmap, R.row_perm, m, bp, bi, bv);
    permute_map(D->umap, R.col_perm, nb, up, ui, uv);
    std::vector<double> zPr(std::max(D->Pr, 1), 0.0), zPc(std::max(D->Pc, 1), 0.0);
    auto nz = [](std::vector<int> &v) { if (v.empty()) v.push_back(0); return v.data(); };
    auto nzd = [](std::vector<double> &v) { if (v.empty()) v.push_back(0.0); return v.data(); };
    dsp_template_desc d;
    memset(&d, 0, sizeof(d));
    d.m = m; d.n = n; d.nb = nb; d.w = R.w; d.Pc = D->Pc; d.Pr = D->Pr;
    d.A_ptr = R.A_ptr.data(); d.A_idx = R.A_idx.data(); d.A_val = R.A_val.data();
    d.asm_ptr = R.asm_ptr.data(); d.asm_col = nz(R.asm_col); d.asm_val = nzd(R.asm_val);
    d.c0 = c0.data(); d.cmap.ptr = cp.data(); d.cmap.idx = nz(ci); d.cmap.val = nzd(cv);
    d.b0 = b0.data(); d.bmap.ptr = bp.data(); d.bmap.idx = nz(bi); d.bmap.val = nzd(bv);
    d.u0 = u0.data(); d.umap.ptr = up.data(); d.umap.idx = nz(ui); d.umap.val = nzd(uv);
    d.o0 = D->o0; d.omap = D->omap ? D->omap : zPr.data(); d.ocmap = D->ocmap ? D->ocmap : zPc.data();
    dsp_template *T = nullptr;
    rc = dsp_lp_template_create(&d, &T);
    if (rc) return rc;
    T->col_perm = R.col_perm; T->row_perm = R.row_perm;
    T->csr_ptr = R.A_ptr; T->csr_idx = R.A_idx; T->asm_qa = R.asm_qa; T->asm_qb = R.asm_qb;
    int *dx = nullptr, *dy = nullptr;
    rc = upload(R.col_perm, &dx);
    if (!rc) { T->dev_allocs.push_back(dx); rc = upload(R.row_perm, &dy); }
    if (rc) { dsp_lp_template_destroy(T); return rc; }
    T->dev_allocs.push_back(dy);
    T->kp.xperm = dx; T->kp.yperm = dy;
    *out = T;
    return 0;
}

int dsp_lp_template_create_dense(const dsp_lp_desc *D, dsp_template **out) {
    if (!out) { g_err = "dsp_lp_template_create_dense: out is NULL"; return DSP_E_ARG; }
    if (!D || D->m <= 0 || D->n <= 0 || !D->A_ptr || !D->A_idx || !D->A_val || !D->u0) { g_err = "dsp_lp_template_create_dense: bad descriptor"; return DSP_E_ARG; }
    if (D->m > kDenseMaxM) {
        g_err = "dsp_lp_template_create_dense: m = " + std::to_string(D->m) + " rows; the dense kernel takes m <= 1024";
        return DSP_E_ARG;
    }
    const int m = D->m, n = D->n, nnz = D->A_ptr[m];
    for (int q = 0; q < nnz; ++q)
        if (D->A_idx[q] < 0 || D->A_idx[q] >= n) { g_err = "dsp_lp_template_create_dense: A_idx out of range"; return DSP_E_ARG; }
    // internal order: bounded columns first (stable), rows as given (the dense factorisation does not care about bandwidth)
    std::vector<int> col_perm, row_perm(m);
    for (int j = 0; j < n; ++j) if (D->u0[j] < 1e300) col_perm.push_back(j);
    const int nb = (int)col_perm.size();
    for (int j = 0; j < n; ++j) if (!(D->u0[j] < 1e300)) col_perm.push_back(j);
    std::vector<int> col_pos(n);
    for (int k = 0; k < n; ++k) col_pos[col_perm[k]] = k;
    for (int i = 0; i < m; ++i) row_perm[i] = i;
    std::vector<int> A_ptr(m + 1, 0), A_idx(nnz);
    std::vector<double> A_val(nnz);
    std::vector<int> rmin(n, m), rmax(n, -1);
    for (int i = 0; i < m; ++i) {
        std::vector<std::pair<int, double>> ent;
        for (int q = D->A_ptr[i]; q < D->A_ptr[i + 1]; ++q) {
            const int j = col_pos[D->A_idx[q]];
            ent.emplace_back(j, D->A_val[q]);
            rmin[j] = std::min(rmin[j], i); rmax[j] = std::max(rmax[j], i);
        }
        std::sort(ent.begin(), ent.end());
        A_ptr[i + 1] = A_ptr[i] + (int)ent.size();
        for (size_t e = 0; e < ent.size(); ++e) { A_idx[A_ptr[i] + e] = ent[e].first; A_val[A_ptr[i] + e] = ent[e].second; }
    }
    int w = 0;                         // half bandwidth of A A' in this row order: rows sharing a column are adjacent
    for (int j = 0; j < n; ++j) if (rmax[j] >= 0) w = std::max(w, rmax[j] - rmin[j]);
    std::vector<double> c0(n), u0(std::max(nb, 1)), b0(m);
    for (int k = 0; k < n; ++k) c0[k] = D->c0 ? D->c0[col_perm[k]] : 0.0;
    for (int k = 0; k < nb; ++k) u0[k] = D->u0[col_perm[k]];
    for (int i = 0; i < m; ++i) b0[i] = D->b0 ? D->b0[i] : 0.0;
    std::vector<int> cp, ci, bp, bi, up, ui;
    std::vector<double> cv, bv, uv;
    permute_map(D->cmap, col_perm, n, cp, ci, cv);
    permute_map(D->bmap, row_perm, m, bp, bi, bv);
    permute_map(D->umap, col_perm, nb, up, ui, uv);
    std::vector<double> zPr(std::max(D->Pr, 1), 0.0), zPc(std::max(D->Pc, 1), 0.0);
    auto nz = [](std::vector<int> &v) { if (v.empty()) v.push_back(0); return v.data(); };
    auto nzd = [](std::vector<double> &v) { if (v.empty()) v.push_back(0.0); return v.data(); };
    dsp_template_desc d;
    memset(&d, 0, sizeof(d));
    d.m = m; d.n = n; d.nb = nb; d.w = w; d.Pc = D->Pc; d.Pr = D->Pr;
    d.c0 = c0.data(); d.cmap.ptr = cp.data(); d.cmap.idx = nz(ci); d.cmap.val = nzd(cv);
    d.b0 = b0.data(); d.bmap.ptr = bp.data(); d.bmap.idx = nz(bi); d.bmap.val = nzd(bv);
    d.u0 = u0.data(); d.umap.ptr = up.data(); d.umap.idx = nz(ui); d.umap.val = nzd(uv);
    d.o0 = D->o0; d.omap = D->omap ? D->omap : zPr.data(); d.ocmap = D->ocmap ? D->ocmap : zPc.data();
    if (int rc = check_maps(&d)) return rc;
    dsp_template *T = new dsp_template();
    struct Guard {
        dsp_template *t;
        ~Guard() { if (t) dsp_lp_template_destroy(t); }
    } guard{T};
    if (int rc = template_init(T, &d)) return rc;
    T->kp.w = w; T->kp.nnz = nnz;
    T->dense_only = true;
    if (int rc = dense_build(T, A_ptr, A_idx, A_val)) return rc;
    T->col_perm = col_perm; T->row_perm = row_perm;
    int *dx = nullptr;
    if (int rc = upload(col_perm, &dx)) return rc;
    T->dev_allocs.push_back(dx);
    T->kp.xperm = dx;                  // rows keep the caller's order: no y permutation
    guard.t = nullptr;
    *out = T;
    return 0;
}

int dsp_lp_template_set_matrix_params(dsp_template *T, int32_t count, const int32_t *row, const int32_t *col, const int32_t *param,
                                      const double *coef) {
    if (!T || count < 0 || (count > 0 && (!row || !col || !param || !coef))) { g_err = "dsp_lp_template_set_matrix_params: bad arguments"; return DSP_E_ARG; }
    if (T->dense_only) { g_err = "dsp_lp_template_set_matrix_params: per-problem matrix coefficients are not supported on a dense template"; return DSP_E_ARG; }
    if (T->csr_ptr.empty()) { g_err = "dsp_lp_template_set_matrix_params: the template must come from dsp_lp_template_create_csr"; return DSP_E_ARG; }
    if (T->kp.w != 1 && T->kp.w != 2 && T->kp.w != 4 && T->kp.w != 8 && T->kp.w != 16 && T->kp.w != 32) { g_err = "bad band"; return DSP_E_ARG; }
    KParams &K = T->kp;
    const int m = K.m, n = K.n, nnz = K.nnz;
    std::vector<int> cpos(n), rpos(m);
    for (int k = 0; k < n; ++k) cpos[T->col_perm[k]] = k;
    for (int k = 0; k < m; ++k) rpos[T->row_perm[k]] = k;
    std::vector<int> q(count), pr(count);
    std::vector<double> cf(count);
    for (int k = 0; k < count; ++k) {
        if (row[k] < 0 || row[k] >= m || col[k] < 0 || col[k] >= n || param[k] < 0 || param[k] >= K.Pr) { g_err = "matrix parameter index out of range"; return DSP_E_ARG; }
        const int i = rpos[row[k]], j = cpos[col[k]];
        int pos = -1;
        for (int t = T->csr_ptr[i]; t < T->csr_ptr[i + 1]; ++t) if (T->csr_idx[t] == j) pos = t;
        if (pos < 0) { g_err = "matrix parameter on an entry that is not in the sparsity pattern of A (store an explicit nominal value)"; return DSP_E_ARG; }
        q[k] = pos; pr[k] = param[k]; cf[k] = coef[k];
    }
    // CSC position -> CSR position: the same stable counting sort dsp_lp_template_create used for the values
    std::vector<int> At_ptr(n + 1, 0), at_from(nnz);
    for (int t = 0; t < nnz; ++t) At_ptr[T->csr_idx[t] + 1]++;
    for (int j = 0; j < n; ++j) At_ptr[j + 1] += At_ptr[j];
    {
        std::vector<int> fill(At_ptr.begin(), At_ptr.end() - 1);
        for (int i = 0; i < m; ++i)
            for (int t = T->csr_ptr[i]; t < T->csr_ptr[i + 1]; ++t) at_from[fill[T->csr_idx[t]]++] = t;
    }
    int *dq, *dp, *daf, *dqa, *dqb; double *dc;
    int rc = upload(q, &dq); if (rc) return rc; T->dev_allocs.push_back(dq);
    rc = upload(pr, &dp); if (rc) return rc; T->dev_allocs.push_back(dp);
    rc = upload(cf, &dc); if (rc) return rc; T->dev_allocs.push_back(dc);
    rc = upload(at_from, &daf); if (rc) return rc; T->dev_allocs.push_back(daf);
    rc = upload(T->asm_qa, &dqa); if (rc) return rc; T->dev_allocs.push_back(dqa);
    rc = upload(T->asm_qb, &dqb); if (rc) return rc; T->dev_allocs.push_back(dqb);
    if (K.n_amap == 0) { K.prob_doubles += 2 * nnz + K.nasm; K.band_doubles += 2 * nnz + K.nasm; }   // this LP's matrix values sit behind its band (in every placement)
    K.n_amap = count; K.amap_q = dq; K.amap_param = dp; K.amap_coef = dc; K.at_from = daf; K.asm_qa = dqa; K.asm_qb = dqb;
    if (count == 0) K.n_amap = 0;
    return 0;
}

int dsp_lp_template_info(const dsp_template *T, int32_t *m, int32_t *n, int32_t *nb, int32_t *w) {
    if (!T) { g_err = "dsp_lp_template_info: null handle"; return DSP_E_ARG; }
    if (m) *m = T->kp.m;
    if (n) *n = T->kp.n;
    if (nb) *nb = T->kp.nb;
    if (w) *w = T->kp.w;
    return 0;
}

}  // extern "C"
