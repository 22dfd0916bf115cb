// emu_parametric.cpp -- TEST INFRASTRUCTURE: the parametric walk of dispatches_b200/csrc/dsp_parametric.cuh (with the crossover's host
// structure builders) compiled with g++ on the lock-step SIMT emulator (simt_emu.h), one emulated warp standing for the CTA, for
// tests/test_parametric_cpu.py.  Never linked into the product.
#include "simt_emu.h"

#define XO_SYNC() __syncwarp()
#include "../../dispatches_b200/csrc/dsp_parametric.cuh"

template <class V>
static std::vector<V> vec(const V *p, long long n) { return p ? std::vector<V>(p, p + n) : std::vector<V>(); }

// the template in internal order (col_perm / row_perm: caller index of every internal column / row, NULL: identity), then the batch and
// its bases; every (LP, direction) pair of the batch runs on one emulated warp of 32 threads
extern "C" int emu_parametric(int m, int n, int nb, int Pc, int Pr, const int *A_ptr, const int *A_idx, const double *A_val,
                              const int *col_perm, const int *row_perm, const double *c0, const int *cm_ptr, const int *cm_idx,
                              const double *cm_val, const double *b0, const int *bm_ptr, const int *bm_idx, const double *bm_val,
                              const double *u0, const int *um_ptr, const int *um_idx, const double *um_val, const double *omap,
                              const double *ocmap, double o0, int nterms, const int *t_q, const int *t_param, const double *t_coef,
                              long long N, const double *cparams, const double *rparams, long long rstride, const int *status,
                              const signed char *col_status, const signed char *row_basic, int K, const double *dir_c,
                              const double *dir_r, int dir_per_lp, const double *theta_end, int S_, double *theta, double *obj,
                              double *dobj, double *d2obj, int *enter, int *leave, signed char *leave_to, int *count,
                              int *pstatus) {
    const std::vector<int> Ap = vec(A_ptr, m + 1), Ai = vec(A_idx, A_ptr[m]), cpm = vec(col_perm, col_perm ? n : 0),
                           rpm = vec(row_perm, row_perm ? m : 0), cmp = vec(cm_ptr, n + 1), cmi = vec(cm_idx, cm_ptr[n]),
                           bmp = vec(bm_ptr, m + 1), bmi = vec(bm_idx, bm_ptr[m]), ump = vec(um_ptr, nb + 1), umi = vec(um_idx, um_ptr[nb]),
                           tq = vec(t_q, nterms), tp = vec(t_param, nterms);
    const std::vector<double> Av = vec(A_val, A_ptr[m]), c0v = vec(c0, n), cmv = vec(cm_val, cm_ptr[n]), bmv = vec(bm_val, bm_ptr[m]),
                              umv = vec(um_val, um_ptr[nb]), om = vec(omap, Pr), ocm = vec(ocmap, Pc), tc = vec(t_coef, nterms),
                              b0v = vec(b0, m), u0v = vec(u0, nb);
    const sens::HostTemplate T{m, n, nb, Pc, Pr, Ap, Ai, Av, cpm, rpm, c0v, cmp, cmi, cmv, bmp, bmi, bmv, ump, umi, umv, om, ocm, tq, tp, tc};
    std::vector<unsigned char> blob, xblob;
    pm::Params P;
    P.L = sens::build_blob(T, blob);
    P.X = xo::build_blob(T, b0v, u0v, xblob);
    P.m = m; P.n = n; P.Pc = Pc; P.Pr = Pr; P.nnz = A_ptr[m]; P.K = K; P.S = S_; P.N = N;
    P.cparams = cparams; P.rparams = rparams; P.rstride = rstride; P.status = status; P.col_status = col_status; P.row_basic = row_basic;
    P.dir_c = Pc > 0 ? dir_c : nullptr; P.dir_r = Pr > 0 ? dir_r : nullptr; P.dir_per_lp = dir_per_lp; P.theta_end = theta_end; P.o0 = o0;
    P.theta = theta; P.obj = obj; P.dobj = dobj; P.d2obj = d2obj; P.enter = enter; P.leave = leave; P.leave_to = leave_to;
    P.count = count; P.pstatus = pstatus;
    P.blob = blob.data(); P.xblob = xblob.data(); P.ws = nullptr; P.ws_stride = 0;
    const sens::View v = sens::view_of(blob.data(), P.L);
    const xo::View X = xo::view_of(xblob.data(), P.X);
    std::vector<double> work((size_t)pm::work_doubles(m, n, P.nnz, Pc, Pr));
    xo::Shared S;
    for (long long pk = 0; pk < N * K; ++pk) emu::run_warp([&](int lane) { pm::pair_body(P, v, X, work.data(), &S, pk, lane, 32); });
    return 0;
}
