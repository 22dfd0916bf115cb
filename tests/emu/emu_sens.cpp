// emu_sens.cpp -- TEST INFRASTRUCTURE: the sensitivity post-pass of dispatches_b200/csrc/dsp_sens.cuh (its host structure builder and
// its warp body) compiled with g++ on the lock-step SIMT emulator (simt_emu.h) for tests/test_sensitivities_cpu.py.  Never linked into
// the product.
#include "simt_emu.h"

#include "../../dispatches_b200/csrc/dsp_sens.cuh"

template <class V>
static std::vector<V> vec(const V *p, long long n) { return p ? std::vector<V>(p, p + n) : std::vector<V>(); }

// the template in internal order (col_perm / row_perm: caller index of every internal column / row, NULL: identity), then the batch;
// every LP of the batch runs on one emulated warp
extern "C" int emu_sens(int m, int n, int nb, int Pc, int Pr, const int *A_ptr, const int *A_idx, const double *A_val, const int *col_perm,
                        const int *row_perm, const double *c0, const int *cm_ptr, const int *cm_idx, const double *cm_val, const int *bm_ptr,
                        const int *bm_idx, const double *bm_val, const int *um_ptr, const int *um_idx, const double *um_val,
                        const double *omap, const double *ocmap, int nterms, const int *t_q, const int *t_param, const double *t_coef,
                        long long N, const double *cparams, const double *rparams, long long rstride, const int *status, const double *x,
                        const double *y, double *rc, double *dcp, double *drp) {
    const std::vector<int> Ap = vec(A_ptr, m + 1), Ai = vec(A_idx, A_ptr[m]), cpm = vec(col_perm, col_perm ? n : 0),
                           rpm = vec(row_perm, row_perm ? m : 0), cmp = vec(cm_ptr, n + 1), cmi = vec(cm_idx, cm_ptr[n]),
                           bmp = vec(bm_ptr, m + 1), bmi = vec(bm_idx, bm_ptr[m]), ump = vec(um_ptr, nb + 1), umi = vec(um_idx, um_ptr[nb]),
                           tq = vec(t_q, nterms), tp = vec(t_param, nterms);
    const std::vector<double> Av = vec(A_val, A_ptr[m]), c0v = vec(c0, n), cmv = vec(cm_val, cm_ptr[n]), bmv = vec(bm_val, bm_ptr[m]),
                              umv = vec(um_val, um_ptr[nb]), om = vec(omap, Pr), ocm = vec(ocmap, Pc), tc = vec(t_coef, nterms);
    const sens::HostTemplate T{m, n, nb, Pc, Pr, Ap, Ai, Av, cpm, rpm, c0v, cmp, cmi, cmv, bmp, bmi, bmv, ump, umi, umv, om, ocm, tq, tp, tc};
    std::vector<unsigned char> blob;
    sens::Params P;
    P.L = sens::build_blob(T, blob);
    P.m = m; P.n = n; P.Pc = Pc; P.Pr = Pr; P.N = N; P.cparams = cparams; P.rparams = rparams; P.rstride = rstride;
    P.status = status; P.x = x; P.y = y; P.rc = rc; P.dcp = dcp; P.drp = drp;
    P.blob = blob.data(); P.blob_in_smem = 0;
    const sens::View v = sens::view_of(blob.data(), P.L);
    for (long long p = 0; p < N; ++p) emu::run_warp([&](int lane) { sens::lp_body<true>(P, v, p, lane); });
    return 0;
}
