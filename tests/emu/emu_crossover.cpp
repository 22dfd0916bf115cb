// emu_crossover.cpp -- TEST INFRASTRUCTURE: the crossover post-pass of dispatches_b200/csrc/dsp_crossover.cuh (its host structure
// builders and its CTA body) compiled with g++ on the lock-step SIMT emulator (simt_emu.h), one emulated warp standing for the CTA, for
// tests/test_crossover_cpu.py and tests/test_crossover_paths*.py.  Never linked into the product.
#include "simt_emu.h"

// the path counters of the LP being run (xo::TR_EVENTS per LP), counted by lane 0; null: not counted
static int *g_trace = nullptr;

#define XO_SYNC() __syncwarp()
#define XO_TRACE(ev) ((tid == 0 && g_trace) ? (void)++g_trace[ev] : (void)0)
#include "../../dispatches_b200/csrc/dsp_crossover.cuh"

template <class V>
static std::vector<V> vec(const V *p, long long n) { return p ? std::vector<V>(p, p + n) : std::vector<V>(); }

extern "C" int emu_crossover_trace_events() { return xo::TR_EVENTS; }

// the template in internal order (col_perm / row_perm: caller index of every internal column / row, NULL: identity), then the batch;
// every LP of the batch runs on one emulated warp of 32 threads.  trace [N, emu_crossover_trace_events()] (or NULL): how often LP p
// took each path of xo::lp_body
extern "C" int emu_crossover(int m, int n, int nb, int Pc, int Pr, const int *A_ptr, const int *A_idx, const double *A_val,
                             const int *col_perm, const int *row_perm, const double *c0, const int *cm_ptr, const int *cm_idx,
                             const double *cm_val, const double *b0, const int *bm_ptr, const int *bm_idx, const double *bm_val,
                             const double *u0, const int *um_ptr, const int *um_idx, const double *um_val, const double *omap,
                             const double *ocmap, double o0, int nterms, const int *t_q, const int *t_param, const double *t_coef,
                             long long N, const double *cparams, const double *rparams, long long rstride, const int *status,
                             const double *x, const double *y, int max_pivots, double *obj, double *x_out, double *y_out,
                             signed char *col_status, signed char *row_basic, int *xstatus, int *pivots, int *trace) {
    const std::vector<int> Ap = vec(A_ptr, m + 1), Ai = vec(A_idx, A_ptr[m]), cpm = vec(col_perm, col_perm ? n : 0),
                           rpm = vec(row_perm, row_perm ? m : 0), cmp = vec(cm_ptr, n + 1), cmi = vec(cm_idx, cm_ptr[n]),
                           bmp = vec(bm_ptr, m + 1), bmi = vec(bm_idx, bm_ptr[m]), ump = vec(um_ptr, nb + 1), umi = vec(um_idx, um_ptr[nb]),
                           tq = vec(t_q, nterms), tp = vec(t_param, nterms);
    const std::vector<double> Av = vec(A_val, A_ptr[m]), c0v = vec(c0, n), cmv = vec(cm_val, cm_ptr[n]), bmv = vec(bm_val, bm_ptr[m]),
                              umv = vec(um_val, um_ptr[nb]), om = vec(omap, Pr), ocm = vec(ocmap, Pc), tc = vec(t_coef, nterms),
                              b0v = vec(b0, m), u0v = vec(u0, nb);
    const sens::HostTemplate T{m, n, nb, Pc, Pr, Ap, Ai, Av, cpm, rpm, c0v, cmp, cmi, cmv, bmp, bmi, bmv, ump, umi, umv, om, ocm, tq, tp, tc};
    std::vector<unsigned char> blob, xblob;
    xo::Params P;
    P.L = sens::build_blob(T, blob);
    P.X = xo::build_blob(T, b0v, u0v, xblob);
    P.m = m; P.n = n; P.Pc = Pc; P.Pr = Pr; P.nnz = A_ptr[m]; P.N = N; P.cparams = cparams; P.rparams = rparams; P.rstride = rstride;
    P.status = status; P.x = x; P.y = y; P.max_pivots = max_pivots > 0 ? max_pivots : 10 * (m + n); P.o0 = o0;
    P.obj = obj; P.x_out = x_out; P.y_out = y_out; P.col_status = col_status; P.row_basic = row_basic; P.xstatus = xstatus;
    P.pivots = pivots; P.blob = blob.data(); P.xblob = xblob.data(); P.ws = nullptr; P.ws_stride = 0;
    const sens::View v = sens::view_of(blob.data(), P.L);
    const xo::View X = xo::view_of(xblob.data(), P.X);
    std::vector<double> work((size_t)xo::work_doubles(m, n, P.nnz));
    xo::Shared S;
    for (long long p = 0; p < N; ++p) {
        if (trace) { g_trace = trace + p * xo::TR_EVENTS; std::fill(g_trace, g_trace + xo::TR_EVENTS, 0); }
        emu::run_warp([&](int lane) { xo::lp_body(P, v, X, work.data(), &S, p, lane, 32); });
        g_trace = nullptr;
    }
    return 0;
}
