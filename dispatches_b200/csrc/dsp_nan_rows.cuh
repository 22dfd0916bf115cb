// dsp_nan_rows.cuh -- the x / y rows of an INFEASIBLE LP are NaN (include/dsp_lp.h), so that a reused output buffer never shows
// another LP's numbers.  Written by lanes lane, lane + step, ... of the LP's warp or lane group.  Out of line: this is the rare
// per-LP path, and inlined into a kernel its loops would compete for the registers of the IPM round.
#ifndef DSP_NAN_ROWS_CUH
#define DSP_NAN_ROWS_CUH
#ifdef __CUDACC__
#define DSP_COLD __noinline__
#else
#define DSP_COLD
#endif
static __device__ DSP_COLD void dsp_nan_rows(double *x, int n, double *y, int m, long long p, int lane, int step) {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    if (x) for (int k = lane; k < n; k += step) x[p * n + k] = nan;
    if (y) for (int k = lane; k < m; k += step) y[p * m + k] = nan;
}
#endif
