/*
 * dsp_lp.h -- C ABI of the H100 batched dispatch-LP solver (libdsp_lp.so).
 *
 * The reference (gmlc-dispatches/dispatches) is pure Python and has no FFI; the boundary this library
 * sits behind is Pyomo's solver-plugin call
 *
 *     opt = pyo.SolverFactory("cbc");  opt.solve(m)        wind_battery_LMP.py:266-267
 *     opt = pyo.SolverFactory('cbc');  opt.solve(m)        wind_battery_PEM_LMP.py:296-298
 *     solver = SolverFactory("gurobi"); solver.solve(m)    nuclear_case/report/price_taker_analysis.py:365,403
 *     SolverFactory('ipopt').solve(m, tee=True)            fossil_case/.../pricetaker_with_multiperiod_integrated_storage_usc.py:126,137
 *
 * invoked once per (design point, LMP signal) by the sweep loops
 * (run_pricetaker_wind_battery.py:37-70, run_pricetaker_wind_PEM.py:100-110, price_taker_analysis.py:372-403).
 * Those calls write an LP file, fork a solver process and parse a .sol file per LP.  Here the shared
 * constraint structure is handed over ONCE (dsp_lp_template_create) and the whole scenario batch is solved
 * by one kernel launch (dsp_lp_solve_batch).  Each entry point below names the reference interface it
 * replaces; INTEGRATION.md shows the ctypes / Pyomo-plugin binding.
 *
 * Problem class (one template = one flowsheet x horizon x design mode):
 *
 *     min c'x + k   s.t.  A x = b,  0 <= x <= u         A: m x n, CSR, shared by the batch
 *     c = c0 + Cmap*cparams   b = b0 + Bmap*rparams   u = u0 + Umap*rparams   k = o0 + omap.rparams + ocmap.cparams
 *
 * Columns 0..nb-1 are the upper-bounded ones.  Rows must be ordered so that A*A' is banded with half
 * bandwidth w (multi-period flowsheets are block tridiagonal in time); asm_* is the assembly list of the
 * lower band of M = A*diag(d)*A':  M[i][i-k] = sum_{p in asm_ptr[i*(w+1)+k] ..} asm_val[p]*d[asm_col[p]].
 * dispatches_b200/lp_template.py computes all of it.
 *
 * Size limits: half bandwidth of A*A' <= 32 (padded to 1,2,4,8,16,32); any m, n -- the per-LP work region lives in shared
 * memory when it fits (up to ~27 000 doubles) and in a device workspace owned by the template handle otherwise.  A wider LP with
 * m <= 1024 goes through dsp_lp_template_create_dense (dense normal equations, below).
 *
 * All pointers in dsp_lp_solve_batch are DEVICE pointers, the call is stream-ordered and does not
 * synchronise.  dsp_lp_solve_batch_host takes HOST pointers and does the copies itself.
 * Return value: 0 on success, a negative DSP_E_* code on argument / launch errors.  Per-problem outcome
 * is reported only through status[] (DSP_OPTIMAL, ...), like SolverResults.solver.termination_condition.
 */
#ifndef DSP_LP_H
#define DSP_LP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dsp_template dsp_template;   /* opaque, owns device copies of the template */

/* sparse affine map in CSR: row r touches params idx[ptr[r]..ptr[r+1]) with coefficients val[..] */
typedef struct {
    const int32_t *ptr;
    const int32_t *idx;
    const double  *val;
} dsp_param_map;

typedef struct {
    int32_t m, n, nb, w;          /* rows, columns, bounded columns (first nb), half bandwidth of A A' */
    int32_t Pc, Pr;               /* lengths of cparams / rparams */
    const int32_t *A_ptr, *A_idx;  const double *A_val;        /* CSR, m rows                         */
    const int32_t *asm_ptr, *asm_col; const double *asm_val;   /* band assembly list, m*(w+1) entries  */
    const double *c0;  dsp_param_map cmap;                     /* n rows  over cparams                 */
    const double *b0;  dsp_param_map bmap;                     /* m rows  over rparams                 */
    const double *u0;  dsp_param_map umap;                     /* nb rows over rparams                 */
    double o0; const double *omap /*[Pr]*/; const double *ocmap /*[Pc]*/;
} dsp_template_desc;

typedef struct {
    double  tol;          /* relative duality-gap tolerance (default 1e-9)              */
    double  feas_tol;     /* relative primal / dual residual tolerance (default 1e-9)   */
    int32_t max_iter;     /* default 60                                                  */
    double  step_frac;    /* fraction of the step to the boundary (default 0.9995)       */
    int32_t device;       /* reserved (the current CUDA device is used); keep -1        */
    double  reg_primal;   /* proximal regularisation of D^-1 in scaled units (default 1e-8; applied as reg/max(1,x^2)): caps the scaling
                             of never-binding columns (throughput, slacks) so A D A' stays factorisable    */
    int32_t kernel;       /* DSP_KERNEL_AUTO (stage kernel when the template has one), _BAND, _STAGE, _STAGE_V1 */
} dsp_opts;

enum { DSP_KERNEL_AUTO = 0, DSP_KERNEL_BAND = 1, DSP_KERNEL_STAGE = 2 /* generation 2: several LPs per warp */,
       DSP_KERNEL_STAGE_V1 = 3 /* generation 1: lane per period, T <= 32 (kept as an independent implementation for tests) */,
       DSP_KERNEL_DENSE = 4 /* dense normal equations, one CTA per LP, m <= 1024: what a dense template runs (AUTO picks it there);
                               on a band template it replaces the band / stage kernels (a cross-check; no per-problem matrices) */ };

/* Stage descriptor of the wind+battery price-taker flowsheet (wind_battery_LMP.py:172-267, reduced form):
 * any T (T <= 96: on chip, several LPs per warp; longer, up to the reference's full-year 8736 periods of
 * run_pricetaker_wind_battery.py:57-58: one warp per LP with its state in a workspace owned by the handle -- csrc/dsp_stage2_long.cuh --
 * followed on the same stream by the band kernel in a retry mode that re-solves only the LPs left non-optimal, so the two launches
 * count as two in dsp_lp_launch_count), per period the columns g,i,o,s,e,p,q and rows r1 (state_evolution, battery.py:145-149),
 * r2 (accumulate_energy_throughput :151-153), r3 (state_of_charge_bounds :155-157, slack p),
 * r4 (wind_power.py:120-122 + splitter, slack q).  Lets dsp_lp_solve_batch run the stage kernels (several LPs per warp,
 * iterate in registers, partitioned block elimination: csrc/dsp_stage2.cuh) instead of the generic band kernel; results
 * are identical up to rounding.    */
typedef struct {
    int32_t T;
    double a, binv, half, delta, dur;   /* charging_eta, 1/discharging_eta, 1/2, degradation_rate, duration  */
    double k_rev;                       /* cost of g_t and o_t = k_rev * cparams[t]                          */
    int32_t wcf_off, p_off;             /* rparams: wind_kw*cf_t at wcf_off+t, battery kW at p_off            */
    const int32_t *col_idx;             /* [T*7] template column of (t, g,i,o,s,e,p,q), -1 if presolved away  */
    const int32_t *row_idx;             /* [T*4] template row of (t, r1..r4)                                  */
} dsp_stage_wb_desc;

/* Stage descriptor of the "single storage chain" family (csrc/dsp_stage_chain1.cuh): ONE row per period; every column appears in
 * one row (a flow of that period) or in two consecutive rows (the state carried to the next period: tank holdup,
 * nuclear_flowsheet_multiperiod_class.py:47-49, price_taker_analysis.py:175-178).  Nothing flowsheet specific: indices and row
 * coefficients of the template itself (dispatches_b200/lp_template.py: detect_chain1 finds them for any template); costs, right-hand
 * sides and bounds come from the template's parameter maps.  T <= 96, NF = 2 or 3 flow slots per period (absent: col_idx -1).                              */
typedef struct {
    int32_t T, NF;
    const int32_t *col_idx;     /* [T*(NF+1)] template column of (t, flow 0..NF-1 | state), -1 if absent                     */
    const int32_t *row_idx;     /* [T] template row of period t                                                              */
    const double  *coef;        /* [T*(NF+1)] coefficient of that column in row t                                            */
    const double  *coef_next;   /* [T] coefficient of the state of period t in row t+1 (0 for the last period)               */
} dsp_stage_chain1_desc;
int dsp_lp_template_set_stage_chain1(dsp_template *t, const dsp_stage_chain1_desc *d);

/* Per-problem status.  DSP_OPTIMAL means: relative primal/dual residuals < feas_tol and relative duality gap < tol; OR, when
 * the complementarity gap has converged (< tol) while residuals / gap sit at the rounding floor of the ill-conditioned normal
 * equations, residuals < 10 feas_tol and gap < 10 tol; OR complementarity < 1e-3 tol with residuals < 100 feas_tol and
 * gap < 1000 tol (the effective worst-case tolerance is therefore 1000 tol = 1e-6 relative on the LP part of the objective at
 * the defaults).  The stage-2 kernel's two looser branches also require |A x - b| < 10 feas_tol relative to the primal scale
 * itself, not to 1 + the scaled |b|.  DSP_INFEASIBLE is reported only for a negative
 * upper bound produced by Umap / rparams; other infeasible / unbounded LPs end as DSP_MAX_ITER / DSP_NUMERICAL.  Every kernel
 * applies one rule: u_j < -1e-9 * beta_b is infeasible, where beta_b = max(max_i |b_i|, max_j u_j) (1 if that is <= 0) is the
 * LP's primal scale; a bound above that is clamped to 0 and the LP is solved (the 1e-9 is a rounding margin, far inside the 1e-7
 * feasibility tolerance of CBC / HiGHS).  Only the bound is clamped: other data derived from the same parameter keep their value
 * (the wind+battery state-of-charge right-hand side duration * P stays at its tiny negative value), so such an LP may still be
 * infeasible by that rounding amount and end DSP_NUMERICAL / DSP_MAX_ITER, which of the two depending on the kernel.  An INFEASIBLE LP has obj = NaN, iters = iterations before the test (0 unless it is a retry), and,
 * when x / y are requested, rows of NaN.
 * iters counts the iterations of both attempts: an LP whose first attempt ends non-optimal is solved again (shorter step, stronger
 * proximal term) and reports first + second, so with max_iter = k a non-optimal LP reports 2k.                              */
enum { DSP_OPTIMAL = 0, DSP_MAX_ITER = 1, DSP_NUMERICAL = 2, DSP_INFEASIBLE = 3 };
enum { DSP_E_ARG = -1, DSP_E_CUDA = -2, DSP_E_SMEM = -3, DSP_E_BUSY = -4 /* a host call is already in flight on this handle */ };

/* Replaces: the per-LP model hand-over inside SolverFactory(..).solve(m) (Pyomo LP/NL writer), done once. */
int dsp_lp_template_create(const dsp_template_desc *desc, dsp_template **out);
void dsp_lp_template_destroy(dsp_template *t);

/* The same hand-over from a PLAIN standard-form LP: rows in any order, columns in any order, an upper bound >= 1e300 (or
 * +inf) marks an unbounded column (its umap row must be empty).  The library derives what dsp_template_desc asks of its caller
 * -- bounded columns first, a bandwidth-reducing (reverse Cuthill-McKee vs natural) row order of A A', the band assembly list --
 * and x / y of dsp_lp_solve_batch come back in the CALLER's column / row order.  This is the entry point a C binding or the
 * Pyomo walker uses (INTEGRATION.md); dsp_lp_analyze_csr is its host-only symbolic part (no CUDA call). */
typedef struct {
    int32_t m, n;                  /* rows of A x = b (inequalities carry the caller's slack columns), columns */
    int32_t Pc, Pr;
    const int32_t *A_ptr, *A_idx;  const double *A_val;        /* CSR, m rows                               */
    const double *c0;  dsp_param_map cmap;                     /* n rows over cparams (c0 may be NULL = 0)   */
    const double *b0;  dsp_param_map bmap;                     /* m rows over rparams (b0 may be NULL = 0)   */
    const double *u0;  dsp_param_map umap;                     /* n rows over rparams; u0[j] >= 1e300: none  */
    double o0; const double *omap /*[Pr] or NULL*/; const double *ocmap /*[Pc] or NULL*/;
} dsp_lp_desc;
int dsp_lp_template_create_csr(const dsp_lp_desc *desc, dsp_template **out);
int dsp_lp_analyze_csr(const dsp_lp_desc *desc, int32_t *nb, int32_t *w, int32_t *w_natural, int32_t *w_rcm,
                       int32_t *col_perm /*[n] or NULL*/, int32_t *row_perm /*[m] or NULL*/);
int dsp_lp_template_info(const dsp_template *t, int32_t *m, int32_t *n, int32_t *nb, int32_t *w);
/* The same hand-over for an LP whose A A' is NOT banded (a design size in a row of every period: solar_battery_hydrogen.py:205-236):
 * any bandwidth, m <= 1024 (larger: DSP_E_ARG).  dsp_lp_solve_batch then runs the dense kernel (csrc/dsp_dense.cuh): one CTA per LP,
 * M = A D A' dense, blocked LDL' over 64 x 64 tiles with the trailing updates on the FP64 tensor cores, M in a workspace owned by
 * the handle.  x / y come back in the caller's order; dsp_lp_template_info reports the true half bandwidth; DSP_KERNEL_BAND / _STAGE
 * on such a template and dsp_lp_template_set_matrix_params return DSP_E_ARG. */
int dsp_lp_template_create_dense(const dsp_lp_desc *desc, dsp_template **out);
/* Per-problem MATRIX coefficients for a template made by dsp_lp_template_create_csr:  A[row][col] = A0[row][col] + sum coef * rparams[param]
 * (row / col in the caller's order; the entry must be in A's pattern).  Needed where a design column is multiplied by per-scenario data --
 * wind system_capacity * capacity_factor[t] with a free wind size, wind_power.py:120-122 + wind_battery_LMP.py:212-216.  The band kernel then
 * re-derives A, A' and the band-assembly products per LP inside its work region (2 nnz + nasm more doubles per LP in flight).        */
int dsp_lp_template_set_matrix_params(dsp_template *t, int32_t count, const int32_t *row, const int32_t *col, const int32_t *param,
                                      const double *coef);

/* Optional: registers the stage structure of a wind+battery template (see dsp_stage_wb_desc). */
int dsp_lp_template_set_stage_wb(dsp_template *t, const dsp_stage_wb_desc *d);

void dsp_lp_default_opts(dsp_opts *o);

/* Replaces: the sweep loop of opt.solve(m) calls (one per scenario).  Device pointers, stream-ordered.
 *   cparams [N,Pc], rparams [N,Pr] (or [1,Pr] broadcast when rparams_stride == 0)
 *   obj [N]  objective c'x + k ; status [N] ; iters [N] ; x [N,n] or NULL ; y [N,m] or NULL          */
int dsp_lp_solve_batch(const dsp_template *t, int64_t N,
                       const double *cparams, const double *rparams, int64_t rparams_stride,
                       const dsp_opts *opts,
                       double *obj, int32_t *status, int32_t *iters, double *x, double *y,
                       void *cuda_stream);

/* Same with HOST pointers: pinned staging, H2D of the parameters, kernel, D2H of the results, one sync.
 * This is the call the Pyomo plugin / sweep drivers make; bench.py's "e2e" number times it.
 * Page-locked caller buffers are DMA'd directly (no staging copy) and go to the GPU in one piece unless the batch exceeds 65 536
 * LPs (then up to 4 chunks on two streams: the copy of one overlaps the kernel of the other); pageable buffers are staged in up to
 * 8 chunks so that the host memcpy overlaps too.  Not re-entrant per template handle: the staging
 * buffers and streams belong to the handle -- use one handle per host thread; a second concurrent call on the same
 * handle returns DSP_E_BUSY.                                                                            */
int dsp_lp_solve_batch_host(dsp_template *t, int64_t N,
                            const double *cparams, const double *rparams, int64_t rparams_stride,
                            const dsp_opts *opts,
                            double *obj, int32_t *status, int32_t *iters, double *x, double *y);

/* Introspection used by tests / bench: kernel launches issued so far, last launch geometry. */
int64_t dsp_lp_launch_count(void);
int dsp_lp_last_launch(int32_t *grid, int32_t *block, int32_t *smem_bytes, int32_t *problems_per_cta);
const char *dsp_lp_last_error(void);
const char *dsp_lp_version(void);
/* measured FP64 FMA throughput of the current device in TFLOP/s (micro-benchmark; -1 on error): denominator of the
 * FP64 roofline fraction reported by bench.py */
double dsp_lp_fp64_peak_tflops(void);

#ifdef __cplusplus
}
#endif
#endif
