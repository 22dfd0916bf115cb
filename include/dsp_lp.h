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
 * m <= 1024 goes through dsp_lp_template_create_dense (dense normal equations, below), one with m <= 4096 through
 * dsp_lp_template_create_dense_cluster (the same on a thread-block cluster per LP).
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
    double  step_frac;    /* fraction of the step to the boundary (default 0.9995), first attempt only (see below) */
    int32_t device;       /* reserved (the current CUDA device is used); keep -1        */
    double  reg_primal;   /* proximal regularisation of D^-1 in scaled units (default 1e-8; applied as reg/max(1,x^2)): caps the scaling
                             of never-binding columns (throughput, slacks) so A D A' stays factorisable.  First attempt only:
                             an LP whose first attempt ends MAX_ITER or NUMERICAL is solved again from the start point with
                             step_frac = 0.99 and 10 x reg_primal (100 x in the long-horizon stage kernel and in
                             DSP_KERNEL_BAND_SPLIT), and iters counts both attempts    */
    int32_t kernel;       /* DSP_KERNEL_AUTO (stage kernel when the template has one), _BAND, _STAGE, _STAGE_V1 */
} dsp_opts;

enum { DSP_KERNEL_AUTO = 0, DSP_KERNEL_BAND = 1, DSP_KERNEL_STAGE = 2 /* generation 2: several LPs per warp */,
       DSP_KERNEL_STAGE_V1 = 3 /* generation 1: lane per period, T <= 32 (kept as an independent implementation for tests) */,
       DSP_KERNEL_DENSE = 4 /* dense normal equations, one CTA per LP, m <= 1024: what a dense template runs (AUTO picks it there);
                               on a band template it replaces the band / stage kernels (a cross-check; no per-problem matrices) */,
       DSP_KERNEL_DENSE_CLUSTER = 5 /* dense normal equations, one thread-block cluster per LP, m <= 4096: what a dense cluster template
                                       runs (AUTO picks it there); on a band template a cross-check like DSP_KERNEL_DENSE */,
       DSP_KERNEL_BAND_SPLIT = 6 /* band template, the horizon split over the warp: one warp per LP, rows cut into 32 chunks, a
                                    partitioned (nested-dissection) band LDL' (csrc/dsp_band_split.cuh); the band kernel's iteration and
                                    status rules.  The band kernel follows on the same stream and re-solves only the LPs it leaves
                                    MAX_ITER / NUMERICAL (two launches).  Needs w <= 8 (w: the half bandwidth rounded up to 1, 2, 4 or
                                    8), m >= 64 w and a template without per-problem matrix coefficients; dense templates are refused;
                                    a stage descriptor is ignored, as with DSP_KERNEL_BAND.  dsp_lp_last_launch reports the split
                                    kernel's grid.  Not chosen by DSP_KERNEL_AUTO. */ };

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
enum { DSP_UNBOUNDED = 4 };        /* only dsp_lp_parametric returns it: the LP is unbounded past a breakpoint */
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
 * on such a template and dsp_lp_template_set_matrix_params return DSP_E_ARG (per-problem matrix coefficients of a dense template are
 * given at creation, below). */
int dsp_lp_template_create_dense(const dsp_lp_desc *desc, dsp_template **out);
/* The same with per-problem MATRIX coefficients, given at creation:  A[row][col] = A0[row][col] + sum coef * rparams[param], the terms of
 * one entry added in the order given (the semantics of dsp_lp_template_set_matrix_params; row / col in the caller's order).  Needed where
 * a design column is multiplied by per-scenario data -- the added-PV size times the capacity factor of every hour with a PV series per
 * scenario, solar_pv.py:82-84 + solar_battery_hydrogen.py:205-236.  An entry outside A's pattern or an index out of range is DSP_E_ARG;
 * count == 0 is dsp_lp_template_create_dense.  At LP load the dense kernel derives the LP's CSR and CSC values and the products of its
 * assembly list into the LP's workspace region (2 nnz + the assembly list's length more doubles per LP in flight). */
int dsp_lp_template_create_dense_with_matrix_params(const dsp_lp_desc *desc, int32_t count, const int32_t *row, const int32_t *col,
                                                    const int32_t *param, const double *coef, dsp_template **out);
/* The same hand-over (same rules and messages, count == 0: no per-problem matrix) for m <= 4096 (larger: DSP_E_ARG).  dsp_lp_solve_batch
 * then runs the dense cluster kernel: one LP per thread-block cluster of 4 CTAs (up to 32 tile rows of 64) or 8, the same iteration
 * and pivot rule as the dense kernel, a left-looking blocked LDL' and the substitutions split over the cluster's CTAs by tile row.  The
 * LP's tiles of M (m^2 / 2 doubles, padded to 64) live in the handle's workspace per cluster in flight.  DSP_KERNEL_BAND / _STAGE /
 * _STAGE_V1 / _DENSE on such a template and dsp_lp_template_set_matrix_params return DSP_E_ARG. */
int dsp_lp_template_create_dense_cluster(const dsp_lp_desc *desc, int32_t count, const int32_t *row, const int32_t *col,
                                         const int32_t *param, const double *coef, dsp_template **out);
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

/* Sensitivities of a solved batch: reduced costs and the objective's derivative in every batch parameter, a post-pass over the
 * (status, x, y) that dsp_lp_solve_batch returned for the same cparams / rparams.  For one LP with returned (x, y):
 *     rc            = c - A'y            A: the LP's own matrix, A0 + sum coef * rparams[param] (per-problem matrix terms)
 *     d obj / d cp  = Cmap' x + ocmap
 *     d obj / d rp  = Bmap' y + Umap' min(rc, 0) + omap - sum over the matrix terms (i, j, q, coef) of coef * y_i * x_j
 * min(rc_j, 0) is minus the upper-bound dual that is optimal for this y.  Where the optimum is unique these are the gradient of the
 * optimal value obj = c'x + k (envelope theorem); at a degenerate optimum they are a subgradient: obj is convex in rparams when rparams
 * does not enter A, and concave in cparams.
 * DEVICE pointers, stream-ordered, no synchronisation, like dsp_lp_solve_batch (the same rparams_stride == 0 broadcast); x [N,n], y [N,m],
 * rc [N,n], d_cparams [N,Pc], d_rparams [N,Pr] in the same (caller's) order as dsp_lp_solve_batch's x and y.  Each output may be NULL; an
 * LP whose status is not DSP_OPTIMAL gets rows of NaN in every requested output.  Every entry is summed in a fixed order by one thread:
 * the results are bitwise reproducible and do not depend on where an LP sits in the batch.  One kernel launch per call (none when
 * N == 0 or every output is NULL); the first call on a handle builds its structure on the host.
 * DSP_E_ARG: NULL handle, N < 0, NULL status / x / y, NULL cparams with Pc > 0 or NULL rparams with Pr > 0. */
int dsp_lp_sensitivities(const dsp_template *t, int64_t N,
                         const double *cparams, const double *rparams, int64_t rparams_stride,
                         const int32_t *status, const double *x, const double *y,
                         double *rc /*[N,n] or NULL*/, double *d_cparams /*[N,Pc] or NULL*/, double *d_rparams /*[N,Pr] or NULL*/,
                         void *cuda_stream);

/* Crossover of a solved batch: for every LP whose status is DSP_OPTIMAL, a basic optimal solution (a vertex) of the same LP, from the
 * (x, y) that dsp_lp_solve_batch returned for the same cparams / rparams.  An interior-point solve returns the analytic centre of the
 * optimal face; a simplex solver (CBC, Gurobi, HiGHS) returns a vertex with basis duals, and this is that answer.  m <= 1024.
 * The LP is  min c'x + k, A x = b, 0 <= x <= u  in the caller's column / row order, with every per-problem parameter and matrix term.
 * A basis is col_status [n] (0: at 0, 1: basic, 2: at u) and row_basic [m] (1: the row's artificial column, a unit column with bounds
 * [0, 0], is basic: a redundant row), m basic variables in all.  The outputs are that basis, its basic solution x_out (every nonbasic
 * column exactly at its bound; a column with u = 0 is reported at the bound the sign of its reduced cost asks for), its duals
 * y_out = B^-T c_B and obj_out = c'x + k.
 * Algorithm (csrc/dsp_crossover.cuh, DESIGN.md 4.6): crash a basis from the most interior columns, push every other column inside its
 * bounds onto a bound, then bounded primal / dual simplex pivots until the basis is primal and dual feasible within 1e-9 of the primal
 * scale max(1, |b|_inf, |u_finite|_inf) and of |c|_inf, and every artificial a column can replace is pivoted out.  One CTA per LP
 * with a dense explicit B^-1 (in shared memory up to m ~ 160, else about 8 m^2 bytes per CTA in flight of the handle's workspace).
 * xstatus [N]: DSP_OPTIMAL (the final basic solution is primal and dual feasible within tolerance), DSP_MAX_ITER (max_pivots pivots;
 * <= 0: DSP_CROSSOVER_DEFAULT_PIVOTS(m, n)), DSP_NUMERICAL (a singular reinversion, or a basis primal and dual infeasible at once);
 * an LP whose input status is not DSP_OPTIMAL keeps that status and gets NaN in x_out / y_out / obj_out, -1 in col_status /
 * row_basic and 0 pivots.  An LP that ends DSP_MAX_ITER or DSP_NUMERICAL gets the state the crossover stopped in: x_out / y_out /
 * obj_out are finite but are not a basic optimal solution (x_out need not even be one of the LP's basic solutions), and col_status is
 * -1 for a column the push had not yet moved onto a bound; callers should use the solve's own x / y for such LPs.
 * pivots [N]: basis changes and bound flips after the crash.
 * DEVICE pointers, stream-ordered, no synchronisation, the rparams_stride == 0 broadcast of dsp_lp_solve_batch.  Results are bitwise
 * reproducible and do not depend on where an LP sits in the batch.  One kernel launch per call (none when N == 0); the first call on
 * a handle builds its structure on the host.
 * DSP_E_ARG: NULL handle, N < 0, m > 1024 ("crossover takes m <= 1024"), and for N > 0 NULL status / x / y / obj_out / x_out / y_out /
 * xstatus, NULL cparams with Pc > 0 or NULL rparams with Pr > 0. */
#define DSP_CROSSOVER_DEFAULT_PIVOTS(m, n) (10 * ((m) + (n)))
int dsp_lp_crossover(const dsp_template *t, int64_t N,
                     const double *cparams, const double *rparams, int64_t rparams_stride,
                     const int32_t *status, const double *x, const double *y,
                     int32_t max_pivots,
                     double *obj_out /*[N]*/, double *x_out /*[N,n]*/, double *y_out /*[N,m]*/,
                     int8_t *col_status /*[N,n] or NULL*/, int8_t *row_basic /*[N,m] or NULL*/,
                     int32_t *xstatus /*[N]*/, int32_t *pivots /*[N] or NULL*/, void *cuda_stream);

/* Ranging over given bases: for every LP and every direction k, the interval [theta_lo, theta_hi] (theta_lo <= 0 <= theta_hi, +-inf
 * where unbounded) of theta over which the LP's basis stays optimal when the parameters move to (cp + theta dir_c[k], rp + theta
 * dir_r[k]), all others fixed; Gurobi's SAObj* / SARHS* answer, for the batch parameters.  m <= 1024.
 * The LP is dsp_lp_crossover's (caller's order, every per-problem parameter and matrix term) and so is the basis: col_status [N,n] and
 * row_basic [N,m], e.g. dsp_lp_crossover's outputs with its status as xstatus.  Only the basis is read: x_B, y and d = c - A'y are
 * recomputed from it.  The basis stays optimal while
 *   primal: 0 <= x_B(theta) <= u_B(theta), u_j(theta) >= 0 for a nonbasic column at u, a basic artificial stays 0 (else [0, 0]);
 *   dual:   d_j(theta) >= 0 at 0, <= 0 at u, for every nonbasic column except those fixed at 0 along the direction (u_j = 0 and no
 *           change of u_j); nonbasic artificials impose nothing.  A column with u_j = 0 may sit at either bound, but where the
 *           direction changes u_j and d_j has the wrong sign for its bound beyond tolerance, the side on which u_j grows is 0.
 * An entry within the crossover's tolerance of its bound (1e-9 of the primal scale max(1, |b|_inf, |u_finite|_inf), of |c|_inf on the
 * dual side) counts as on it: a direction pushing it outwards gives 0 on that side.  An entry whose rate of change is at most 1e-9 of
 * the direction's scale (max(|Bmap dir_r|_inf, |Umap dir_r|_inf) on the primal side, |Cmap dir_c|_inf on the dual side) does not block.
 * Inside the range obj(theta) = obj + dobj theta + d2obj theta^2 / 2 exactly; d2obj = 2 dc'dx is 0 unless the direction moves both c
 * and b / u.  A direction with a nonzero dir_r entry on a parameter that enters a matrix term moves A: its column of every output is
 * NaN.
 * Directions: dir_c [K,Pc] and dir_r [K,Pr] shared by the batch (dir_stride == 0), or per LP [N,K,Pc] / [N,K,Pr] (dir_stride != 0);
 * a NULL dir_c or dir_r does not move those parameters.
 * rstatus [N]: DSP_OPTIMAL (ranges computed), DSP_NUMERICAL (the basis does not have m members or has a column at an infinite bound,
 * its reinversion is singular, or it is not primal and dual feasible within the tolerances above at theta = 0), or the input xstatus
 * where that is not DSP_OPTIMAL; every LP that is not DSP_OPTIMAL gets NaN rows.
 * Algorithm (csrc/dsp_ranging.cuh, DESIGN.md 4.7): dsp_lp_crossover's layout, one CTA per LP, B^-1 by Gauss-Jordan, then per direction
 * two dense m x m products and the ratio tests.  DEVICE pointers, stream-ordered, no synchronisation, the rparams_stride == 0
 * broadcast of dsp_lp_solve_batch.  Results are bitwise reproducible and do not depend on where an LP sits in the batch.  One kernel
 * launch per call (none when N == 0 or K == 0).
 * DSP_E_ARG: NULL handle, N < 0, K < 0, m > 1024 ("ranging takes m <= 1024"), and for N > 0 and K > 0 NULL xstatus / col_status /
 * row_basic / theta_lo / theta_hi / rstatus, NULL cparams with Pc > 0 or NULL rparams with Pr > 0. */
int dsp_lp_ranging(const dsp_template *t, int64_t N,
                   const double *cparams, const double *rparams, int64_t rparams_stride,
                   const int32_t *xstatus, const int8_t *col_status, const int8_t *row_basic,
                   int32_t K, const double *dir_c /*[K,Pc] or NULL*/, const double *dir_r /*[K,Pr] or NULL*/,
                   int64_t dir_stride /* 0: directions shared by the batch; else per LP, [N,K,Pc] / [N,K,Pr] */,
                   double *theta_lo /*[N,K]*/, double *theta_hi /*[N,K]*/,
                   double *dobj /*[N,K] or NULL*/, double *d2obj /*[N,K] or NULL*/,
                   int32_t *rstatus /*[N]*/, void *cuda_stream);

/* Parametric walk over given bases: for every LP and every direction k, the exact optimal value of the LP at the parameters
 * (cp + theta dir_c[k], rp + theta dir_r[k]) for theta from 0 up to theta_end[k] (+inf allowed), as an event log of the basis changes
 * along the way; a parametric simplex from dsp_lp_ranging's range to the next basis, repeated.  m <= 1024.
 * The LP and the basis are dsp_lp_ranging's (col_status [N,n], row_basic [N,m], xstatus [N], e.g. dsp_lp_crossover's outputs); the basis
 * must be optimal at theta = 0.  At every theta the LP is formed afresh from the parameters, p + theta dir with one fma each.
 * Outputs per (LP, direction) pair, [N,K,S] (S events at most) and [N,K]:
 *   event 0: theta = 0, obj = c'x + k of the basis, enter = leave = leave_to = -1;
 *   event e >= 1: one basis change or bound flip at theta[e] >= theta[e-1]; obj[e] recomputed from the new basis there; enter the
 *     entering variable (n + i: the artificial of row i; -1 for a bound flip), leave the leaving or flipped variable, leave_to the
 *     bound it goes to (0: at 0, 2: at u);
 *   dobj[e], d2obj[e]: the right derivatives of the segment that starts at event e, so that up to the next event (or theta_end)
 *     obj(theta) = obj[e] + dobj[e] (theta - theta[e]) + d2obj[e] (theta - theta[e])^2 / 2 exactly (d2obj = 0 unless the direction
 *     moves both c and b / u).  Events at equal theta are degenerate pivots; the last of them defines the segment.  Applying the
 *     events in order to the start basis gives the basis of every segment.  The curve is convex along a direction that moves only b / u
 *     and concave along one that moves only c;
 *   a walk that ends INFEASIBLE or UNBOUNDED has a last event at the breakpoint with enter = leave = leave_to = -1 and NaN dobj / d2obj:
 *     the curve stops there;
 *   entries from count on are NaN (-1 for enter / leave / leave_to).
 * pstatus [N,K]: DSP_OPTIMAL (the walk reached theta_end, or no basis change happens past the last event), DSP_INFEASIBLE (past the
 * last event no point is feasible: a dual simplex step finds no entering column, or an upper bound at which a column sits reaches 0),
 * DSP_UNBOUNDED (past the last event the objective is unbounded below), DSP_MAX_ITER (S events before theta_end; the log so far is
 * kept), DSP_NUMERICAL (the start basis is not a basis with every nonbasic column at a finite bound, its reinversion is singular, it is
 * not primal and dual feasible within dsp_lp_ranging's tolerances, or after an event a reinversion is singular or the basis is primal
 * and dual infeasible at once; a direction with a nonzero dir_r entry on a parameter that enters a matrix term, which moves A, gets
 * count 0 and NaN rows), or the input xstatus where that is not DSP_OPTIMAL (count 0, NaN rows).
 * Rules at a breakpoint (csrc/dsp_parametric.cuh, DESIGN.md 4.8): the blocking entry of the range is the one with the smallest ratio,
 * primal before dual, then the lowest variable index; a basic variable at a bound leaves by a dual simplex pivot, a reduced cost at 0
 * enters by a primal simplex pivot (or flips to its other bound), each ratio test ordered by (ratio, its derivative in theta, the
 * larger |alpha|, index) so that the new basis stays optimal just past the breakpoint; a fixed column (u = 0) that the direction
 * unfixes at the bound its reduced cost does not ask for flips at once.  After 50 zero-length events in a row, ratio-test ties go to
 * the lowest index (not Bland's rule: a walk that cycles ends DSP_MAX_ITER at S events).  An artificial leaves to 0 (leave_to 0).
 * Exactness: on every template the tests cover, each segment's objective is the exact optimum to 1e-9 relative and each breakpoint
 * the exact end of its basis' range to 1e-8.  On LPs with redundant rows and long degenerate stretches (the PV + battery + hydrogen
 * design templates) a replayed segment basis may miss exact optimality by a rounding-sized violation (a degenerate basic variable at
 * about -1e-13 after a primal pivot whose ratio test skips it: its entry in the pivot column is below the pivot tolerance); the
 * objective and breakpoints still hold to those bars.
 * Directions: dir_c / dir_r as dsp_lp_ranging's (shared with dir_stride == 0, else per LP); theta_end [K], or [N,K] per LP.  One CTA
 * per (LP, direction) pair.  DEVICE pointers, stream-ordered; the call reads theta_end back to check it (it waits for the stream up
 * to that point), the walks run asynchronously.  The rparams_stride == 0 broadcast of dsp_lp_solve_batch.  Results are bitwise
 * reproducible and do not depend on where a pair sits in the batch.  One kernel launch per call (none when N == 0 or K == 0).
 * DSP_E_ARG: NULL handle, N < 0, K < 0, S < 1, m > 1024 ("parametric takes m <= 1024"), and for N > 0 and K > 0 NULL xstatus /
 * col_status / row_basic / theta / obj / dobj / count / pstatus, NULL theta_end or a negative or NaN entry of it, NULL cparams with
 * Pc > 0 or NULL rparams with Pr > 0. */
int dsp_lp_parametric(const dsp_template *t, int64_t N,
                      const double *cparams, const double *rparams, int64_t rparams_stride,
                      const int32_t *xstatus, const int8_t *col_status, const int8_t *row_basic,
                      int32_t K, const double *dir_c /*[K,Pc] or NULL*/, const double *dir_r /*[K,Pr] or NULL*/,
                      int64_t dir_stride /* 0: shared by the batch; else per LP, [N,K,Pc] / [N,K,Pr] */,
                      const double *theta_end /*[K], or [N,K] when dir_stride != 0; each >= 0, +inf allowed*/,
                      int32_t S /* events per walk, >= 1 */,
                      double *theta /*[N,K,S]*/, double *obj /*[N,K,S]*/, double *dobj /*[N,K,S]*/, double *d2obj /*[N,K,S] or NULL*/,
                      int32_t *enter /*[N,K,S] or NULL*/, int32_t *leave /*[N,K,S] or NULL*/, int8_t *leave_to /*[N,K,S] or NULL*/,
                      int32_t *count /*[N,K]*/, int32_t *pstatus /*[N,K]*/, void *cuda_stream);

/* Introspection used by tests / bench: kernel launches issued so far, last launch geometry (grid in CTAs, block, dynamic shared
 * memory; problems_per_cta: LPs per CTA, or for the dense cluster kernel the cluster size in CTAs). */
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
