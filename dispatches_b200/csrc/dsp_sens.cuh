// dsp_sens.cuh -- sensitivity post-pass of a solved batch (dsp_lp_sensitivities, include/dsp_lp.h).
//
// For one LP  min c'x + k  s.t.  A x = b, 0 <= x <= u  with the returned (x, y):
//     rc            = c - A'y                                   (A: the LP's own matrix, every entry A0 + sum coef * rp[param])
//     d obj / d cp  = Cmap' x + ocmap
//     d obj / d rp  = Bmap' y + Umap' min(rc, 0) + omap - sum over matrix terms (i, j, q, coef) of coef * y_i * x_j
// min(rc_j, 0) is minus the upper-bound dual w_j that is optimal for this y, so (y, -w) is an element of the subdifferential of the
// optimal value in (b, u): a gradient where the optimum is unique, a subgradient otherwise.
//
// Layout: persistent CTAs, one warp per LP, LPs handed out grid-stride.  Every output entry has one owner lane that sums its terms in
// a fixed order (no atomics, no shuffles), so the results are bitwise reproducible and do not depend on where an LP sits in the batch.
// The template structure is one blob in the CALLER's column / row order (the order x, y and rc have in memory), built on the host once
// per handle; a CTA stages it into shared memory when it fits, else reads it through the read-only data path.
//
// Plain C++ over a lane index: tests/emu compiles this file with g++ on the SIMT emulator and checks it against the numpy mirror.
#pragma once

#include <string.h>

#include <vector>

namespace sens {

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define SNS __device__ __forceinline__
#else
#define SNS inline
#endif

// element offsets of the blob's arrays: doubles first (from the blob's start), then int32 (from ioff bytes)
struct Layout {
    // doubles
    long long c0, At_val, cm_val, omap, ocmap, cT_val, bT_val, uT_val, tc_coef, tp_coef;
    // int32
    long long At_ptr, At_idx, cm_ptr, cm_idx, cT_ptr, cT_col, bT_ptr, bT_row, uT_ptr, uT_col, tc_ptr, tc_param, tp_ptr, tp_row, tp_col;
    long long ioff;      // byte offset of the int32 part (a multiple of 8)
    long long bytes;     // whole blob, a multiple of 16
};

struct Params {
    int m, n, Pc, Pr;
    long long N;
    const double *cparams, *rparams;
    long long rstride;
    const int *status;
    const double *x, *y;
    double *rc, *dcp, *drp;           // each may be null
    const unsigned char *blob;        // global copy of the structure
    Layout L;
    int blob_in_smem;
};

// views of the blob at base (shared or global)
struct View {
    const double *c0, *At_val, *cm_val, *omap, *ocmap, *cT_val, *bT_val, *uT_val, *tc_coef, *tp_coef;
    const int *At_ptr, *At_idx, *cm_ptr, *cm_idx, *cT_ptr, *cT_col, *bT_ptr, *bT_row, *uT_ptr, *uT_col, *tc_ptr, *tc_param, *tp_ptr,
        *tp_row, *tp_col;
};

SNS View view_of(const unsigned char *base, const Layout &L) {
    const double *d = (const double *)base;
    const int *i = (const int *)(base + L.ioff);
    View v;
    v.c0 = d + L.c0; v.At_val = d + L.At_val; v.cm_val = d + L.cm_val; v.omap = d + L.omap; v.ocmap = d + L.ocmap;
    v.cT_val = d + L.cT_val; v.bT_val = d + L.bT_val; v.uT_val = d + L.uT_val; v.tc_coef = d + L.tc_coef; v.tp_coef = d + L.tp_coef;
    v.At_ptr = i + L.At_ptr; v.At_idx = i + L.At_idx; v.cm_ptr = i + L.cm_ptr; v.cm_idx = i + L.cm_idx; v.cT_ptr = i + L.cT_ptr;
    v.cT_col = i + L.cT_col; v.bT_ptr = i + L.bT_ptr; v.bT_row = i + L.bT_row; v.uT_ptr = i + L.uT_ptr; v.uT_col = i + L.uT_col;
    v.tc_ptr = i + L.tc_ptr; v.tc_param = i + L.tc_param; v.tp_ptr = i + L.tp_ptr; v.tp_row = i + L.tp_row;
    v.tp_col = i + L.tp_col;
    return v;
}

// a load of template structure: through the read-only data path when it sits in global memory (G), a plain load from shared memory
template <bool G, class V>
SNS V ld(const V *p) {
#if defined(__CUDA_ARCH__)
    if (G) return __ldg(p);
#endif
    return *p;
}

// reduced cost of column j:  c0_j + sum Cmap[j,:] cp  -  sum_i A_ij y_i, every A_ij the LP's own entry A0_ij + sum coef rp[param]
template <bool G>
SNS double reduced_cost(const View &v, int j, const double *cp, const double *rp, const double *y) {
    double c = ld<G>(v.c0 + j);
    for (int e = ld<G>(v.cm_ptr + j), e1 = ld<G>(v.cm_ptr + j + 1); e < e1; ++e) c = fma(ld<G>(v.cm_val + e), cp[ld<G>(v.cm_idx + e)], c);
    double r = c;
    for (int e = ld<G>(v.At_ptr + j), e1 = ld<G>(v.At_ptr + j + 1); e < e1; ++e) {
        double a = ld<G>(v.At_val + e);
        for (int k = ld<G>(v.tc_ptr + e), k1 = ld<G>(v.tc_ptr + e + 1); k < k1; ++k) a = fma(ld<G>(v.tc_coef + k), rp[ld<G>(v.tc_param + k)], a);
        r = fma(-a, y[ld<G>(v.At_idx + e)], r);
    }
    return r;
}

// the outputs of LP p, computed by the 32 lanes of one warp (lane: 0..31); entry k of every output is owned by lane k % 32
template <bool G>
SNS void lp_body(const Params &P, const View &v, long long p, int lane) {
    const int n = P.n, Pc = P.Pc, Pr = P.Pr;
    if (P.status[p] != 0) {       // not DSP_OPTIMAL: rows of NaN
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        if (P.rc) for (int j = lane; j < n; j += 32) P.rc[p * n + j] = nan;
        if (P.dcp) for (int q = lane; q < Pc; q += 32) P.dcp[p * Pc + q] = nan;
        if (P.drp) for (int q = lane; q < Pr; q += 32) P.drp[p * Pr + q] = nan;
        return;
    }
    const double *x = P.x + p * n, *y = P.y + p * P.m;
    const double *cp = P.cparams ? P.cparams + p * Pc : nullptr;
    const double *rp = P.rparams ? P.rparams + p * P.rstride : nullptr;
    if (P.rc)
        for (int j = lane; j < n; j += 32) P.rc[p * n + j] = reduced_cost<G>(v, j, cp, rp, y);
    if (P.dcp)
        for (int q = lane; q < Pc; q += 32) {
            double s = 0.0;
            for (int e = ld<G>(v.cT_ptr + q), e1 = ld<G>(v.cT_ptr + q + 1); e < e1; ++e) s = fma(ld<G>(v.cT_val + e), x[ld<G>(v.cT_col + e)], s);
            P.dcp[p * Pc + q] = s + ld<G>(v.ocmap + q);
        }
    if (P.drp)
        for (int q = lane; q < Pr; q += 32) {
            double s = 0.0;
            for (int e = ld<G>(v.bT_ptr + q), e1 = ld<G>(v.bT_ptr + q + 1); e < e1; ++e) s = fma(ld<G>(v.bT_val + e), y[ld<G>(v.bT_row + e)], s);
            for (int e = ld<G>(v.uT_ptr + q), e1 = ld<G>(v.uT_ptr + q + 1); e < e1; ++e) {
                const double r = reduced_cost<G>(v, ld<G>(v.uT_col + e), cp, rp, y);
                s = fma(ld<G>(v.uT_val + e), r < 0.0 ? r : 0.0, s);
            }
            s += ld<G>(v.omap + q);
            for (int e = ld<G>(v.tp_ptr + q), e1 = ld<G>(v.tp_ptr + q + 1); e < e1; ++e)
                s = fma(-ld<G>(v.tp_coef + e) * y[ld<G>(v.tp_row + e)], x[ld<G>(v.tp_col + e)], s);
            P.drp[p * Pr + q] = s;
        }
}

// ---- host: the structure blob
// A template in internal order (what dsp_lp.cu keeps on the host): the CSR of A0, the parameter maps (umap: the first nb columns),
// the caller column / row of every internal column / row (empty: identity) and the per-problem matrix terms (CSR position, rparams
// index, coefficient) in the caller's order.
struct HostTemplate {
    int m, n, nb, Pc, Pr;
    const std::vector<int> &A_ptr, &A_idx;
    const std::vector<double> &A_val;
    const std::vector<int> &col_perm, &row_perm;
    const std::vector<double> &c0;
    const std::vector<int> &cm_ptr, &cm_idx;
    const std::vector<double> &cm_val;
    const std::vector<int> &bm_ptr, &bm_idx;
    const std::vector<double> &bm_val;
    const std::vector<int> &um_ptr, &um_idx;
    const std::vector<double> &um_val;
    const std::vector<double> &omap, &ocmap;
    const std::vector<int> &t_q, &t_param;
    const std::vector<double> &t_coef;
};

// entries (key, idx, idx2, val) grouped by key in [0, nkey), stably: entries pushed in ascending idx stay so within a group; dst[e]:
// where pushed entry e landed
struct Grouped {
    std::vector<int> ptr, idx, idx2, dst;
    std::vector<double> val;
};
inline Grouped group(int nkey, const std::vector<int> &key, const std::vector<int> &idx, const std::vector<int> &idx2,
                     const std::vector<double> &val) {
    Grouped G;
    G.ptr.assign(nkey + 1, 0);
    for (int k : key) G.ptr[k + 1]++;
    for (int k = 0; k < nkey; ++k) G.ptr[k + 1] += G.ptr[k];
    std::vector<int> fill(G.ptr.begin(), G.ptr.end() - 1);
    G.idx.resize(key.size()); G.val.resize(key.size()); G.idx2.resize(idx2.size()); G.dst.resize(key.size());
    for (size_t e = 0; e < key.size(); ++e) {
        const int d = G.dst[e] = fill[key[e]]++;
        G.idx[d] = idx[e]; G.val[d] = val[e];
        if (!idx2.empty()) G.idx2[d] = idx2[e];
    }
    return G;
}

// The structure in the caller's column / row order: the CSC of A0 and c0, Cmap by column; the transposed maps Cmap', Bmap', Umap' by
// parameter; the matrix terms grouped by CSC entry (param) and by parameter (row, column).  Lists run in ascending caller index,
// matrix terms in the caller's order within a group.  Returns the layout; blob receives the bytes.
inline Layout build_blob(const HostTemplate &T, std::vector<unsigned char> &blob) {
    const int m = T.m, n = T.n;
    std::vector<int> ccol(n), crow(m), rpos(m), kpos(n);       // caller column / row of an internal one, and the inverses
    for (int k = 0; k < n; ++k) ccol[k] = T.col_perm.empty() ? k : T.col_perm[k];
    for (int k = 0; k < m; ++k) crow[k] = T.row_perm.empty() ? k : T.row_perm[k];
    for (int k = 0; k < m; ++k) rpos[crow[k]] = k;
    for (int k = 0; k < n; ++k) kpos[ccol[k]] = k;
    std::vector<int> qrow(T.A_ptr[m]);
    for (int i = 0; i < m; ++i) for (int q = T.A_ptr[i]; q < T.A_ptr[i + 1]; ++q) qrow[q] = i;
    std::vector<int> key, idx, idx2;
    std::vector<double> val;
    auto clear = [&] { key.clear(); idx.clear(); idx2.clear(); val.clear(); };
    auto push = [&](int k, int i, double v) { key.push_back(k); idx.push_back(i); val.push_back(v); };
    std::vector<int> pushed(T.A_ptr[m]);                      // push index of every CSR position
    for (int R = 0; R < m; ++R)
        for (int q = T.A_ptr[rpos[R]]; q < T.A_ptr[rpos[R] + 1]; ++q) { pushed[q] = (int)key.size(); push(ccol[T.A_idx[q]], R, T.A_val[q]); }
    const Grouped At = group(n, key, idx, idx2, val);
    std::vector<double> c0(n);
    clear();
    for (int C = 0; C < n; ++C) {
        c0[C] = T.c0[kpos[C]];
        for (int e = T.cm_ptr[kpos[C]]; e < T.cm_ptr[kpos[C] + 1]; ++e) push(C, T.cm_idx[e], T.cm_val[e]);
    }
    const Grouped Cm = group(n, key, idx, idx2, val);
    clear();
    for (int C = 0; C < n; ++C)
        for (int e = T.cm_ptr[kpos[C]]; e < T.cm_ptr[kpos[C] + 1]; ++e) push(T.cm_idx[e], C, T.cm_val[e]);
    const Grouped CT = group(T.Pc, key, idx, idx2, val);
    clear();
    for (int R = 0; R < m; ++R)
        for (int e = T.bm_ptr[rpos[R]]; e < T.bm_ptr[rpos[R] + 1]; ++e) push(T.bm_idx[e], R, T.bm_val[e]);
    const Grouped BT = group(T.Pr, key, idx, idx2, val);
    clear();
    for (int C = 0; C < n; ++C)
        if (kpos[C] < T.nb)
            for (int e = T.um_ptr[kpos[C]]; e < T.um_ptr[kpos[C] + 1]; ++e) push(T.um_idx[e], C, T.um_val[e]);
    const Grouped UT = group(T.Pr, key, idx, idx2, val);
    clear();
    for (size_t e = 0; e < T.t_q.size(); ++e) push(At.dst[pushed[T.t_q[e]]], T.t_param[e], T.t_coef[e]);
    const Grouped TC = group(T.A_ptr[m], key, idx, idx2, val);
    clear();
    for (size_t e = 0; e < T.t_q.size(); ++e) { push(T.t_param[e], crow[qrow[T.t_q[e]]], T.t_coef[e]); idx2.push_back(ccol[T.A_idx[T.t_q[e]]]); }
    const Grouped TP = group(T.Pr, key, idx, idx2, val);
    // the doubles, then the int32 arrays
    Layout L;
    std::vector<double> dv;
    std::vector<int> iv;
    auto pd = [&dv](const std::vector<double> &v) { const long long at = (long long)dv.size(); dv.insert(dv.end(), v.begin(), v.end()); return at; };
    auto pi = [&iv](const std::vector<int> &v) { const long long at = (long long)iv.size(); iv.insert(iv.end(), v.begin(), v.end()); return at; };
    L.c0 = pd(c0); L.At_val = pd(At.val); L.cm_val = pd(Cm.val); L.omap = pd(T.omap); L.ocmap = pd(T.ocmap); L.cT_val = pd(CT.val);
    L.bT_val = pd(BT.val); L.uT_val = pd(UT.val); L.tc_coef = pd(TC.val); L.tp_coef = pd(TP.val);
    L.At_ptr = pi(At.ptr); L.At_idx = pi(At.idx); L.cm_ptr = pi(Cm.ptr); L.cm_idx = pi(Cm.idx); L.cT_ptr = pi(CT.ptr); L.cT_col = pi(CT.idx);
    L.bT_ptr = pi(BT.ptr); L.bT_row = pi(BT.idx); L.uT_ptr = pi(UT.ptr); L.uT_col = pi(UT.idx); L.tc_ptr = pi(TC.ptr);
    L.tc_param = pi(TC.idx); L.tp_ptr = pi(TP.ptr); L.tp_row = pi(TP.idx); L.tp_col = pi(TP.idx2);
    L.ioff = (long long)dv.size() * 8;
    L.bytes = (L.ioff + (long long)iv.size() * 4 + 15) / 16 * 16;
    blob.assign((size_t)L.bytes, 0);
    if (!dv.empty()) memcpy(blob.data(), dv.data(), dv.size() * 8);
    if (!iv.empty()) memcpy(blob.data() + L.ioff, iv.data(), iv.size() * 4);
    return L;
}

}  // namespace sens
