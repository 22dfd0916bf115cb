// dsp_band.cuh -- warp-level band LDL' factorisation and substitution sweeps of the generic band kernel (dsp_lp.cu).
//
// Storage (one LP, one warp): lower band of M = A D A', row-major, W1 = W + 1 slots per row: Mb[i*W1 + k] = M[i][i-k]; the array
// carries W zero rows in front and behind, the solve vector W zero entries in front and behind (no bounds checks in the sweeps).
// After the factorisation the diagonal slot holds 1/d_i (0 for a non-positive pivot) and the off-diagonal slots the UNSCALED
// column entries L[i][i-k] * d_{i-k}.
//
// The sweeps walk the band IN PLACE: every pivot step is load -> FMA -> store -> __syncwarp on the memory the band lives in -- shared
// memory in the "smem" / "hybrid" placements of dsp_lp.cu, the L1-cached global workspace in the "ws" placement (the active window of
// a sweep stays in L1, so a step costs about the same there).  A register-window variant (active window in registers sliding by warp
// shuffles, band streamed with loads issued 8 steps ahead; bit-identical results on the emulator) was tried and rejected as
// slower -- in the workspace placement the time is in the element-wise / CSR passes that stream the per-LP vectors through L2, not in the sweeps.
//
// Plain C++ over warp builtins: tests/emu compiles this file with g++ on the SIMT emulator and checks it against a dense solve.
#pragma once

namespace band {

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define BND __device__ __forceinline__
#else
#define BND inline
#endif
constexpr unsigned BFULL = 0xffffffffu;

BND double dmaxd(double a, double b) { return a > b ? a : b; }
BND double frcpd(double x) {          // reciprocal: MUFU seed + 2 Newton steps (no IEEE division)
    double r;
#if defined(__CUDA_ARCH__)
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#else
    r = (double)(1.0f / (float)x);     // emulation: any ~20-bit seed
    if (!(r == r) || r == 0.0 || r > 1e300 || r < -1e300) r = 1.0 / x;
#endif
    double e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    e = fma(-x, r, 1.0);
    return fma(r, e, r);
}

// ------------------------------------------------------------------------------------------------------- in place
template <int W>
BND void band_factor(double *Mb, int m, int lane) {
    constexpr int W1 = W + 1, NP = W * W, PASSES = (NP + 31) / 32;
    int off_lr[PASSES], off_lq[PASSES], off_t[PASSES];
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps) {
        const int idx = lane + 32 * ps;
        const int r = 1 + idx / W, q = 1 + idx % W;
        const bool ok = (idx < NP) && (q <= r);
        off_lr[ps] = ok ? r * W1 + r : -1;
        off_lq[ps] = q * W1 + q;
        off_t[ps] = r * W1 + (r - q);
    }
    for (int j = 0; j < m; ++j) {
        double *row = Mb + j * W1;
        const double piv = row[0];
        const double inv = piv > 0.0 ? frcpd(piv) : 0.0;
#pragma unroll
        for (int ps = 0; ps < PASSES; ++ps) {
            if (off_lr[ps] >= 0) row[off_t[ps]] -= row[off_lr[ps]] * row[off_lq[ps]] * inv;
        }
        __syncwarp();
        if (lane == 0) row[0] = inv;
    }
    __syncwarp();
}

// solve M v = r in place (v carries W padding entries in front and behind)
template <int W>
BND void band_solve(const double *Mb, double *v, int m, int lane) {
    constexpr int W1 = W + 1;
    const int r = (lane % W) + 1;                 // lanes >= W idle in the sweeps
    const bool on = lane < W;                     // W <= 32
    for (int j = 0; j < m; ++j) {                 // forward: L t = r  (column sweeps)
        const double t = v[j] * Mb[j * W1];
        if (on) v[j + r] -= Mb[(j + r) * W1 + r] * t;
        __syncwarp();
    }
    for (int j = lane; j < m; j += 32) v[j] *= Mb[j * W1];      // t' = D^-1 t
    __syncwarp();
    for (int i = m - 1; i > 0; --i) {             // backward: L' v = t'
        const double vi = v[i];
        if (on) v[i - r] -= Mb[(i - r) * W1] * Mb[i * W1 + r] * vi;
        __syncwarp();
    }
}

#undef BND
}  // namespace band
