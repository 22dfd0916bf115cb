// emu_dense.cpp -- TEST INFRASTRUCTURE: the tile routines of the dense kernel (dispatches_b200/csrc/dsp_dense.cuh) -- blocked LDL',
// panel sweeps, trailing updates (FMA fallback of the mma) and substitutions -- compiled with g++ on the lock-step SIMT emulator
// (simt_emu.h), the CTA run as one warp, for tests/test_dense_mirror.py.  Never linked into the product.
#include "simt_emu.h"

#include "../../dispatches_b200/csrc/dsp_band.cuh"
#include "../../dispatches_b200/csrc/dsp_dense.cuh"

// M: mp x mp row-major (its lower triangle is read), mp = nt * 64; v: mp.  On exit M holds the unit-lower factor L (L = W D^-1 in the
// off-diagonal tiles), dinv the reciprocal pivots (0 for a non-positive pivot) and v the solution of M v = r.
extern "C" int emu_dense_factor_solve(int nt, double *M, double *v, double *dinv) {
    using namespace dense;
    const int mp = nt * TS;
    std::vector<double> G((size_t)tiles_doubles(nt)), SA(TS * LDS), SB(TS * LDS);
    for (int I = 0; I < nt; ++I)
        for (int J = 0; J <= I; ++J)
            for (int r = 0; r < TS; ++r)
                for (int q = 0; q < TS; ++q) G[(size_t)tile_index(I, J) * TILE + r * TS + q] = M[(size_t)(I * TS + r) * mp + J * TS + q];
    emu::run_warp([&](int lane) {
        factor(G.data(), nt, SA.data(), SB.data(), dinv, 0, 1, lane);
        solve(G.data(), nt, dinv, v, 0, 1, lane);
    });
    for (size_t e = 0; e < (size_t)mp * mp; ++e) M[e] = 0.0;
    for (int I = 0; I < nt; ++I)
        for (int J = 0; J <= I; ++J)
            for (int r = 0; r < TS; ++r)
                for (int q = 0; q < TS; ++q) {
                    const int i = I * TS + r, j = J * TS + q;
                    const double g = G[(size_t)tile_index(I, J) * TILE + r * TS + q];
                    if (j < i) M[(size_t)i * mp + j] = I == J ? g : g * dinv[j];
                    if (j == i) M[(size_t)i * mp + j] = 1.0;
                }
    return 0;
}
