// emu_band_split.cpp -- TEST INFRASTRUCTURE: the partitioned band factorisation / substitutions of dispatches_b200/csrc/dsp_band_split.cuh
// compiled with g++ on the lock-step SIMT emulator (simt_emu.h) for tests/test_band_split_cpu.py.  Never linked into the product.
#include "simt_emu.h"

#include "../../dispatches_b200/csrc/dsp_band_split.cuh"

// Mb: (W + 1) * Sr * 32 doubles in, the factor out; G: W * Sr * 32 doubles out (the spike); v: Sr * 32 doubles, the right-hand side in,
// the solution out (all in the split layout, Sr = ceil(m / 32))
template <int W>
static void run(int m, double *Mb, double *G, double *v) {
    const int Sr = (m + 31) / 32;
    std::vector<double> E(W * W * 32), X(W * W + W);
    bsplit::Factor<W> F;
    F.Mb = Mb; F.G = G; F.E = E.data(); F.X = X.data(); F.Sr = Sr; F.m = m;
    emu::run_warp([&](int lane) {
        bsplit::split_factor<W>(F, lane);
        bsplit::split_solve<W>(F, v, lane);
    });
}

extern "C" int emu_band_split_factor_solve(int W, int m, double *Mb, double *G, double *v) {
    if (m < 64 * W) return -2;
    switch (W) {
        case 1: run<1>(m, Mb, G, v); return 0;
        case 2: run<2>(m, Mb, G, v); return 0;
        case 4: run<4>(m, Mb, G, v); return 0;
        case 8: run<8>(m, Mb, G, v); return 0;
        case 16: run<16>(m, Mb, G, v); return 0;
        case 32: run<32>(m, Mb, G, v); return 0;
    }
    return -1;
}
