// emu_dense_cluster.cpp -- TEST INFRASTRUCTURE: the cluster factorisation and substitutions of the dense cluster kernel
// (dispatches_b200/csrc/dsp_dense.cuh: cluster_column, cluster_panel, cluster_fwd, cluster_bwd) compiled with g++ on the lock-step SIMT
// emulator (simt_emu.h).  The C ranks of a cluster run one after another between the cluster barriers, each as one warp with its own
// staged-tile buffers, sharing G, dinv and v -- valid because inside a phase a rank writes only its own rows and reads only what earlier
// phases finished.  For tests/test_dense_cluster_cpu.py; never linked into the product.
#include "simt_emu.h"

#include "../../dispatches_b200/csrc/dsp_band.cuh"
#include "../../dispatches_b200/csrc/dsp_dense.cuh"

using namespace dense;

static void pack(int nt, const double *M, std::vector<double> &G) {
    const int mp = nt * TS;
    G.assign((size_t)tiles_doubles(nt), 0.0);
    for (int I = 0; I < nt; ++I)
        for (int J = 0; J <= I; ++J)
            for (int r = 0; r < TS; ++r)
                for (int q = 0; q < TS; ++q) G[(size_t)tile_index(I, J) * TILE + r * TS + q] = M[(size_t)(I * TS + r) * mp + J * TS + q];
}

// M: mp x mp row-major (its lower triangle is read), mp = nt * 64; v: mp.  Runs the cluster routines with C ranks; on exit G holds the
// lower tiles of the factor (tiles_doubles(nt) doubles, the workspace layout), dinv the reciprocal pivots and v the solution of M v = r.
extern "C" int emu_dense_cluster_factor_solve(int nt, int C, const double *M, double *v, double *dinv, double *G_out) {
    std::vector<double> G;
    pack(nt, M, G);
    std::vector<std::vector<double>> SB(C), SC(C), SA(C);
    for (int r = 0; r < C; ++r) { SB[r].resize(TS * LDS); SC[r].resize(kGroup * TS * LDS); SA[r].resize(kGroup * TS * LDS); }
    double *g = G.data();
    for (int J = 0; J < nt; ++J) {
        for (int r = 0; r < C; ++r)
            emu::run_warp([&](int lane) { cluster_column(g, nt, J, r, C, SB[r].data(), SC[r].data(), SA[r].data(), dinv, 0, 1, lane); });
        for (int r = 0; r < C; ++r) emu::run_warp([&](int lane) { cluster_panel(g, nt, J, r, C, SA[r].data(), SB[r].data(), 0, 1, lane); });
    }
    for (int K = 0; K < nt; ++K)
        for (int r = 0; r < C; ++r) emu::run_warp([&](int lane) { cluster_fwd(g, nt, K, r, C, dinv, v, 0, 1, lane); });
    for (int K = nt - 1; K >= 0; --K)
        for (int r = 0; r < C; ++r) emu::run_warp([&](int lane) { cluster_bwd(g, nt, K, r, C, dinv, v, 0, 1, lane); });
    memcpy(G_out, g, G.size() * sizeof(double));
    return 0;
}

// the single-CTA routines (factor, solve) on the same input, for the bitwise comparison
extern "C" int emu_dense_single_factor_solve(int nt, const double *M, double *v, double *dinv, double *G_out) {
    std::vector<double> G, SA(TS * LDS), SB(TS * LDS);
    pack(nt, M, G);
    emu::run_warp([&](int lane) {
        factor(G.data(), nt, SA.data(), SB.data(), dinv, 0, 1, lane);
        solve(G.data(), nt, dinv, v, 0, 1, lane);
    });
    memcpy(G_out, G.data(), G.size() * sizeof(double));
    return 0;
}

extern "C" int emu_dense_first_own(int J, int rank, int C) { return first_own(J, rank, C); }
extern "C" int emu_dense_group() { return kGroup; }
extern "C" long long emu_dense_tiles_doubles(int nt) { return tiles_doubles(nt); }
