// dsp_dense.cuh -- blocked dense LDL' factorisation and substitutions of the dense IPM kernel (dsp_lp.cu, dsp_ipm_dense_kernel).
//
// One CTA per LP.  M = A D A' (m <= 1024) is padded to mp = nt * TS rows with decoupled unit rows and kept as its lower TS x TS tiles
// in a per-CTA region of the handle's device workspace, tile-major: tile (I, J), I >= J, starts at tile_index(I, J) * TILE, row-major
// with stride TS.  Factorisation: right-looking blocked LDL' over the tiles; every tile it works on is staged into one of two shared
// memory buffers (row stride LDS = TS + 1, so a lane per row is free of bank conflicts):
//   * diagonal tile: unblocked LDL' by one warp with the band kernel's pivot rule (1/d = 0 for a non-positive pivot: the row is
//     decoupled), strictly lower part -> unit-lower L, 1/d -> dinv[];
//   * panel: every tile below it becomes W = L21 D = A21 L11^-T (row sweeps, 4 lanes per row);
//   * trailing update  A(I,J) -= W(I,K) D^-1 W(J,K)'  on the FP64 tensor cores (mma.sync m8n8k4 .f64), an 8-row strip per warp.
// After the factorisation a diagonal tile holds L (strictly lower), an off-diagonal tile W = L D (unscaled, like the band kernel's
// off-diagonal slots), dinv[] the reciprocal pivots.  Substitutions: forward L t = r with D^-1 folded in, backward L' v = t'.
//
// Plain C++ over warp builtins: tests/emu compiles this file with g++ on the SIMT emulator, which runs the CTA as a single warp
// (nwarps = 1, DENSE_SYNC a warp barrier), with an FMA fallback for the mma.  The emulator checks it against numpy.
#pragma once

namespace dense {

#if defined(__CUDA_ARCH__) || defined(__CUDACC__)
#define DNS __device__ __forceinline__
#define DENSE_SYNC() __syncthreads()
#else
#define DNS inline
#define DENSE_SYNC() __syncwarp()
#endif
constexpr unsigned DFULL = 0xffffffffu;
constexpr int TS = 64;             // tile edge
constexpr int LDS = TS + 1;        // row stride of a tile staged in shared memory
constexpr int TILE = TS * TS;      // doubles per tile in the workspace

// workspace layout, shared with the host set-up (dsp_lp.cu)
#if defined(__CUDACC__)
__host__ __device__
#endif
inline int tile_index(int I, int J) { return I * (I + 1) / 2 + J; }
#if defined(__CUDACC__)
__host__ __device__
#endif
inline long long tiles_doubles(int nt) { return (long long)nt * (nt + 1) / 2 * TILE; }

// D = A B + C for one 8x8 block: A 8x4 row-major (lane holds A[lane/4][lane%4]), B 4x8 column-major (lane holds B[lane%4][lane/4]),
// C / D 8x8 (lane holds row lane/4, columns 2 (lane%4) and 2 (lane%4) + 1)
DNS void mma884(double &c0, double &c1, double a, double b, int lane) {
#if defined(__CUDA_ARCH__)
    double d0, d1;
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};"
        : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(c0), "d"(c1));
    c0 = d0; c1 = d1;
#else
    const int g = lane >> 2, t = lane & 3;
    for (int k = 0; k < 4; ++k) {
        const double ak = __shfl_sync(DFULL, a, g * 4 + k);
        const double b0 = __shfl_sync(DFULL, b, (2 * t) * 4 + k);
        const double b1 = __shfl_sync(DFULL, b, (2 * t + 1) * 4 + k);
        c0 = fma(ak, b0, c0);
        c1 = fma(ak, b1, c1);
    }
#endif
}

// unblocked LDL' of a staged diagonal tile S by one warp.  On exit the strictly lower part holds the unit-lower L and dinv[j] = 1/d_j,
// 0 for a non-positive pivot (the band kernel's rule, dsp_band.cuh)
DNS void tile_factor(double *S, double *dinv, int lane) {
    for (int j = 0; j < TS; ++j) {
        const double piv = S[j * LDS + j];
        const double inv = piv > 0.0 ? band::frcpd(piv) : 0.0;
        for (int r = j + 1 + lane; r < TS; r += 32) {
            const double lr = S[r * LDS + j] * inv;
            for (int q = j + 1; q <= r; ++q) S[r * LDS + q] -= lr * S[q * LDS + j];
        }
        if (lane == 0) dinv[j] = inv;
        __syncwarp();
    }
    for (int r = lane; r < TS; r += 32)
        for (int q = 0; q < r; ++q) S[r * LDS + q] *= dinv[q];
    __syncwarp();
}

// rows [row0, row0 + 8) of a staged panel tile B <- B L11^-T (L11: the factored diagonal tile S), one warp: 4 lanes per row, the lane
// owns the columns q = lane mod 4
DNS void tile_panel8(const double *S, double *B, int row0, int lane) {
    double *br = B + (row0 + (lane >> 2)) * LDS;
    const int g = lane & 3;
    for (int j = 0; j < TS - 1; ++j) {
        const double wj = br[j];
        for (int q = g; q < TS; q += 4)
            if (q > j) br[q] -= wj * S[q * LDS + j];
        __syncwarp();
    }
}

// 8-row strip of a trailing update: C[row0 .. row0+8)[:] -= A[row0 .. row0+8)[:] * B'  (A, B staged, stride LDS; C with row stride
// LDC: a workspace tile, or a staged one): 8 column blocks x 16 k-steps of mma m8n8k4, the strip of C in registers
template <int LDC = TS>
DNS void tile_update8(double *C, const double *A, const double *B, int row0, int lane) {
    const int g = lane >> 2, t = lane & 3;
    double *cr = C + (row0 + g) * LDC + 2 * t;
    double acc[16];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) { acc[2 * nb] = cr[nb * 8]; acc[2 * nb + 1] = cr[nb * 8 + 1]; }
    const double *ar = A + (row0 + g) * LDS + t;
    const double *bcol = B + g * LDS + t;
#pragma unroll 4
    for (int k0 = 0; k0 < TS; k0 += 4) {
        const double a = -ar[k0];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) mma884(acc[2 * nb], acc[2 * nb + 1], a, bcol[nb * 8 * LDS + k0], lane);
    }
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) { cr[nb * 8] = acc[2 * nb]; cr[nb * 8 + 1] = acc[2 * nb + 1]; }
}

// staged copies between a workspace tile (stride TS) and a shared-memory buffer (stride LDS), scaled by col[] when given
DNS void stage_in(double *S, const double *G, const double *col, int tid, int nthr) {
    for (int e = tid; e < TILE; e += nthr) S[(e >> 6) * LDS + (e & 63)] = col ? G[e] * col[e & 63] : G[e];
}
DNS void stage_out(double *G, const double *S, int tid, int nthr) {
    for (int e = tid; e < TILE; e += nthr) G[e] = S[(e >> 6) * LDS + (e & 63)];
}

// blocked right-looking LDL' of the nt x nt lower tiles G in place; SA, SB: two staged-tile buffers; dinv [nt * TS]
DNS void factor(double *G, int nt, double *SA, double *SB, double *dinv, int warp, int nwarps, int lane) {
    const int tid = warp * 32 + lane, nthr = nwarps * 32;
    for (int K = 0; K < nt; ++K) {
        double *GKK = G + (long long)tile_index(K, K) * TILE;
        DENSE_SYNC();
        stage_in(SA, GKK, nullptr, tid, nthr);
        DENSE_SYNC();
        if (warp == 0) tile_factor(SA, dinv + K * TS, lane);
        DENSE_SYNC();
        stage_out(GKK, SA, tid, nthr);
        for (int I = K + 1; I < nt; ++I) {                     // panel
            double *GIK = G + (long long)tile_index(I, K) * TILE;
            DENSE_SYNC();
            stage_in(SB, GIK, nullptr, tid, nthr);
            DENSE_SYNC();
            for (int s = warp; s < TS / 8; s += nwarps) tile_panel8(SA, SB, s * 8, lane);
            DENSE_SYNC();
            stage_out(GIK, SB, tid, nthr);
        }
        const double *dK = dinv + K * TS;
        for (int J = K + 1; J < nt; ++J) {                     // trailing update, a block column at a time
            DENSE_SYNC();
            stage_in(SB, G + (long long)tile_index(J, K) * TILE, nullptr, tid, nthr);
            for (int I = J; I < nt; ++I) {
                DENSE_SYNC();
                stage_in(SA, G + (long long)tile_index(I, K) * TILE, dK, tid, nthr);
                DENSE_SYNC();
                for (int s = warp; s < TS / 8; s += nwarps) tile_update8(G + (long long)tile_index(I, J) * TILE, SA, SB, s * 8, lane);
            }
        }
    }
    DENSE_SYNC();
}

// forward on a diagonal tile: L t = v, then v <- dinv t
DNS void tile_fwd(const double *G, const double *dinv, double *v, int lane) {
    for (int j = 0; j < TS - 1; ++j) {
        const double vj = v[j];
        for (int q = lane; q < TS; q += 32)
            if (q > j) v[q] -= G[q * TS + j] * vj;
        __syncwarp();
    }
    for (int q = lane; q < TS; q += 32) v[q] *= dinv[q];
    __syncwarp();
}
// backward on a diagonal tile: L' v = v in place
DNS void tile_bwd(const double *G, double *v, int lane) {
    for (int j = TS - 1; j > 0; --j) {
        const double vj = v[j];
        for (int q = lane; q < j; q += 32) v[q] -= G[j * TS + q] * vj;
        __syncwarp();
    }
}
// v -= W u  (an off-diagonal tile, lane per row)
DNS void tile_gemv_sub(const double *W, const double *u, double *v, int lane) {
    for (int r = lane; r < TS; r += 32) {
        double acc = 0.0;
        for (int k = 0; k < TS; ++k) acc = fma(W[r * TS + k], u[k], acc);
        v[r] -= acc;
    }
    __syncwarp();
}
// v -= dinv (W' u)  (an off-diagonal tile, lane per column: L = W D^-1)
DNS void tile_gemvt_sub(const double *W, const double *u, const double *dinv, double *v, int lane) {
    for (int c = lane; c < TS; c += 32) {
        double acc = 0.0;
        for (int r = 0; r < TS; ++r) acc = fma(W[r * TS + c], u[r], acc);
        v[c] -= dinv[c] * acc;
    }
    __syncwarp();
}

// M v = r in place with the factor of `factor` (v: nt * TS entries, zero in the padding rows)
DNS void solve(const double *G, int nt, const double *dinv, double *v, int warp, int nwarps, int lane) {
    for (int K = 0; K < nt; ++K) {
        if (warp == 0) tile_fwd(G + (long long)tile_index(K, K) * TILE, dinv + K * TS, v + K * TS, lane);
        DENSE_SYNC();
        for (int I = K + 1 + warp; I < nt; I += nwarps) tile_gemv_sub(G + (long long)tile_index(I, K) * TILE, v + K * TS, v + I * TS, lane);
        DENSE_SYNC();
    }
    for (int K = nt - 1; K >= 0; --K) {
        if (warp == 0) tile_bwd(G + (long long)tile_index(K, K) * TILE, v + K * TS, lane);
        DENSE_SYNC();
        for (int J = warp; J < K; J += nwarps)
            tile_gemvt_sub(G + (long long)tile_index(K, J) * TILE, v + K * TS, dinv + J * TS, v + J * TS, lane);
        DENSE_SYNC();
    }
}

// ---- one LP per thread-block cluster (dsp_ipm_dense_cluster_kernel, m <= 4096)
// The C ranks (CTAs) of a cluster share the lower tiles G, dinv and the substitution vector v of their LP.  Tile row I belongs to
// rank I mod C.  The factorisation and the substitutions run in phases separated by cluster barriers.  Invariant: inside a phase a
// rank writes only tiles and entries of v of its own rows (and the owner of a diagonal block its dinv block), and reads only what
// earlier phases finished.  So the ranks may as well run one after another between the barriers (tests/emu does), and the result does
// not depend on C.  Every tile also sees the operations of `factor` / `solve` in the same order, so the factor and the solution are
// bitwise those of the single-CTA routines.
constexpr int kGroup = 2;          // target tiles a rank accumulates together

// the first tile row I >= J that rank `rank` of C owns (nt or more: none)
DNS int first_own(int J, int rank, int C) { return J + ((rank - J % C) % C + C) % C; }

// factorisation phase 1 of block column J on rank `rank`: each of its target tiles (I, J), I >= J, becomes
// A(I,J) - sum_{K<J} W(I,K) D_K^-1 W(J,K)', accumulated over K in ascending order in a staged buffer and written back once (left-looking,
// Crout order); the owner of (J, J) then factors it into L_JJ and dinv_J.  W(J,K) is staged once per group of kGroup target tiles.
// SB: one staged-tile buffer; SC, SA: kGroup buffers each, TS * LDS doubles apart
DNS void cluster_column(double *G, int nt, int J, int rank, int C, double *SB, double *SC, double *SA, double *dinv, int warp, int nwarps,
                        int lane) {
    const int tid = warp * 32 + lane, nthr = nwarps * 32;
    for (int I0 = first_own(J, rank, C); I0 < nt; I0 += C * kGroup) {
        const int left = (nt - 1 - I0) / C + 1, ng = left < kGroup ? left : kGroup;
        DENSE_SYNC();
        for (int g = 0; g < ng; ++g) stage_in(SC + g * TS * LDS, G + (long long)tile_index(I0 + g * C, J) * TILE, nullptr, tid, nthr);
        for (int K = 0; K < J; ++K) {
            DENSE_SYNC();
            stage_in(SB, G + (long long)tile_index(J, K) * TILE, nullptr, tid, nthr);
            for (int g = 0; g < ng; ++g)
                stage_in(SA + g * TS * LDS, G + (long long)tile_index(I0 + g * C, K) * TILE, dinv + K * TS, tid, nthr);
            DENSE_SYNC();
            for (int g = 0; g < ng; ++g)
                for (int s = warp; s < TS / 8; s += nwarps) tile_update8<LDS>(SC + g * TS * LDS, SA + g * TS * LDS, SB, s * 8, lane);
        }
        DENSE_SYNC();
        if (I0 == J && warp == 0) tile_factor(SC, dinv + J * TS, lane);
        DENSE_SYNC();
        for (int g = 0; g < ng; ++g) stage_out(G + (long long)tile_index(I0 + g * C, J) * TILE, SC + g * TS * LDS, tid, nthr);
    }
}

// factorisation phase 2 of block column J on rank `rank`: its tiles below the diagonal become W = A L_JJ^-T (L_JJ from phase 1)
DNS void cluster_panel(double *G, int nt, int J, int rank, int C, double *SA, double *SB, int warp, int nwarps, int lane) {
    const int tid = warp * 32 + lane, nthr = nwarps * 32;
    const int I0 = first_own(J + 1, rank, C);
    if (I0 >= nt) return;
    DENSE_SYNC();
    stage_in(SA, G + (long long)tile_index(J, J) * TILE, nullptr, tid, nthr);
    for (int I = I0; I < nt; I += C) {
        double *GIJ = G + (long long)tile_index(I, J) * TILE;
        DENSE_SYNC();
        stage_in(SB, GIJ, nullptr, tid, nthr);
        DENSE_SYNC();
        for (int s = warp; s < TS / 8; s += nwarps) tile_panel8(SA, SB, s * 8, lane);
        DENSE_SYNC();
        stage_out(GIJ, SB, tid, nthr);
    }
}

// forward substitution phase K (0 <= K < nt) on rank `rank`: its rows I >= K take the update of block K-1, then the owner of row K
// finishes it (L t = v, v <- dinv t, as in `solve`)
DNS void cluster_fwd(const double *G, int nt, int K, int rank, int C, const double *dinv, double *v, int warp, int nwarps, int lane) {
    if (K > 0) {
        int c = 0;
        for (int I = first_own(K, rank, C); I < nt; I += C, ++c)
            if (c % nwarps == warp) tile_gemv_sub(G + (long long)tile_index(I, K - 1) * TILE, v + (K - 1) * TS, v + I * TS, lane);
        DENSE_SYNC();
    }
    if (K % C == rank) {
        if (warp == 0) tile_fwd(G + (long long)tile_index(K, K) * TILE, dinv + K * TS, v + K * TS, lane);
        DENSE_SYNC();
    }
}

// backward substitution phase K (nt > K >= 0) on rank `rank`: its rows J <= K take the update of block K+1, then the owner of row K
// finishes it (L' v = v)
DNS void cluster_bwd(const double *G, int nt, int K, int rank, int C, const double *dinv, double *v, int warp, int nwarps, int lane) {
    if (K + 1 < nt) {
        int c = 0;
        for (int J = rank; J <= K; J += C, ++c)
            if (c % nwarps == warp)
                tile_gemvt_sub(G + (long long)tile_index(K + 1, J) * TILE, v + (K + 1) * TS, dinv + J * TS, v + J * TS, lane);
        DENSE_SYNC();
    }
    if (K % C == rank) {
        if (warp == 0) tile_bwd(G + (long long)tile_index(K, K) * TILE, v + K * TS, lane);
        DENSE_SYNC();
    }
}

#undef DNS
#undef DENSE_SYNC
}  // namespace dense
