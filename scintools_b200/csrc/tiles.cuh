// Dynspec.cut_dyn on the device: the secondary spectrum and ACF of every tile of a dynamic
// spectrum in one batched pass of the FFT engine (drivers sspec_tiles / acf_tiles in
// dynspec.cu).  This header holds what those drivers add to the engine: the per-tile
// statistics and the load / store functors that map the batch onto the engine's plain row
// and column passes.  Barrier-free apart from warp shuffles, so tests/host_emu can compile it
// for the CPU (SB_HOST_EMU).
//
// Layout.  The parent spectrum dyn [nf][ld] is read in place: tile `tile` (row-major over the
// nfc x ntc grid, tile = ii * ntc + jj) is dyn[ii*fnum + f][jj*tnum + t].  A group of ntile
// consecutive tiles starting at tile0 is transformed at once:
//   rows    : row item r = tl * fnum + f (tl = tile - tile0) -> half spectrum of tile row f;
//   H       : H[f][tl * tp + k], all tiles' half spectra side by side (tp = per-tile pitch),
//             so one column pass over ntile * tp columns transforms every tile;
//   columns : the store functor maps column c back to (tl = c / tp, k = c % tp) and drops
//             the pitch padding k >= kmax.
// Every pass works on one tile's own rows or columns, so nothing (a NaN included) crosses
// from one tile into another.
#pragma once
#ifndef SB_HOST_EMU
#include "common.cuh"
#include "fft_functors.cuh"
#endif

namespace sb {

// sums[4 tl + 0..2] += sum d, sum wt[t] wf[f] d (wt non-null), sum d^2 over the tile's pixels.
// One warp per item (tile, chunk of rpi rows); the caller zeroes sums.
__global__ void __launch_bounds__(256)
tile_stats_kernel(const float* __restrict__ dyn, long ld, int fnum, int tnum, int ntc,
                  int tile0, int ntile, int rpi, const float* __restrict__ wt,
                  const float* __restrict__ wf, double* __restrict__ sums) {
    const int lane = threadIdx.x & 31;
    const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nwarp = ((long)gridDim.x * blockDim.x) >> 5;
    const int chunks = (fnum + rpi - 1) / rpi;
    const long items = (long)ntile * chunks;
    for (long it = warp; it < items; it += nwarp) {
        const int tl = (int)(it / chunks);
        const int f0 = (int)(it - (long)tl * chunks) * rpi;
        const int f1 = f0 + rpi < fnum ? f0 + rpi : fnum;
        const int tile = tile0 + tl, ii = tile / ntc, jj = tile - ii * ntc;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int f = f0; f < f1; ++f) {
            const float* src = dyn + (size_t)(ii * fnum + f) * ld + (size_t)jj * tnum;
            const float fw = wt ? wf[f] : 0.f;
            for (int t = lane; t < tnum; t += 32) {
                const float v = src[t];
                s0 += v;
                if (wt) s1 += (double)(wt[t] * fw) * v;
                s2 += (double)v * v;
            }
        }
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
            atomicAdd(sums + 4 * tl, s0);
            atomicAdd(sums + 4 * tl + 1, s1);
            atomicAdd(sums + 4 * tl + 2, s2);
        }
    }
}

// One thread per tile.  acf_den == 0 (secondary spectrum): cst[tl] = (mu1, mu2) of
// calc_sspec, mu1 = mean(d), mu2 = mean(wt wf (d - mu1)) (0 without a window), narrowed as
// DynRowLoad narrows them.  acf_den > 0 (ACF): cst[tl].x = 1 / (acf_den sum d^2), the factor
// that brings the zero lag of the unnormalised inverse transform (acf_den = PF * PT times
// the tile's sum of squares, by Parseval) to 1.
__global__ void tile_stats_final_kernel(const double* __restrict__ sums, int ntile, double n,
                                        double swt, double swf, int windowed, double acf_den,
                                        float2* __restrict__ cst) {
    const int tl = blockIdx.x * blockDim.x + threadIdx.x;
    if (tl >= ntile) return;
    const double* s = sums + 4 * tl;
    if (acf_den > 0.0) {
        cst[tl] = make_float2((float)(1.0 / (acf_den * s[2])), 0.f);
        return;
    }
    const double mu1 = s[0] / n;
    cst[tl] = make_float2((float)mu1, (float)(windowed ? (s[1] - mu1 * swt * swf) / n : 0.0));
}

// rows: item r = tl * fnum + f -> (x[2n], x[2n+1]) of tile row f, x = (d - mu1) wt wf - mu2
// (cst non-null; the window only when wt is) or the raw d (cst null); zero past tnum
struct TileRowLoad {
    const float* dyn;
    long ld;
    int fnum, tnum, ntc, tile0;
    const float* wt;       // [tnum] or null
    const float* wf;       // [fnum]
    const float2* cst;     // [ntile] (mu1, mu2) or null
    __device__ __forceinline__ int live(int N) const {
        const int l = (tnum + 1) >> 1;
        return l < N ? l : N;
    }
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        const int tl = (int)(row / fnum), f = (int)(row - (long)tl * fnum);
        const int tile = tile0 + tl, ii = tile / ntc, jj = tile - ii * ntc;
        const float* src = dyn + (size_t)(ii * fnum + f) * ld + (size_t)jj * tnum;
        const float2 m = cst ? cst[tl] : make_float2(0.f, 0.f);
        float x[2];
        for (int h = 0; h < 2; ++h) {
            const int t = 2 * n + h;
            float v = 0.f;
            if (t < tnum) {
                v = src[t] - m.x;
                if (wt) v *= wt[t] * wf[f];
                v -= m.y;
            }
            x[h] = v;
        }
        return make_float2(x[0], x[1]);
    }
};
__device__ __forceinline__ int row_load_live(const TileRowLoad& l, int N) { return l.live(N); }

struct TileHalfStore {   // X[k] of row item tl * fnum + f -> H[f][tl * tp + k]
    float2* H;
    long pitch;          // row pitch of H: ntile * tp
    int tp, fnum;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        const long tl = row / fnum, f = row - tl * fnum;
        H[f * pitch + tl * tp + k] = v;
    }
};

// last column pass of the secondary spectrum: column c = tl * tp + k -> SspecStore of tile
// tl (its plane of `plane` floats in the output), k < kmax
struct TileSspecStore {
    SspecStore s;
    int tp, kmax;
    size_t plane;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int tl = c / tp, kk = c - tl * tp;
        if (kk >= kmax) return;
        SspecStore t = s;
        t.sec += (size_t)tl * plane;
        t(y, k, kk, v);
    }
};

// final row pass of the ACF: row item tl * rows + i -> AcfRowLoad / AcfRowStore of tile tl
// (its columns tl * tp + k of Q, its plane of the output, its factor cst[tl].x)
struct TileAcfRowLoad {
    AcfRowLoad a;
    int rows, tp;
    __device__ __forceinline__ float2 operator()(long row, int k) const {
        const long tl = row / rows;
        AcfRowLoad t = a;
        t.Q += tl * tp;
        return t(row - tl * rows, k);
    }
};
struct TileAcfRowStore {
    AcfRowStore s;
    int rows;
    size_t plane;
    const float2* cst;
    __device__ __forceinline__ void operator()(long row, int n, float2 z) const {
        const long tl = row / rows;
        AcfRowStore t = s;
        t.acf += (size_t)tl * plane;
        t.scale = &cst[tl].x;
        t(row - tl * rows, n, z);
    }
};

}  // namespace sb
