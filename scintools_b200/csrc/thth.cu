// theta-theta curvature sweep: crop mask, gather (nearest-bin remap of the
// conjugate spectrum onto the theta-theta grid), Hermitian fill and the
// dominant-eigenvalue solve.  General path: the per-eta matrix lives in a
// global scratch slab (L2 / HBM), one CTA per eta runs a Lanczos iteration.
//
// Reference behaviour reproduced (scintools/ththmod.py):
//   thth_map :56-116, thth_redmap :119-173, Eval_calc :371-401,
//   eta loop of single_search :789-799 (failure -> NaN).
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../include/scint_b200.h"   // SB_ETA_* status bits, tests/host_emu too
#include "drivers.cuh"
#include "lanczos.cuh"
#include "thth.cuh"

namespace sb {

// --------------------------------------------------------------------------
// crop mask + compaction: th_pnts of thth_redmap (ththmod.py:153-156)
// one warp per eta
// --------------------------------------------------------------------------
// one warp: the kept centres of geometry g at curvature eta into out[0 .. *nred)
__device__ __forceinline__ void thth_crop_warp(const ThthGeom& g, double eta,
                                               int* __restrict__ out, int* __restrict__ nred) {
    int lane = threadIdx.x;
    int base = 0;
    for (int k0 = 0; k0 < g.n; k0 += 32) {
        int k = k0 + lane;
        bool keep = false;
        if (k < g.n) {
            double t = g.th[k];
            keep = (__dmul_rn(__dmul_rn(t, t), eta) < g.tau_absmax) &&
                   (fabs(t) < g.fd_half);
        }
        unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) out[base + __popc(m & ((1u << lane) - 1u))] = k;
        base += __popc(m);
    }
    if (lane == 0) *nred = base;
}

__global__ void thth_prep_kernel(ThthGeom g, const double* __restrict__ etas,
                                 int neta, int ld, int* __restrict__ idx,
                                 int* __restrict__ nred) {
    int e = blockIdx.x;
    if (e >= neta) return;
    thth_crop_warp(g, etas[e], idx + (size_t)e * ld, nred + e);
}

// the same for a table of geometries, one per item (sb_asymmetry_batch: one per chunk)
__global__ void thth_prep_table_kernel(const ThthGeom* __restrict__ geoms,
                                       const double* __restrict__ etas, int ld,
                                       int* __restrict__ idx, int* __restrict__ nred) {
    const int e = blockIdx.x;
    const ThthGeom g = geoms[e];
    thth_crop_warp(g, etas[e], idx + (size_t)e * ld, nred + e);
}

// --------------------------------------------------------------------------
// rare path: would numpy raise IndexError anywhere in the full N x N map?
// (fd_inv < -nfd on a point that passes the pnts mask, ththmod.py:100-104)
// --------------------------------------------------------------------------
__device__ __forceinline__ void thth_indexerr_body(const ThthGeom& g, double eta,
                                                   int* __restrict__ status) {
    long long total = (long long)g.n * g.n;
    bool bad = false;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
         p < total; p += (long long)gridDim.x * blockDim.x) {
        int i = (int)(p / g.n), j = (int)(p % g.n);
        ThthPoint pt = thth_point(g, eta, g.th[j], g.th[i]);
        bad |= pt.index_error;
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0)
        atomicOr(status, SB_ETA_INDEX_ERROR);
}

__global__ void thth_indexerr_kernel(ThthGeom g, const double* __restrict__ etas,
                                     int* __restrict__ status) {
    int e = blockIdx.y;
    thth_indexerr_body(g, etas[e], status + e);
}

// per item e0 + blockIdx.y of a geometry table
__global__ void thth_indexerr_table_kernel(const ThthGeom* __restrict__ geoms,
                                           const double* __restrict__ etas, int e0,
                                           int* __restrict__ status) {
    const int e = e0 + blockIdx.y;
    const ThthGeom g = geoms[e];
    thth_indexerr_body(g, etas[e], status + e);
}

// --------------------------------------------------------------------------
// build the cropped theta-theta matrix for a batch of etas: STRICT UPPER
// triangle only (the matrix is Hermitian with zero diagonal; the eigen kernel
// uses every stored element twice).  M[e] is [ld][ld] float2; inside the active
// 32x32 tiles columns >= nred and the diagonal are zero, the lower triangle is not
// touched.  Two kernels, one per gather source (thth_gather_source chooses):
// thth_build_kernel reads the spectrum itself, thth_build_copy_kernel the compact copy.
// --------------------------------------------------------------------------
#define SB_BUILD_EB 8      // thth_build_kernel: curvatures per CTA
#define SB_COPY_EB 32      // thth_build_copy_kernel: curvatures per CTA, one per lane
#define SB_COPY_RB 4       // thth_build_copy_kernel: rows of a 32 x 32 tile per band

// Diagnostic builds for profiles/probe_build_split.py, never the shipped library:
// 1 = stores only (every gathered value is a constant), 2 = gathers only (the stores sit
// behind a predicate the compiler cannot prove false and that is never true).
#ifndef SB_BUILD_PROBE
#define SB_BUILD_PROBE 0
#endif

// fp32 pair -> fp16 pair (re | im << 16, round to nearest even) for eig_half.cu
__device__ __forceinline__ unsigned pack_f16x2(float2 v) {
#ifdef SB_HOST_EMU
    const __half2 h = __floats2half2_rn(v.x, v.y);
    return (unsigned)h.x | ((unsigned)h.y << 16);
#else
    unsigned r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(v.y), "f"(v.x));   // hi = first source
    return r;
#endif
}

// max |re|, |im| over the part of the conjugate spectrum the gather can touch
// (rows x ncols of a [rows][pitch] array): the bound that keeps the scaled fp16
// triangle finite.  out: non-negative float as uint bits (atomicMax), pre-zeroed.
// VEC: float4 loads of two complex columns, for a 16-byte aligned cs with an even pitch
// (every row 16-byte aligned); otherwise one float2 per column (an odd pitch starts every
// other row 8 bytes off a 16-byte boundary).
template <bool VEC>
__global__ void cs_absmax_kernel(const float2* __restrict__ cs, long long rows, long long ncols,
                                 long long pitch, unsigned* __restrict__ out) {
    float m = 0.f;
    const long long per_row = VEC ? ncols >> 1 : ncols;
    const long long total = rows * per_row;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / per_row, c = i - r * per_row;
        if (VEC) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(cs + r * pitch) + c);
            m = fmaxf(fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), fmaxf(fabsf(q.z), fabsf(q.w))), m);
        } else {
            const float2 q = __ldg(cs + r * pitch + c);
            m = fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), m);
        }
    }
    if (VEC && (ncols & 1)) {                        // odd tail column
        for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows;
             r += (long long)gridDim.x * blockDim.x) {
            const float2 q = __ldg(cs + r * pitch + ncols - 1);
            m = fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), m);
        }
    }
    if (!(m == m)) m = 3.0e38f;                      // NaN in the CS: treat as huge
    m = fminf(m, 3.0e38f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

// Element of a valid pair (col >= 0) as thth_map stores it: the gathered value (hit: tau_inv
// inside the spectrum, otherwise zero) conjugated in the mirrored half, |.| for the
// incoherent map, times the Jacobian wf = sqrt|2 eta (th2 - th1)| (ththmod.py:104-107), with
// nan_to_num.
__device__ __forceinline__ float2 thth_element(float2 val, bool hit, bool conj, int coherent,
                                               float wf) {
    float2 v = make_float2(0.f, 0.f);
    if (hit) {
        v = val;
        if (conj) v.y = -v.y;
        if (!coherent) v = make_float2(hypotf(v.x, v.y), 0.f);
    }
    v.x *= wf;
    v.y *= wf;
    if (!(fabsf(v.x) <= 3.402823466e+38f) || !(fabsf(v.y) <= 3.402823466e+38f)) {
        v.x = nan_to_num(v.x);
        v.y = nan_to_num(v.y);
    }
    return v;
}

// One warp: row la (of 32) of a tile of the fp16 copy Mw that eig_half.cu iterates on, lane =
// column holding element v (low: below the diagonal, stored as zero), scaled by the power of
// two hscale; woff: word offset of the lane's column group in its block row, i.e.
// ((2 ta + (la >> 4)) * ld / 8 + b / 8) * 128 + (la & 15) * 8 for row 32 ta + la, column b.
// Block layout of eig_half.cu's tensor-core mat-vec: 512-byte blocks of 16 rows x 8 columns,
// block (I, G) at ((I * ld / 8 + G) * 512) bytes, a block row = [re x 8 | im x 8] (32 bytes):
// the 8 lanes of a column group trade halves so that lane i stores 4-byte word i of it -- one
// store instruction, four full 32-byte sectors per warp (2-byte stores would be slower).
// Elements on / below the diagonal of a diagonal block are zeros (the MMA has no masks);
// 16 x 16 sub-blocks entirely below the diagonal are never read.
__device__ __forceinline__ void thth_store_f16_row(unsigned* __restrict__ Mw, unsigned woff, bool diag,
                                                   int la, float2 v, bool low, float hscale) {
    const int lane = threadIdx.x & 31;
    const unsigned h = low ? 0u : pack_f16x2(make_float2(v.x * hscale, v.y * hscale));
    const int i8 = lane & 7, s0 = (lane & ~7) + 2 * (i8 & 3);
    const unsigned ha = __shfl_sync(0xffffffffu, h, s0);
    const unsigned hb = __shfl_sync(0xffffffffu, h, s0 + 1);
    const unsigned word = i8 < 4 ? ((ha & 0xffffu) | (hb << 16)) : ((ha >> 16) | (hb & 0xffff0000u));
    if (!(diag && (lane >> 4) < (la >> 4)) && (SB_BUILD_PROBE != 2 || woff == ~0u)) {
        // the two 16-byte halves of a block row are stored swapped in rows 4-7 and 12-15: a
        // LINEAR copy of the block into shared memory is then conflict free for both ldmatrix
        // forms (eig_half.cu), so a bulk copy can fetch it
        const unsigned swz = (unsigned)(((la & 15) >> 2) & 1) << 2;
        Mw[woff + ((unsigned)i8 ^ swz)] = word;
    }
}

// Per-curvature power of two of the fp16 copy: the one that puts absmax * max Jacobian of
// this curvature just below 2^15 (absmax: device scalar from cs_absmax_kernel, span: max
// |theta2 - theta1|); 2^floor(log2(2^15 / bound)) is the exponent field of the quotient.
__device__ __forceinline__ float thth_hscale(double eta, const unsigned* __restrict__ absmax, float span) {
    const float seta = sqrtf((float)(2.0 * eta));
    const float bound = __uint_as_float(*absmax) * seta * sqrtf(span);
    float hs = 1.f;
    if (bound > 0.f && bound < 3.0e38f) {
        const float q = 32768.f / bound;
        hs = q >= 1.1754944e-38f ? __uint_as_float(__float_as_uint(q) & 0x7f800000u) : 1.1754944e-38f;
    }
    return hs;
}

// Gather from the spectrum itself (thth_build_kernel): grid = (groups of SB_BUILD_EB etas,
// tile pairs), block = 32 x 8, lane = column of the tile.  PACK == 0: the fp32 triangle
// only; PACK == 2: also the fp16 copy (thth_store_f16_row).
//
// Everything of thth_map's index math that does not depend on eta is computed
// once per (row, column) pair and kept in registers while the CTA walks its
// SB_BUILD_EB curvatures: d = theta1^2 - theta2^2, fd_inv with its Hermitian
// half-plane column / conjugation flag, sqrt|theta2 - theta1|.  Per curvature
// only tau_inv = floor((eta d - tau0 + dtau/2) / dtau) (same fp64 operations in
// the same order as thth_point, so the bins stay bit-exact), one gather and the
// Jacobian remain.  The cached pair is re-derived whenever the crop of the next
// curvature moves the pair (idx differs).
// ROWS = 4 rows of the tile per thread (block = 32 x 8 threads).  Per curvature the
// body runs in three phases -- (1) tau_inv and the offset of every row, (2) ALL the
// gathers back to back, (3) Jacobian, clean-up, stores -- so that ROWS independent
// gathers are in flight per thread.  Every gather costs a DRAM sector of its own: the
// curvatures of a pair walk down a spectrum column, rows apart.
// Three CTAs per SM (80 registers; 40-44 bytes of spill stores per thread in the PACK == 2
// instances on sm_90).  Measured on 1024 curvatures of an irregular 512-edge grid (H100 SXM,
// 700 W power limit, thth_build per launch, alternated in one run with the variant): 2.38 ms;
// 2.68-2.90 ms with the lane-per-curvature structure of thth_build_copy_kernel, whose 32
// lanes then read 32 spectrum rows, each a DRAM sector of its own, per load instruction.
// An earlier run measured four CTAs per SM at 2.41 against 2.23 ms.
template <int PACK, typename OFF>
__global__ void __launch_bounds__(256, 3)
thth_build_kernel(ThthGeom g, const double* __restrict__ etas, int eta0, int nbatch,
                  int ld, const int* __restrict__ idx,
                  const int* __restrict__ nred, float2* __restrict__ M,
                  unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span) {
    // eta is the FAST grid index: CTAs resident at the same time work on the
    // same 32x32 tile for neighbouring curvatures
    // pair index -> (ta <= tb)
    constexpr int ROWS = 4, TY = 32 / ROWS;
    int p = blockIdx.y, ta = 0;
    const int T = ld / 32;
    while (p >= T - ta) { p -= T - ta; ++ta; }
    const int tb = ta + p;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int b = tb * 32 + tx;
    const double ntau_d = (double)g.ntau;
    // cached eta-independent state of this thread's column and its ROWS rows
    int cj = -2;
    double thj = 0.0;
    int ci[ROWS];
    double dk[ROWS];
    int col[ROWS];          // CS column to gather; < 0: never a valid point
    unsigned conj = 0u;     // bit k: the point lies in the mirrored (fd < 0) half
    float wk[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) { ci[k] = -2; dk[k] = 0.0; col[k] = -1; wk[k] = 0.f; }
    const int e_end = min(nbatch, (int)(blockIdx.x + 1) * SB_BUILD_EB);
    // per-curvature power-of-two scale of the fp16 copy, once per CTA
    SB_SHARED float s_hscale[SB_BUILD_EB];
    if (PACK != 0) {
        const int lin = ty * 32 + tx;
        if (lin < SB_BUILD_EB) {
            const int e = blockIdx.x * SB_BUILD_EB + lin;
            s_hscale[lin] = e < e_end ? thth_hscale(etas[eta0 + e], absmax, span) : 1.f;
        }
        __syncthreads();
    }
    // eta-independent store offsets: fp32 element (row a0 + TY k, column b) and, PACK == 2,
    // the 4-byte word of the fp16 block row this lane stores (thth_store_f16_row)
    const unsigned foff0 = (unsigned)(ta * 32 + ty) * (unsigned)ld + (unsigned)b;
    const unsigned frow = (unsigned)TY * (unsigned)ld;
    const unsigned woff0 = ((unsigned)(2 * ta) * (unsigned)(ld >> 3) + (unsigned)(b >> 3)) * 128u +
                           (unsigned)ty * 8u;
    for (int e = blockIdx.x * SB_BUILD_EB; e < e_end; ++e) {
        const int n = nred[eta0 + e];
        if (tb * 32 >= n) continue;  // never read by the eigen kernel
        const double eta = etas[eta0 + e];
        const int* id = idx + (size_t)(eta0 + e) * ld;
        const int j = b < n ? id[b] : -1;
        if (j != cj) {
            cj = j;
            thj = j >= 0 ? g.th[j] : 0.0;
#pragma unroll
            for (int k = 0; k < ROWS; ++k) ci[k] = -2;
        }
        const float seta = sqrtf((float)(2.0 * eta));
        float2* Me = M + (size_t)e * ld * ld;
        // power of two: |element| * hscale < 2^15
        const float hscale = PACK != 0 ? s_hscale[e - blockIdx.x * SB_BUILD_EB] : 1.f;
        // ---- phase 1: offsets
        OFF off[ROWS];          // element offset into the CS (OFF = unsigned when it fits)
        unsigned hit = 0u;
#pragma unroll
        for (int k = 0; k < ROWS; ++k) {
            const int la = ty + TY * k;
            off[k] = 0;
            if (ta == tb && tx < la) continue;      // lower triangle: not stored
            const int a = ta * 32 + la;
            const int i = a < n ? id[a] : -1;
            if (i != ci[k]) {
                ci[k] = i;
                col[k] = -1;
                conj &= ~(1u << k);
                wk[k] = 0.f;
                dk[k] = 0.0;
                if (i >= 0 && j > i && i + j != g.n - 1) {
                    // th1 = theta of the column, th2 = theta of the row (ththmod.py:86-87)
                    const double th1 = thj, th2 = g.th[i];
                    dk[k] = __dsub_rn(__dmul_rn(th1, th1), __dmul_rn(th2, th2));
                    wk[k] = sqrtf((float)fabs(th2 - th1));
                    bool mirrored;
                    col[k] = thth_pair_column(g, th1, th2, &mirrored);
                    if (mirrored) conj |= 1u << k;
                }
            }
            if (col[k] >= 0) {
                const double aa = __dadd_rn(__dsub_rn(__dmul_rn(eta, dk[k]), g.tau0), g.half_dtau);
                const double tqd = floor_div_fast(aa, g.dtau, g.inv_dtau);
                if (tqd > 0.0 && tqd < ntau_d) {            // tau_inv > 0 and < ntau (ththmod.py:100)
                    const int tq = (int)tqd;
                    const int r = (conj >> k) & 1u ? (int)g.ntau - tq : tq;
                    off[k] = (OFF)r * (OFF)g.cs_pitch + (OFF)col[k];
                    hit |= 1u << k;
                }
            }
        }
        // ---- phase 2: the gathers, all in flight together (a miss reads element 0, ignored)
        float2 val[ROWS];
#pragma unroll
        for (int k = 0; k < ROWS; ++k) val[k] = SB_BUILD_PROBE == 1 ? make_float2(1.f, 0.f) : __ldg(g.cs + off[k]);
        // ---- phase 3
#pragma unroll
        for (int k = 0; k < ROWS; ++k) {
            const int la = ty + TY * k;
            const bool low = ta == tb && tx < la;       // below the diagonal: fp32 copy not stored
            float2 v = make_float2(0.f, 0.f);
            if (!low) {
                if (col[k] >= 0)
                    v = thth_element(val[k], (hit >> k) & 1u, (conj >> k) & 1u, g.coherent, seta * wk[k]);
                if (SB_BUILD_PROBE != 2 || eta0 < 0) Me[foff0 + (unsigned)k * frow] = v;
            }
            if (PACK == 2)
                thth_store_f16_row(Mb + (size_t)e * ld * ld, woff0 + (unsigned)(la >> 4) * (unsigned)(ld >> 3) * 128u +
                                   (unsigned)((la & 15) - ty) * 8u, ta == tb, la, v, low, hscale);
        }
    }
}

// Everything of thth_map's index math that does not depend on eta, for the pair of row
// centre i and column centre j (th1 = theta of the column, th2 = theta of the row,
// ththmod.py:86-87): d = theta1^2 - theta2^2, the slot in the copy of the spectrum column
// of fd_inv with the Hermitian half-plane conjugation flag, and sqrt|theta2 - theta1|.
// col < 0: the pair is never a valid point (i or j cropped, on / below the diagonal, on the
// anti-diagonal, outside the fd axis, or a column the copy does not hold -- then the error
// word is raised and no address is formed from it).
struct ThthPair {
    double d;
    int col;
    float w;
    bool conj;
};

__device__ __forceinline__ ThthPair thth_pair_state(const ThthGeom& g, int i, int j,
                                                    const ThthCopy& copy) {
    ThthPair s{0.0, -1, 0.f, false};
    if (i >= 0 && j > i && i + j != g.n - 1) {
        const double th1 = g.th[j], th2 = g.th[i];
        s.d = __dsub_rn(__dmul_rn(th1, th1), __dmul_rn(th2, th2));
        s.w = sqrtf((float)fabs(th2 - th1));
        int c = thth_pair_column(g, th1, th2, &s.conj);
        if (c >= 0) {
            c = copy.slot_of_col[c];
            if (c < 0) atomicOr(copy.err, 1);
        }
        s.col = c;
    }
    return s;
}

// Gather from the compact copy of the spectrum columns the grid reaches (ThthCopy,
// thth.cuh), delay axis contiguous.  grid = (groups of SB_COPY_EB = 32 etas, tile pairs),
// block = 32 x 8; lane l of every warp works on curvature e0 + l, and a CTA whose group
// starts past the batch returns at once.
// * The crop of the 32 curvatures (idx rows, -1 past nred) for the tile's rows and columns
//   is staged in shared memory once per CTA.  The pair state (ThthPair) of every element is
//   computed once, by one thread, for the crop of the first curvature that has the tile (the
//   reference); a lane whose own crop puts other centres on the element's row or column (bit
//   masks per lane, made once) computes its own.  At the benchmark's sizes every curvature
//   of a group has the same crop.  The states of the next band are computed while the
//   current one is stored (two buffers).
// * Gathers, per band of SB_COPY_RB rows: a warp walks elements, its 32 lanes gather the
//   element for 32 neighbouring curvatures, whose delay bins are close: on the benchmark's
//   grid one load instruction touches 15 distinct 32-byte sectors of the copy on average
//   (counted on the host from its axes) instead of 32, one per lane, when the lanes ran
//   over columns.  Per lane only tau_inv = floor((eta d - tau0 + dtau/2) / dtau)
//   remains (the same fp64 operations in the same order as thth_point, so the bins stay
//   bit-exact).  K = 2 elements per step (offsets, both gathers, then the elements) into a
//   shared tile [curvature][element].
// * Stores: per curvature and row, a warp writes the 32 columns of the fp32 triangle (256
//   coalesced bytes) and, PACK == 2, the row of the fp16 blocks (thth_store_f16_row).
// Four CTAs per SM: 64 registers, no spills, 47 KB of static shared memory each.  Measured on
// the headline sweep (H100 SXM, 700 W power limit, thth_build per 1024-eta launch, the 0.24
// ms copy included; variants built from one source and alternated with the previous kernel,
// 1.72-1.76 ms, in two runs): 1.35-1.37 ms; 1.45-1.47 ms with three CTAs per SM and K = 4;
// 1.63 ms with K = 8 (spills); 1.58 ms with one band per CTA, no band loop; 1.85-1.98 ms
// with 128-thread CTAs of two-row bands.  The lane-per-column kernel before it took 1.76 ms,
// and 1.78-1.84 ms with streaming stores of the triangles, an L2 evict-last policy on the
// gathers, the tile pairs ordered by diagonal, or four CTAs per SM.
template <int PACK, typename OFF>
__global__ void __launch_bounds__(256, 4)
thth_build_copy_kernel(ThthGeom g, const double* __restrict__ etas, int eta0, int nbatch,
                       int ld, const int* __restrict__ idx,
                       const int* __restrict__ nred, float2* __restrict__ M,
                       unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span,
                       ThthCopy copy) {
    constexpr int EB = SB_COPY_EB, RB = SB_COPY_RB, NEL = RB * 32, NW = 8, K = 2;
    static_assert(EB == 32 && NEL % (NW * K) == 0 && NEL + 32 <= NW * 32,
                  "one curvature per lane, whole steps, a spare warp for the masks");
    // pair index -> (ta <= tb)
    int p = blockIdx.y, ta = 0;
    const int T = ld / 32;
    while (p >= T - ta) { p -= T - ta; ++ta; }
    const int tb = ta + p;
    const bool diag = ta == tb;
    const int lane = threadIdx.x, warp = threadIdx.y, tid = warp * 32 + lane;
    const int e0 = blockIdx.x * EB, ne = min(EB, nbatch - e0);

    SB_SHARED int s_i[EB][33];                   // row centres of each curvature, -1: none
    SB_SHARED int s_j[EB][33];                   // column centres
    SB_SHARED float s_hscale[EB];
    SB_SHARED unsigned s_act;                    // bit l: curvature e0 + l has this tile
    SB_SHARED unsigned s_mi[EB], s_mj[EB];       // bit r / c: same row / column centre as the reference
    SB_SHARED ThthPair s_ref[2][NEL];            // pair states of a band under the reference crop
    SB_SHARED float2 s_v[EB][NEL + 1];           // gathered elements (+1: lanes on different banks)

    for (int t = tid; t < EB * 64; t += NW * 32) {
        const int l = t >> 6, c = t & 63;
        int v = -1;
        if (l < ne) {
            const int x = c < 32 ? tb * 32 + c : ta * 32 + (c - 32);
            if (x < nred[eta0 + e0 + l]) v = idx[(size_t)(eta0 + e0 + l) * ld + x];
        }
        if (c < 32) s_j[l][c] = v;
        else s_i[l][c - 32] = v;
    }
    if (warp == 0) {
        bool act = false;
        float hs = 1.f;
        if (lane < ne) {
            const int e = eta0 + e0 + lane;
            act = tb * 32 < nred[e];                 // otherwise never read by the eigen kernel
            if (PACK != 0) hs = thth_hscale(etas[e], absmax, span);
        }
        s_hscale[lane] = hs;
        const unsigned m = __ballot_sync(0xffffffffu, act);
        if (lane == 0) s_act = m;
    }
    __syncthreads();
    const unsigned act = s_act;
    if (act == 0u) return;
    const int ref = __ffs(act) - 1;
    // pair states of band `band` under the reference crop, one element per thread tid < NEL
    auto ref_states = [&](int band, ThthPair* out) {
        const int r = band * RB + (tid >> 5), c = tid & 31;
        out[tid] = diag && c < r ? ThthPair{0.0, -1, 0.f, false}
                                 : thth_pair_state(g, s_i[ref][r], s_j[ref][c], copy);
    };
    if (tid < NEL) {
        ref_states(0, s_ref[0]);
    } else if (tid < NEL + 32) {
        const int l = tid - NEL;
        unsigned mi = 0u, mj = 0u;
#pragma unroll
        for (int c = 0; c < 32; ++c) {
            mi |= (unsigned)(s_i[l][c] == s_i[ref][c]) << c;
            mj |= (unsigned)(s_j[l][c] == s_j[ref][c]) << c;
        }
        s_mi[l] = mi;
        s_mj[l] = mj;
    }
    __syncthreads();

    const bool mine = (act >> lane) & 1u;
    const double eta = mine ? etas[eta0 + e0 + lane] : 0.0;
    const float seta = sqrtf((float)(2.0 * eta));
    const unsigned mi = s_mi[lane], mj = s_mj[lane];
    const double ntau_d = (double)g.ntau;
    int buf = 0;
    for (int band = 0; band < 32 / RB; ++band, buf ^= 1) {
        const int r0 = band * RB;                // first tile row of the band
        // ---- gathers: lane = curvature e0 + lane, warp w on elements w, w + NW, ...
        const ThthPair* sref = s_ref[buf];
#pragma unroll 1
        for (int q0 = warp; q0 < NEL; q0 += NW * K) {
            ThthPair ps[K];
            OFF off[K];         // element offset into the copy (OFF = unsigned when it fits)
            unsigned hit = 0u;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int el = q0 + NW * k, r = r0 + (el >> 5), c = el & 31;
                off[k] = 0;
                ps[k].col = -1;
                if (!mine || (diag && c < r)) continue;     // lower triangle: not stored
                if ((mi >> r) & (mj >> c) & 1u) ps[k] = sref[el];
                else ps[k] = thth_pair_state(g, s_i[lane][r], s_j[lane][c], copy);
                if (ps[k].col >= 0) {
                    const double aa = __dadd_rn(__dsub_rn(__dmul_rn(eta, ps[k].d), g.tau0), g.half_dtau);
                    const double tqd = floor_div_fast(aa, g.dtau, g.inv_dtau);
                    if (tqd > 0.0 && tqd < ntau_d) {        // tau_inv > 0 and < ntau (ththmod.py:100)
                        const int tq = (int)tqd;
                        const int rr = ps[k].conj ? (int)g.ntau - tq : tq;
                        off[k] = (OFF)ps[k].col * (OFF)copy.tau_pitch + (OFF)rr;
                        hit |= 1u << k;
                    }
                }
            }
            // all K gathers in flight together (a miss reads element 0, ignored)
            float2 val[K];
#pragma unroll
            for (int k = 0; k < K; ++k)
                val[k] = SB_BUILD_PROBE == 1 ? make_float2(1.f, 0.f) : __ldg(copy.base + off[k]);
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int el = q0 + NW * k;
                if (!mine || (diag && (el & 31) < r0 + (el >> 5))) continue;
                s_v[lane][el] = ps[k].col >= 0 ? thth_element(val[k], (hit >> k) & 1u, ps[k].conj,
                                                              g.coherent, seta * ps[k].w)
                                               : make_float2(0.f, 0.f);
            }
        }
        __syncthreads();
        // the next band's reference states, while this one is stored
        if (tid < NEL && band + 1 < 32 / RB) ref_states(band + 1, s_ref[buf ^ 1]);

        // ---- stores: warp w on (curvature, band row) q = w, w + NW, ..., lane = column
#pragma unroll 1
        for (int q = warp; q < EB * RB; q += NW) {
            const int l = q / RB, la = r0 + q % RB;
            if (!((act >> l) & 1u)) continue;
            const bool low = diag && lane < la;     // below the diagonal: fp32 copy not stored
            const float2 v = low ? make_float2(0.f, 0.f) : s_v[l][(la - r0) * 32 + lane];
            const size_t e = (size_t)(e0 + l);
            if (!low && (SB_BUILD_PROBE != 2 || eta0 < 0))
                M[e * ld * ld + (unsigned)(ta * 32 + la) * (unsigned)ld + (unsigned)(tb * 32 + lane)] = v;
            if (PACK == 2)
                thth_store_f16_row(Mb + e * ld * ld, ((unsigned)(2 * ta + (la >> 4)) * (unsigned)(ld >> 3) +
                                   (unsigned)((tb * 32 + lane) >> 3)) * 128u + (unsigned)(la & 15) * 8u,
                                   diag, la, v, low, s_hscale[l]);
        }
        __syncthreads();
    }
}

// --------------------------------------------------------------------------
// compact copy of the spectrum columns a theta grid reaches (ThthCopy, thth.cuh)
// --------------------------------------------------------------------------
// mark[c] = 1 for every stored column c that some pair (i, j), j > i, i + j != n - 1, of
// ALL n centres maps to: a superset of what any curvature's cropped grid gathers, and
// independent of the curvature.  mark: int [thth_ncols(g)], zeroed by the caller.
__global__ void thth_colmark_kernel(ThthGeom g, int* __restrict__ mark) {
    const long long total = (long long)g.n * g.n;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(p / g.n), j = (int)(p % g.n);
        if (!(j > i && i + j != g.n - 1)) continue;
        bool mirrored;
        const int c = thth_pair_column(g, g.th[j], g.th[i], &mirrored);
        if (c >= 0) mark[c] = 1;
    }
}

// One block: marks -> slot_of_col [ncols] (slots in column order, -1 = not reached),
// col_of_slot [ncols] (first *nslots entries valid) and *nslots.  No slot >= cap is handed
// out (cap = the slot count the copy was sized for): such a column stays unmapped and
// *err is raised.
constexpr int SLOT_THREADS = 256;
__global__ void __launch_bounds__(SLOT_THREADS)
thth_colslots_kernel(const int* __restrict__ mark, int ncols, int cap,
                     int* __restrict__ slot_of_col, int* __restrict__ col_of_slot,
                     int* __restrict__ nslots, int* __restrict__ err) {
    SB_SHARED int s_cnt[SLOT_THREADS];
    const int t = threadIdx.x;
    const int per = (ncols + SLOT_THREADS - 1) / SLOT_THREADS;
    const int c0 = min(t * per, ncols), c1 = min(c0 + per, ncols);
    int cnt = 0;
    for (int c = c0; c < c1; ++c) cnt += mark[c] != 0;
    s_cnt[t] = cnt;
    __syncthreads();
    int s = 0, total = 0;
    for (int k = 0; k < SLOT_THREADS; ++k) {
        if (k < t) s += s_cnt[k];
        total += s_cnt[k];
    }
    for (int c = c0; c < c1; ++c) {
        int slot = -1;
        if (mark[c] != 0) {
            if (s < cap) { slot = s; col_of_slot[s] = c; }
            else atomicOr(err, 1);
            ++s;
        }
        slot_of_col[c] = slot;
    }
    if (t == 0) *nslots = total;
}

// C[slot][r] = CS[r][col_of_slot[slot]], C: float2 [nslots][tau_pitch].  32 x 32 tiles
// through shared memory, so that the reads run along the columns (neighbouring slots are
// neighbouring columns on a uniform grid) and the writes along the delay axis.
// grid = (ceil(ntau / 32), ceil(nslots / 32)), block = 32 x 8.
__global__ void __launch_bounds__(256)
cs_compact_kernel(const float2* __restrict__ cs, long long ntau, long long cs_pitch,
                  const int* __restrict__ col_of_slot, int nslots, long long tau_pitch,
                  float2* __restrict__ C) {
    SB_SHARED float2 tile[32][33];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const long long r0 = (long long)blockIdx.x * 32;
    const int s0 = blockIdx.y * 32;
    const int c = s0 + tx < nslots ? col_of_slot[s0 + tx] : -1;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const long long r = r0 + ty + 8 * k;
        if (c >= 0 && r < ntau) tile[ty + 8 * k][tx] = __ldg(cs + r * cs_pitch + c);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int s = s0 + ty + 8 * k;
        const long long r = r0 + tx;
        if (s < nslots && r < ntau) C[(long long)s * tau_pitch + r] = tile[tx][ty + 8 * k];
    }
}

// --------------------------------------------------------------------------
// Lanczos on the Hermitian matrix: largest ALGEBRAIC eigenvalue
// (scipy eigsh(..., k=1, which="LA"), ththmod.py:398-401), start vector =
// row n//2 (thth_start_vector, thth_lanczos: thth.cuh).
// --------------------------------------------------------------------------
// One CTA per eta.  The matrix is stored as its strict upper triangle; a warp
// owns rows a = warp, warp+NW, ... and for every stored element A[a][b] adds
//   A[a][b] * v[b]        to the row sum of a   (warp-shuffle reduction), and
//   conj(A[a][b]) * v[a]  to a per-lane accumulator of column b,
// so each element is read once per Lanczos step (half the traffic of a full
// mat-vec).  Direct 16-byte loads, any ld <= 4096, columns in chunks of 512.
constexpr int EIG_THREADS = 512;

__global__ void __launch_bounds__(EIG_THREADS)
thth_eig_kernel(const float2* __restrict__ Mbase, int ld,
                const int* __restrict__ nred, int eta0,
                double* __restrict__ eigs, int* __restrict__ status,
                int* __restrict__ iters, double tol, double etol, int max_iter) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int THREADS = EIG_THREADS, NW = THREADS / 32;
    LanczosShared& S = *reinterpret_cast<LanczosShared*>(smem_raw);
    float2* v = reinterpret_cast<float2*>(smem_raw + sizeof(LanczosShared));
    float2* vp = v + ld;
    float2* w = vp + ld;          // row sums, then the new Lanczos vector
    float2* u = w + ld;           // column sums
    float2* part = u + ld;        // [NW][512] per-warp column partials
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int e = blockIdx.x;
    const int n = nred[eta0 + e];
    const float2* M = Mbase + (size_t)e * ld * ld;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);

    if (status[eta0 + e] & SB_ETA_INDEX_ERROR) {
        if (tid == 0) { eigs[eta0 + e] = qnan; iters[eta0 + e] = 0; }
        return;
    }
    if (n < 3) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= SB_ETA_TOO_SMALL;
        }
        return;
    }
    if (!thth_start_vector<NW>(M, ld, n, v, vp, S.red[0])) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= SB_ETA_ZERO_START;
        }
        return;
    }

    const int ncol4 = (n + 1) >> 1;      // float4 = two complex columns
    const int nchunk = (n + 511) / 512;  // column chunks of 512
    auto matvec = [&]() {
        for (int c = tid; c < ld; c += THREADS) w[c] = make_float2(0.f, 0.f);
        __syncthreads();
        for (int cb = 0; cb < nchunk; ++cb) {
            float4 yc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) yc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int chunk_end = min(n, (cb + 1) * 512);
            // rows a = warp + NW*k with a + 1 < chunk_end
            const int K = (chunk_end - 2 >= warp) ? (chunk_end - 2 - warp) / NW + 1 : 0;
            for (int k = 0; k < K; ++k) {
                const int a = warp + NW * k;
                const int first4 = (a + 1) >> 1;
                const float2 xa = v[a];
                float4 mm[8];
                const float4* row = reinterpret_cast<const float4*>(M + (size_t)a * ld);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c4 = cb * 256 + lane + 32 * j;
                    mm[j] = (c4 >= first4 && c4 < ncol4) ? __ldg(row + c4)
                                                         : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                float rx = 0.f, ry = 0.f;
                const int jskip = (first4 - cb * 256) >> 5;   // groups entirely left of the diagonal
                thth_row_fma([&](int j, int) { return mm[j]; }, v, ld, cb * 256, jskip, xa, rx, ry, yc);
                rx = warp_sum(rx);
                ry = warp_sum(ry);
                if (lane == 0) { w[a].x += rx; w[a].y += ry; }
            }
            thth_fold_columns<NW>(yc, part, u, cb * 512, ld);
        }
    };
    const int m = thth_lanczos<NW>(S, matvec, v, vp, w, u, n, max_iter, tol, etol);
    if (tid == 0) {
        eigs[eta0 + e] = fabs(S.theta);  // np.abs(w[0])
        iters[eta0 + e] = m;
        if (!S.done) status[eta0 + e] |= SB_ETA_NOT_CONVERGED;
    }
}

// --------------------------------------------------------------------------
// Full N x N map for the thth_map API / parity tests (not the sweep path).
// --------------------------------------------------------------------------
__global__ void thth_map_kernel(ThthGeom g, double eta, int hermitian,
                                float2* __restrict__ out,
                                int* __restrict__ tau_inv,
                                int* __restrict__ fd_inv,
                                unsigned char* __restrict__ pnts,
                                int* __restrict__ err) {
    long long total = (long long)g.n * g.n;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
         p < total; p += (long long)gridDim.x * blockDim.x) {
        int i = (int)(p / g.n), j = (int)(p % g.n);
        double thi = g.th[i], thj = g.th[j];
        ThthPoint pt = thth_point(g, eta, thj, thi);
        if (pt.index_error) atomicOr(err, SB_ETA_INDEX_ERROR);
        if (tau_inv) tau_inv[p] = (int)max(min(pt.tq, (long long)INT_MAX), (long long)INT_MIN);
        if (fd_inv) fd_inv[p] = (int)max(min(pt.fq, (long long)INT_MAX), (long long)INT_MIN);
        if (pnts) pnts[p] = pt.pnt ? 1 : 0;
        if (!out) continue;
        float2 v;
        if (!hermitian) {
            v = thth_value(g, eta, thj, thi, pt);
        } else if (i == j || i + j == g.n - 1) {
            v = make_float2(0.f, 0.f);
        } else if (j > i) {
            v = thth_value(g, eta, thj, thi, pt);
            v.x = nan_to_num(v.x);
            v.y = nan_to_num(v.y);
        } else {  // conj of the upper element (j, i)
            ThthPoint pu = thth_point(g, eta, thi, thj);
            v = thth_value(g, eta, thi, thj, pu);
            v.x = nan_to_num(v.x);
            v.y = -nan_to_num(v.y);
        }
        out[p] = v;
    }
}

#ifndef SB_HOST_EMU
// --------------------------------------------------------------------------
// host drivers
// --------------------------------------------------------------------------
// Items per launch of a batched driver: as many as per_item bytes each fit the per-launch
// budget of the work buffers, 3 GiB or SB_SWEEP_SLAB_MB (tests use it to force batching);
// at least 1, at most cap (the largest batch the caller's grid takes) and at most count.
int sweep_batch(size_t per_item, int count, int cap) {
    unsigned long long slab = 3ull << 30;
    if (const char* ev = getenv("SB_SWEEP_SLAB_MB")) {
        const long mb = atol(ev);
        if (mb > 0) slab = (unsigned long long)mb << 20;
    }
    unsigned long long b = slab / per_item;
    if (b < 1) b = 1;
    if (b > (unsigned long long)cap) b = cap;
    if (b > (unsigned long long)count) b = count;
    return (int)b;
}

static bool lower_check_needed(const ThthGeom& g, const double* th_host) {
    // The fd argument th1 - th2 spans [-(max(th) - min(th)), max(th) - min(th)]; the
    // smallest fd_inv comes from the negative end on an ascending fd axis and from the
    // positive end on a descending one (dfd < 0), so take the smaller of the two.
    double tmin = th_host[0], tmax = th_host[0];
    for (int k = 1; k < g.n; ++k) {
        tmin = th_host[k] < tmin ? th_host[k] : tmin;
        tmax = th_host[k] > tmax ? th_host[k] : tmax;
    }
    const double lo = floor(((tmin - tmax) - g.fd0 + g.half_dfd) / g.dfd);
    const double hi = floor(((tmax - tmin) - g.fd0 + g.half_dfd) / g.dfd);
    const double worst = (lo < hi ? lo : hi) - 2.0;
    return !(worst >= -(double)g.nfd);
}

// crop masks (d_idx [neta][ld], d_nred) and the IndexError status bit of every eta;
// d_status is cleared first
int thth_prep(const ThthGeom& g, const double* th_host, const double* d_etas, int neta, int ld,
              int* d_idx, int* d_nred, int* d_status, cudaStream_t st) {
    SB_CUDA(cudaMemsetAsync(d_status, 0, neta * sizeof(int), st));
    prof_begin(PROF_THTH_PREP, st);
    thth_prep_kernel<<<neta, 32, 0, st>>>(g, d_etas, neta, ld, d_idx, d_nred);
    prof_end(PROF_THTH_PREP, st);
    SB_LAUNCH_CHECK();
    // one curvature per gridDim.y row, which CUDA caps at 65535: launches of at most 65535
    const bool check = lower_check_needed(g, th_host);
    for (int e0 = 0; check && e0 < neta; e0 += 65535) {
        const int nb = neta - e0 < 65535 ? neta - e0 : 65535;
        thth_indexerr_kernel<<<dim3(64, nb), 256, 0, st>>>(g, d_etas + e0, d_status + e0);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

// thth_prep for a table of n geometries, one curvature each: geoms / th_host on the host,
// the same geometries in d_geoms on the device
int thth_prep_table(const ThthGeom* geoms, const double* const* th_host, const ThthGeom* d_geoms,
                    const double* d_etas, int n, int ld, int* d_idx, int* d_nred, int* d_status,
                    cudaStream_t st) {
    SB_CUDA(cudaMemsetAsync(d_status, 0, n * sizeof(int), st));
    thth_prep_table_kernel<<<n, 32, 0, st>>>(d_geoms, d_etas, ld, d_idx, d_nred);
    SB_LAUNCH_CHECK();
    bool check = false;
    for (int k = 0; k < n && !check; ++k) check = lower_check_needed(geoms[k], th_host[k]);
    for (int e0 = 0; check && e0 < n; e0 += 65535) {
        const int nb = n - e0 < 65535 ? n - e0 : 65535;
        thth_indexerr_table_kernel<<<dim3(64, nb), 256, 0, st>>>(d_geoms, d_etas, e0, d_status);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

// Where the gathers of one sweep call read (ThthCopy, thth.cuh), made once per call and
// shared by its curvature batches.
//
// The table of reached columns is built on the device (thth_colmark_kernel,
// thth_colslots_kernel) on every call; the host only needs the slot count, to size the
// copy and to choose.  It is read back once per geometry (one stream synchronise) and kept:
// the table depends on the theta centres and the fd axis only, and the kernels are
// deterministic, so later calls with the same geometry get the same count without a
// read-back, and hand it to thth_colslots_kernel as the cap no slot may reach.
//
// The copy is used when the 32-byte sectors the direct gather would read, one per
// gathered element (neighbouring curvatures of a pair sit a whole CS row apart), are at
// least twice the bytes of making the copy (a sector read + 8 bytes written per element):
// few curvatures, or a grid whose pairs all fall on different columns, gather from the
// spectrum itself.
struct ColCache {
    bool valid = false;
    long long nfd = 0;
    int cs_half = 0, n = 0;
    double fd0 = 0, dfd = 0, half_dfd = 0, inv_dfd = 0;
    std::vector<double> th;
    int nslots = 0;
    bool checked = false;   // the error word has been read back after a sweep from the copy
};
static ColCache g_colcache;

int thth_gather_source(const ThthGeom& g, const double* th_host, int neta, ThthCopy* copy,
                       cudaStream_t st) {
    const int ncols = (int)(g.cs_half ? g.nfd / 2 + 1 : g.nfd);
    const size_t tab_bytes = ((size_t)(3 * (size_t)ncols + 2) * sizeof(int) + 255) & ~(size_t)255;
    ColCache& cc = g_colcache;
    const bool hit = cc.valid && cc.nfd == g.nfd && cc.cs_half == g.cs_half && cc.n == g.n &&
                     cc.fd0 == g.fd0 && cc.dfd == g.dfd && cc.half_dfd == g.half_dfd &&
                     cc.inv_dfd == g.inv_dfd &&
                     memcmp(cc.th.data(), th_host, (size_t)g.n * sizeof(double)) == 0;
    // [mark | slot_of_col | col_of_slot | nslots, err] then the copy
    auto build_table = [&](int* tab, int cap) -> int {
        int* mark = tab;
        int* slot_of_col = tab + ncols;
        int* col_of_slot = tab + 2 * (size_t)ncols;
        int* tail = tab + 3 * (size_t)ncols;
        // zero: marks, the error word, and col_of_slot (an entry the scan does not write
        // is column 0, inside the spectrum)
        SB_CUDA(cudaMemsetAsync(tab, 0, tab_bytes, st));
        const long long pairs = (long long)g.n * g.n;
        int blocks = (int)((pairs + 255) / 256);
        if (blocks > num_sms() * 16) blocks = num_sms() * 16;
        thth_colmark_kernel<<<blocks, 256, 0, st>>>(g, mark);
        SB_LAUNCH_CHECK();
        thth_colslots_kernel<<<1, SLOT_THREADS, 0, st>>>(mark, ncols, cap, slot_of_col,
                                                         col_of_slot, tail, tail + 1);
        SB_LAUNCH_CHECK();
        return SB_OK;
    };
    if (!hit) {
        int* tab = (int*)workspace(WS_TABLE, tab_bytes);
        if (!tab) return SB_ERR_NOMEM;
        int rc = build_table(tab, INT_MAX);
        if (rc) return rc;
        int nslots = 0;
        SB_CUDA(cudaMemcpyAsync(&nslots, tab + 3 * (size_t)ncols, sizeof(int),
                                cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
        if (nslots < 0 || nslots > ncols) {
            set_error("theta-theta column table: %d slots for %d columns", nslots, ncols);
            return SB_ERR_CUDA;
        }
        cc.valid = true;
        cc.nfd = g.nfd; cc.cs_half = g.cs_half; cc.n = g.n;
        cc.fd0 = g.fd0; cc.dfd = g.dfd; cc.half_dfd = g.half_dfd; cc.inv_dfd = g.inv_dfd;
        cc.th.assign(th_host, th_host + g.n);
        cc.nslots = nslots;
        cc.checked = false;
    }
    const int nslots = cc.nslots;
    const long long tau_pitch = (g.ntau + 3) / 4 * 4;
    const double pairs = 0.5 * (double)g.n * (double)(g.n - 1);
    const double direct_bytes = 32.0 * (double)neta * pairs;
    const double copy_bytes = 40.0 * (double)nslots * (double)g.ntau;
    if (nslots == 0 || direct_bytes < 2.0 * copy_bytes) {
        *copy = ThthCopy{nullptr, 0, 0, nullptr, nullptr};
        return SB_OK;
    }
    unsigned char* ws = (unsigned char*)workspace(
        WS_TABLE, tab_bytes + (size_t)nslots * (size_t)tau_pitch * sizeof(float2));
    if (!ws) return SB_ERR_NOMEM;
    int* tab = (int*)ws;
    float2* C = (float2*)(ws + tab_bytes);
    prof_begin(PROF_THTH_BUILD, st);
    int rc = build_table(tab, nslots);
    if (!rc) {
        const dim3 grid((unsigned)((g.ntau + 31) / 32), (unsigned)((nslots + 31) / 32));
        cs_compact_kernel<<<grid, dim3(32, 8), 0, st>>>(g.cs, g.ntau, g.cs_pitch,
                                                        tab + 2 * (size_t)ncols, nslots,
                                                        tau_pitch, C);
    }
    prof_end(PROF_THTH_BUILD, st);
    if (rc) return rc;
    SB_LAUNCH_CHECK();
    *copy = ThthCopy{C, tau_pitch, nslots, tab + ncols, tab + 3 * (size_t)ncols + 1};
    return SB_OK;
}

// After the gathers of a sweep: the first sweep of a geometry that read the copy waits for
// them and reports a raised error word (a pair whose column the table did not hold: its
// element was left zero).  Later sweeps of the same geometry do not wait.
int thth_gather_check(const ThthCopy& copy, cudaStream_t st) {
    if (!copy.base || g_colcache.checked) return SB_OK;
    int err = 0;
    SB_CUDA(cudaMemcpyAsync(&err, copy.err, sizeof(int), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    if (err) {
        set_error("theta-theta gather: a pair of the grid maps to a spectrum column that the "
                  "table of reached columns does not hold");
        return SB_ERR_CUDA;
    }
    g_colcache.checked = true;
    return SB_OK;
}

// gather of etas e0 .. e0 + nb - 1, from the copy if there is one and from the spectrum
// otherwise, into the fp32 strict upper triangles d_M [nb][ld][ld] and, PACK == 2, the fp16
// copy d_Mb; 32-bit offsets whenever what is gathered from has fewer than 2^32 elements
template <int PACK>
static void thth_build_launch(const ThthGeom& g, const ThthCopy& copy, const double* d_etas,
                              int e0, int nb, int ld, const int* d_idx, const int* d_nred,
                              float2* d_M, unsigned* d_Mb, const unsigned* d_absmax, float span,
                              cudaStream_t st) {
    const int T = ld / 32;
    const dim3 block(32, 8);
    if (copy.base) {
        const dim3 grid((nb + SB_COPY_EB - 1) / SB_COPY_EB, T * (T + 1) / 2);
        if ((unsigned long long)copy.nslots * (unsigned long long)copy.tau_pitch < (1ull << 32))
            thth_build_copy_kernel<PACK, unsigned><<<grid, block, 0, st>>>(
                g, d_etas, e0, nb, ld, d_idx, d_nred, d_M, d_Mb, d_absmax, span, copy);
        else
            thth_build_copy_kernel<PACK, size_t><<<grid, block, 0, st>>>(
                g, d_etas, e0, nb, ld, d_idx, d_nred, d_M, d_Mb, d_absmax, span, copy);
        return;
    }
    const dim3 grid((nb + SB_BUILD_EB - 1) / SB_BUILD_EB, T * (T + 1) / 2);
    if ((unsigned long long)g.ntau * (unsigned long long)g.cs_pitch < (1ull << 32))
        thth_build_kernel<PACK, unsigned><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                  d_nred, d_M, d_Mb, d_absmax, span);
    else
        thth_build_kernel<PACK, size_t><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                d_nred, d_M, d_Mb, d_absmax, span);
}

// fp32 strict upper triangles [nb][ld][ld] of etas e0 .. e0 + nb - 1 (no fp16 copy)
int thth_build_f32(const ThthGeom& g, const ThthCopy& copy, const double* d_etas, int e0, int nb,
                   int ld, const int* d_idx, const int* d_nred, float2* d_M, cudaStream_t st) {
    thth_build_launch<0>(g, copy, d_etas, e0, nb, ld, d_idx, d_nred, d_M, nullptr, nullptr, 0.f, st);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int eta_sweep(const ThthGeom& g, const double* th_host, const double* d_etas,
              int neta, double tol, int max_iter, double* d_eigs,
              int* d_status, int* d_nred, int* d_iters, cudaStream_t st) {
    if (neta <= 0) return SB_OK;
    if (max_iter <= 0 || max_iter > SB_LANCZOS_MAXIT) max_iter = SB_LANCZOS_MAXIT;
    const int ld = (g.n + 31) / 32 * 32;
    if (ld > 4096) {
        set_error("theta-theta grid of %d centres exceeds the supported 4096", g.n);
        return SB_ERR_UNSUPPORTED;
    }
    int* d_idx = (int*)workspace(WS_INDEX, (size_t)neta * ld * sizeof(int));
    if (!d_idx) return SB_ERR_NOMEM;
    int rc = thth_prep(g, th_host, d_etas, neta, ld, d_idx, d_nred, d_status, st);
    if (rc) return rc;
    ThthCopy copy;
    rc = thth_gather_source(g, th_host, neta, &copy, st);
    if (rc) return rc;
    const size_t per = (size_t)ld * ld * sizeof(float2);
    const int batch = sweep_batch(per, neta, INT_MAX);
    float2* d_M = (float2*)workspace(WS_BATCH, per * batch);
    if (!d_M) return SB_ERR_NOMEM;
    // default solver for ld <= 512 (eig_half.cu): iterates on the fp16 copy written by the
    // build kernel.  Larger grids, and every grid with SB_EIG_FP32=1, run the fp32
    // thth_eig_kernel, the reference the default solver is checked against.
    const bool fp16 = (ld <= 512) && !getenv("SB_EIG_FP32");
    unsigned* d_Mb = nullptr;
    // scale of the fp16 copy: max |CS| over what the gather can reach, max |theta2 - theta1|
    unsigned* d_absmax = nullptr;
    float span = 0.f;
    size_t smem = 0;
    if (fp16) {
        d_Mb = (unsigned*)workspace(WS_PLANE3, per / 2 * batch);
        if (!d_Mb) return SB_ERR_NOMEM;
        ScalarBlock* sc = scalar_block();
        if (!sc) return SB_ERR_NOMEM;
        d_absmax = &sc->sweep_scale;
        if (g.cs_bound) {       // the caller knows a bound (sb_cs_bound_f32): no scan
            SB_CUDA(cudaMemcpyAsync(d_absmax, g.cs_bound, sizeof(float), cudaMemcpyDeviceToDevice, st));
        } else {
            SB_CUDA(cudaMemsetAsync(d_absmax, 0, sizeof(unsigned), st));
            const long long ncols = g.cs_half ? (g.cs_valid_cols > 0 ? g.cs_valid_cols : g.nfd / 2 + 1)
                                              : g.nfd;
            if (g.cs_pitch % 2 == 0 && ((uintptr_t)g.cs & 15) == 0)
                cs_absmax_kernel<true><<<num_sms() * 8, 256, 0, st>>>(g.cs, g.ntau, ncols, g.cs_pitch,
                                                                      d_absmax);
            else
                cs_absmax_kernel<false><<<num_sms() * 8, 256, 0, st>>>(g.cs, g.ntau, ncols, g.cs_pitch,
                                                                       d_absmax);
            SB_LAUNCH_CHECK();
        }
        double tmin = th_host[0], tmax = th_host[0];
        for (int k = 1; k < g.n; ++k) {
            tmin = th_host[k] < tmin ? th_host[k] : tmin;
            tmax = th_host[k] > tmax ? th_host[k] : tmax;
        }
        span = (float)((tmax - tmin) * 1.0001);
    } else {
        // Lanczos state, v, vp, w, u and the per-warp column partials
        smem = sizeof(LanczosShared) + 4 * (size_t)ld * sizeof(float2) +
               (size_t)(EIG_THREADS / 32) * 4096;
        SB_CUDA(cudaFuncSetAttribute(thth_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    }
    for (int e0 = 0; e0 < neta; e0 += batch) {
        const int nb = neta - e0 < batch ? neta - e0 : batch;
        prof_begin(PROF_THTH_BUILD, st);
        if (fp16)
            thth_build_launch<2>(g, copy, d_etas, e0, nb, ld, d_idx, d_nred, d_M, d_Mb, d_absmax, span, st);
        else
            thth_build_launch<0>(g, copy, d_etas, e0, nb, ld, d_idx, d_nred, d_M, nullptr, nullptr, 0.f,
                                 st);
        prof_end(PROF_THTH_BUILD, st);
        SB_LAUNCH_CHECK();
        prof_begin(PROF_THTH_EIG, st);
        if (fp16) {
            rc = eig_half_launch(d_M, d_Mb, ld, d_nred, e0, nb, d_eigs, d_status, d_iters, tol,
                                 2e-7, max_iter, st);
            if (rc) return rc;
        } else {
            thth_eig_kernel<<<nb, EIG_THREADS, smem, st>>>(d_M, ld, d_nred, e0, d_eigs, d_status,
                                                           d_iters, tol, 2e-7, max_iter);
        }
        prof_end(PROF_THTH_EIG, st);
        SB_LAUNCH_CHECK();
    }
    return thth_gather_check(copy, st);
}

__global__ void thth_mask_kernel(ThthGeom g, double eta,
                                 unsigned char* __restrict__ mask) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= g.n) return;
    double t = g.th[k];
    mask[k] = ((__dmul_rn(__dmul_rn(t, t), eta) < g.tau_absmax) &&
               (fabs(t) < g.fd_half)) ? 1 : 0;
}

int thth_map(const ThthGeom& g, double eta, int hermitian, float2* d_out,
             int* d_tau_inv, int* d_fd_inv, unsigned char* d_pnts,
             unsigned char* d_th_pnts, int* d_err, cudaStream_t st) {
    if (d_th_pnts) {
        thth_mask_kernel<<<(g.n + 255) / 256, 256, 0, st>>>(g, eta, d_th_pnts);
        SB_LAUNCH_CHECK();
    }
    if (!d_err) return SB_OK;
    SB_CUDA(cudaMemsetAsync(d_err, 0, sizeof(int), st));
    long long total = (long long)g.n * g.n;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    thth_map_kernel<<<blocks, 256, 0, st>>>(g, eta, hermitian, d_out, d_tau_inv,
                                            d_fd_inv, d_pnts, d_err);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
