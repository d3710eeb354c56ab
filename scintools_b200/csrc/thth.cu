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

#include "drivers.cuh"
#include "lanczos.cuh"
#include "thth.cuh"

namespace sb {

// status codes per eta (also in include/scint_b200.h)
enum { ST_OK = 0, ST_INDEX_ERROR = 1, ST_ZERO_START = 2, ST_TOO_SMALL = 4,
       ST_NOT_CONVERGED = 8 };

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
        atomicOr(status, ST_INDEX_ERROR);
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
// uses every stored element twice).  grid = (tile pairs, etas in batch),
// block = 32 x 8.  M[e] is [ld][ld] float2; inside the active 32x32 tiles
// columns >= nred and the diagonal are zero, the lower triangle is not touched.
// --------------------------------------------------------------------------
#define SB_BUILD_EB 8

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

// PACK == 2: also write the fp16 copy Mb that eig_half.cu iterates on,
// scaled by the power of two that puts absmax * max Jacobian of this curvature just
// below 2^15 (absmax: device scalar from cs_absmax_kernel, span: max |theta2 - theta1|).
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
// gathers are in flight per thread.
// COPY: the gathers read the compact copy of the spectrum columns the grid reaches
// (ThthCopy, thth.cuh), delay axis contiguous, where neighbouring curvatures of a pair fall
// in the same or the next 32-byte sector and the whole copy is re-read from L2
// (thth_build_copy_kernel); otherwise the spectrum itself, where every gather costs a DRAM
// sector of its own (thth_build_kernel).  thth_gather_source chooses.
// PACK == 0: the fp32 triangle only.  PACK == 2: also the fp16 copy in the block layout
// of eig_half.cu's tensor-core mat-vec: 512-byte blocks of 16 rows x 8 columns, block
// (I, G) at ((I * ld / 8 + G) * 512) bytes, a block row = [re x 8 | im x 8] (the halves
// swapped in rows 4-7, 12-15); the part of a diagonal block on / below the diagonal is
// written as zeros (the MMA has no masks).
// Three CTAs per SM (80 registers; spill stores per thread in the PACK == 2 instances on
// sm_90: 40-44 bytes reading the spectrum, 12-20 bytes reading the copy).  Measured on the
// headline sweep from the compact copy (H100 SXM, 700 W power limit, thth_build per
// 1024-eta launch, copy included), variants built from one source and alternated in one
// run: 1.76 ms as is; 1.78 ms with streaming (__stcs) stores of the triangles, alone or with
// an L2 evict-last policy on the gathers; 1.84 ms with the tile pairs ordered by diagonal;
// 1.78 ms with four CTAs per SM (64 registers, ~170 bytes of spills), which also slows the
// gather from the spectrum itself (2.41 against 2.23 ms on an irregular grid).  None of
// them is kept.
template <int PACK, typename OFF, bool COPY>
__device__ __forceinline__ void
thth_build_body(const ThthGeom& g, const double* __restrict__ etas, int eta0, int nbatch,
                int ld, const int* __restrict__ idx,
                const int* __restrict__ nred, float2* __restrict__ M,
                unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span,
                const ThthCopy& copy) {
    // eta is the FAST grid index: CTAs resident at the same time work on the
    // same 32x32 tile for neighbouring curvatures, whose gathers fall on
    // the same / adjacent delay bins for small |theta1^2 - theta2^2| (L2 reuse)
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
    int col[ROWS];          // CS column (COPY: slot of the copy) to gather; < 0: never a valid point
    unsigned conj = 0u;     // bit k: the point lies in the mirrored (fd < 0) half
    float wk[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) { ci[k] = -2; dk[k] = 0.0; col[k] = -1; wk[k] = 0.f; }
    const int e_end = min(nbatch, (int)(blockIdx.x + 1) * SB_BUILD_EB);
    // per-curvature power-of-two scale of the fp16 copy, once per CTA (it was ~40 instructions
    // of log2f / exp2f per thread and curvature): 2^floor(log2(2^15 / bound)) is the exponent
    // field of the quotient
    __shared__ float s_hscale[SB_BUILD_EB];
    if (PACK != 0) {
        const int lin = ty * 32 + tx;
        if (lin < SB_BUILD_EB) {
            const int e = blockIdx.x * SB_BUILD_EB + lin;
            float hs = 1.f;
            if (e < e_end) {
                const float seta = sqrtf((float)(2.0 * etas[eta0 + e]));
                const float bound = __uint_as_float(*absmax) * seta * sqrtf(span);
                if (bound > 0.f && bound < 3.0e38f) {
                    const float q = 32768.f / bound;
                    hs = q >= 1.1754944e-38f ? __uint_as_float(__float_as_uint(q) & 0x7f800000u) : 1.1754944e-38f;
                }
            }
            s_hscale[lin] = hs;
        }
        __syncthreads();
    }
    // eta-independent store offsets: fp32 element (row a0 + TY k, column b) and, PACK == 2,
    // the 4-byte word of the fp16 block row this lane stores (see phase 3)
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
        OFF off[ROWS];          // element offset into the CS / the copy (OFF = unsigned when it fits)
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
                    int c = thth_pair_column(g, th1, th2, &mirrored);
                    if (COPY && c >= 0) {
                        c = copy.slot_of_col[c];
                        // a column the copy does not hold: the element stays zero, no
                        // address is formed from it
                        if (c < 0) atomicOr(copy.err, 1);
                    }
                    col[k] = c;
                    if (mirrored) conj |= 1u << k;
                }
            }
            if (col[k] >= 0) {
                const double aa = __dadd_rn(__dsub_rn(__dmul_rn(eta, dk[k]), g.tau0), g.half_dtau);
                const double tqd = floor_div_fast(aa, g.dtau, g.inv_dtau);
                if (tqd > 0.0 && tqd < ntau_d) {            // tau_inv > 0 and < ntau (ththmod.py:100)
                    const int tq = (int)tqd;
                    const int r = (conj >> k) & 1u ? (int)g.ntau - tq : tq;
                    off[k] = COPY ? (OFF)col[k] * (OFF)copy.tau_pitch + (OFF)r
                                  : (OFF)r * (OFF)g.cs_pitch + (OFF)col[k];
                    hit |= 1u << k;
                }
            }
        }
        // ---- phase 2: the gathers, all in flight together (a miss reads element 0, ignored)
        float2 val[ROWS];
        const float2* __restrict__ from = COPY ? copy.base : g.cs;
#pragma unroll
        for (int k = 0; k < ROWS; ++k) val[k] = __ldg(from + off[k]);
        // ---- phase 3
#pragma unroll
        for (int k = 0; k < ROWS; ++k) {
            const int la = ty + TY * k;
            const bool low = ta == tb && tx < la;       // below the diagonal: fp32 copy not stored
            float2 v = make_float2(0.f, 0.f);
            if (!low) {
                if (col[k] >= 0) {
                    if ((hit >> k) & 1u) {
                        v = val[k];
                        if ((conj >> k) & 1u) v.y = -v.y;
                        if (!g.coherent) v = make_float2(hypotf(v.x, v.y), 0.f);
                    }
                    // Jacobian sqrt|2 eta (th2 - th1)| (ththmod.py:107)
                    const float wf = seta * wk[k];
                    v.x *= wf;
                    v.y *= wf;
                    if (!(fabsf(v.x) <= 3.402823466e+38f) || !(fabsf(v.y) <= 3.402823466e+38f)) {
                        v.x = nan_to_num(v.x);
                        v.y = nan_to_num(v.y);
                    }
                }
                const unsigned o = foff0 + (unsigned)k * frow;
                Me[o] = v;
            }
            if (PACK == 2) {
                // block row of 8 columns = [re x 8 | im x 8] (32 bytes): the 8 lanes of a column
                // group trade halves so that lane i stores 4-byte word i of it -- one store
                // instruction, four full 32-byte sectors per warp (2-byte stores would be slower).
                // Elements on / below the diagonal of a diagonal block are zeros (the MMA has
                // no masks); 16 x 16 sub-blocks entirely below the diagonal are never read.
                const unsigned h = low ? 0u : pack_f16x2(make_float2(v.x * hscale, v.y * hscale));
                const int i8 = tx & 7, s0 = (tx & ~7) + 2 * (i8 & 3);
                const unsigned ha = __shfl_sync(0xffffffffu, h, s0);
                const unsigned hb = __shfl_sync(0xffffffffu, h, s0 + 1);
                const unsigned word = i8 < 4 ? ((ha & 0xffffu) | (hb << 16)) : ((ha >> 16) | (hb & 0xffff0000u));
                if (!(ta == tb && (tx >> 4) < (la >> 4))) {
                    // row a = 32 ta + ty + TY k: block row 2 ta + (la >> 4), row (la & 15) in it
                    unsigned* Mw = Mb + (size_t)e * ld * ld;
                    // the two 16-byte halves of a block row are stored swapped in rows 4-7 and
                    // 12-15: a LINEAR copy of the block into shared memory is then conflict free for
                    // both ldmatrix forms (eig_half.cu), so a bulk copy can fetch it
                    const unsigned swz = (unsigned)(((la & 15) >> 2) & 1) << 2;
                    Mw[woff0 + (unsigned)(la >> 4) * (unsigned)(ld >> 3) * 128u + (unsigned)((la & 15) - ty) * 8u +
                       ((unsigned)i8 ^ swz)] = word;
                }
            }
        }
    }
}

template <int PACK, typename OFF>
__global__ void __launch_bounds__(256, 3)
thth_build_kernel(ThthGeom g, const double* __restrict__ etas, int eta0, int nbatch,
                  int ld, const int* __restrict__ idx,
                  const int* __restrict__ nred, float2* __restrict__ M,
                  unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span) {
    thth_build_body<PACK, OFF, false>(g, etas, eta0, nbatch, ld, idx, nred, M, Mb, absmax, span,
                                      ThthCopy{nullptr, 0, 0, nullptr, nullptr});
}

template <int PACK, typename OFF>
__global__ void __launch_bounds__(256, 3)
thth_build_copy_kernel(ThthGeom g, const double* __restrict__ etas, int eta0, int nbatch,
                       int ld, const int* __restrict__ idx,
                       const int* __restrict__ nred, float2* __restrict__ M,
                       unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span,
                       ThthCopy copy) {
    thth_build_body<PACK, OFF, true>(g, etas, eta0, nbatch, ld, idx, nred, M, Mb, absmax, span,
                                     copy);
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
// row n//2.  No re-orthogonalisation: only the top Ritz value is wanted.
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

    if (status[eta0 + e] & ST_INDEX_ERROR) {
        if (tid == 0) { eigs[eta0 + e] = qnan; iters[eta0 + e] = 0; }
        return;
    }
    if (n < 3) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= ST_TOO_SMALL;
        }
        return;
    }
    // v0 = row n//2 of the Hermitian matrix (ththmod.py:398-399)
    const int h = n / 2;
    double part0 = 0.0;
    for (int c = tid; c < ld; c += THREADS) {
        float2 x = make_float2(0.f, 0.f);
        if (c < n && c > h) x = M[(size_t)h * ld + c];
        else if (c < h) { x = M[(size_t)c * ld + h]; x.y = -x.y; }
        v[c] = x;
        vp[c] = make_float2(0.f, 0.f);
        part0 += (double)x.x * x.x + (double)x.y * x.y;
    }
    part0 = warp_sum(part0);
    if (lane == 0) S.red[0][warp] = part0;
    if (tid == 0) {
        S.done = 0; S.lo = 0.0; S.theta = 0.0; S.res = 0.0;
        S.next_check = 1; S.m_last = 0; S.beta2[0] = 0.0;
    }
    __syncthreads();
    double nrm2 = 0.0;
    for (int k = 0; k < NW; ++k) nrm2 += S.red[0][k];
    if (!(nrm2 > 0.0) || !isfinite(nrm2)) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= ST_ZERO_START;
        }
        return;
    }
    {
        float s = (float)(1.0 / sqrt(nrm2));
        for (int c = tid; c < ld; c += THREADS) { v[c].x *= s; v[c].y *= s; }
    }
    __syncthreads();

    const int ncol4 = (n + 1) >> 1;      // float4 = two complex columns
    const int nchunk = (n + 511) / 512;  // column chunks of 512
    float beta_prev = 0.f;
    int m = 0;
    for (int it = 0; it < max_iter; ++it) {
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
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (j < jskip) continue;
                    const int c4 = cb * 256 + lane + 32 * j;
                    const float4 q = mm[j];
                    const float4 x = (2 * c4 < ld) ? *reinterpret_cast<const float4*>(v + 2 * c4)
                                                   : make_float4(0.f, 0.f, 0.f, 0.f);
                    // explicit FMA chains (16 FFMA per two complex elements)
                    rx = fmaf(q.x, x.x, rx); rx = fmaf(-q.y, x.y, rx);
                    rx = fmaf(q.z, x.z, rx); rx = fmaf(-q.w, x.w, rx);
                    ry = fmaf(q.x, x.y, ry); ry = fmaf(q.y, x.x, ry);
                    ry = fmaf(q.z, x.w, ry); ry = fmaf(q.w, x.z, ry);
                    // conj(A) * v[a]
                    yc[j].x = fmaf(q.x, xa.x, yc[j].x); yc[j].x = fmaf(q.y, xa.y, yc[j].x);
                    yc[j].y = fmaf(q.x, xa.y, yc[j].y); yc[j].y = fmaf(-q.y, xa.x, yc[j].y);
                    yc[j].z = fmaf(q.z, xa.x, yc[j].z); yc[j].z = fmaf(q.w, xa.y, yc[j].z);
                    yc[j].w = fmaf(q.z, xa.y, yc[j].w); yc[j].w = fmaf(-q.w, xa.x, yc[j].w);
                }
                rx = warp_sum(rx);
                ry = warp_sum(ry);
                if (lane == 0) { w[a].x += rx; w[a].y += ry; }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float4*>(part + warp * 512 + 2 * (lane + 32 * j)) = yc[j];
            __syncthreads();
            for (int c = tid; c < 512; c += THREADS) {
                float sx = 0.f, sy = 0.f;
#pragma unroll
                for (int k = 0; k < NW; ++k) { sx += part[k * 512 + c].x; sy += part[k * 512 + c].y; }
                if (cb * 512 + c < ld) u[cb * 512 + c] = make_float2(sx, sy);
            }
            __syncthreads();
        }
        // ---- alpha = Re <v, A v>
        double apart = 0.0;
        for (int c = tid; c < n; c += THREADS) {
            float2 x = w[c];
            x.x += u[c].x;
            x.y += u[c].y;
            w[c] = x;
            apart += (double)(v[c].x * x.x + v[c].y * x.y);
        }
        apart = warp_sum(apart);
        if (lane == 0) S.red[0][warp] = apart;
        __syncthreads();
        double alpha = 0.0;
        for (int k = 0; k < NW; ++k) alpha += S.red[0][k];
        // ---- w -= alpha v + beta_prev vp ; beta = ||w||
        const float af = (float)alpha;
        double bpart = 0.0;
        for (int c = tid; c < n; c += THREADS) {
            float2 x = w[c];
            x.x -= af * v[c].x + beta_prev * vp[c].x;
            x.y -= af * v[c].y + beta_prev * vp[c].y;
            w[c] = x;
            bpart += (double)x.x * x.x + (double)x.y * x.y;
        }
        bpart = warp_sum(bpart);
        if (lane == 0) S.red[1][warp] = bpart;
        __syncthreads();
        double b2 = 0.0;
        for (int k = 0; k < NW; ++k) b2 += S.red[1][k];
        const double beta = sqrt(b2);
        m = it + 1;
        if (tid == 0) { S.alpha[it] = alpha; S.beta[m] = beta; S.beta2[m] = b2; }
        __syncthreads();
        const bool last = (it + 1 == max_iter);
        if (warp == 0 && (m >= S.next_check || last || !(beta > 0.0)))
            lanczos_check(S, m, tol, etol);
        __syncthreads();
        if (S.done || !isfinite(alpha)) break;
        // ---- rotate: vp = v, v = w / beta
        const float ib = (float)(1.0 / beta);
        for (int c = tid; c < n; c += THREADS) {
            float2 x = w[c];
            vp[c] = v[c];
            v[c] = make_float2(x.x * ib, x.y * ib);
        }
        beta_prev = (float)beta;
        __syncthreads();
    }
    if (tid == 0) {
        eigs[eta0 + e] = fabs(S.theta);  // np.abs(w[0])
        iters[eta0 + e] = m;
        if (!S.done) status[eta0 + e] |= ST_NOT_CONVERGED;
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
        if (pt.index_error) atomicOr(err, ST_INDEX_ERROR);
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
    const dim3 grid((nb + SB_BUILD_EB - 1) / SB_BUILD_EB, T * (T + 1) / 2), block(32, 8);
    if (copy.base) {
        if ((unsigned long long)copy.nslots * (unsigned long long)copy.tau_pitch < (1ull << 32))
            thth_build_copy_kernel<PACK, unsigned><<<grid, block, 0, st>>>(
                g, d_etas, e0, nb, ld, d_idx, d_nred, d_M, d_Mb, d_absmax, span, copy);
        else
            thth_build_copy_kernel<PACK, size_t><<<grid, block, 0, st>>>(
                g, d_etas, e0, nb, ld, d_idx, d_nred, d_M, d_Mb, d_absmax, span, copy);
    } else if ((unsigned long long)g.ntau * (unsigned long long)g.cs_pitch < (1ull << 32)) {
        thth_build_kernel<PACK, unsigned><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                  d_nred, d_M, d_Mb, d_absmax, span);
    } else {
        thth_build_kernel<PACK, size_t><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                d_nred, d_M, d_Mb, d_absmax, span);
    }
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
