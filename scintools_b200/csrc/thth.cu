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

#include <type_traits>

#include "bf16_pack.cuh"
#include "lanczos.cuh"
#include "thth.cuh"
#include "tma.cuh"

namespace sb {

#ifndef SB_HOST_EMU
// eig_cluster.cu: on-chip (cluster shared memory) solver for ld <= 512
int eig_cluster_launch(const float2* d_M, int ld, int n_max, const int* d_nred, int e0,
                       int nb, double* d_eigs, int* d_status, int* d_iters, double tol,
                       double etol, int max_iter, cudaStream_t st);

// eig_half.cu: bf16 iteration + fp32 Rayleigh quotient (default for ld <= 512)
int eig_half_launch(const float2* d_M, const unsigned* d_Mb, int ld, const int* d_nred, int e0,
                    int nb, double* d_eigs, int* d_status, int* d_iters, double tol, double etol,
                    int max_iter, bool tensor, cudaStream_t st);

#endif  // SB_HOST_EMU

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
__global__ void cs_absmax_kernel(const float2* __restrict__ cs, long long rows, long long ncols,
                                 long long pitch, unsigned* __restrict__ out) {
    float m = 0.f;
    const long long per_row4 = ncols >> 1;          // float4 = two complex columns
    const long long total = rows * per_row4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / per_row4, c = i - r * per_row4;
        const float4 q = __ldg(reinterpret_cast<const float4*>(cs + r * pitch) + c);
        m = fmaxf(fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), fmaxf(fabsf(q.z), fabsf(q.w))), m);
    }
    if (ncols & 1) {                                 // odd tail column
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

// PACK: also write the fp16 copy Mb (re | im << 16) that eig_half.cu iterates on,
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
// ROWS rows of the tile per thread (block = 32 x 32/ROWS threads).  Per curvature the
// body runs in three phases -- (1) tau_inv and the CS offset of every row, (2) ALL the
// gathers back to back, (3) Jacobian, clean-up, stores -- so that ROWS independent
// L2 / DRAM gathers are in flight per thread: the kernel is bound by the latency of
// these random 8-byte loads (long-scoreboard stalls dominate with one load in flight),
// not by its instruction count.
// PACK == 2: the fp16 copy in the block layout of eig_half.cu's tensor-core mat-vec:
// 512-byte blocks of 16 rows x 8 columns, block (I, G) at ((I * ld / 8 + G) * 512) bytes,
// a block row = [re x 8 | im x 8] (the halves swapped in rows 4-7, 12-15); the part of a
// diagonal block on / below the diagonal is written as zeros (the MMA has no masks).
// ROWS == 4: three CTAs per SM (80 registers).  ptxas still spills at 80 registers, but
// less: 40-48 bytes of stores and 56-68 bytes of loads per thread in the PACK == 2
// instances on sm_90, against ~200 / ~150 bytes at four CTAs (64 registers), where the
// gather runs ~15 % slower on the headline sweep (H100 SXM, 400 W power limit: 2.8-2.9 ms
// instead of 2.4 ms per 1024-eta launch).
template <int PACK, int ROWS, typename OFF>
__global__ void __launch_bounds__(32 * (32 / ROWS), ROWS == 8 ? 5 : 3)
thth_build_kernel(ThthGeom g, const double* __restrict__ etas, int eta0, int nbatch,
                  int ld, const int* __restrict__ idx,
                  const int* __restrict__ nred, float2* __restrict__ M,
                  unsigned* __restrict__ Mb, const unsigned* __restrict__ absmax, float span) {
    // eta is the FAST grid index: CTAs resident at the same time work on the
    // same 32x32 tile for neighbouring curvatures, whose gathers fall on
    // the same / adjacent CS rows for small |theta1^2 - theta2^2| (L2 reuse)
    // pair index -> (ta <= tb)
    constexpr int TY = 32 / ROWS;
    int p = blockIdx.y, ta = 0;
    const int T = ld / 32;
    while (p >= T - ta) { p -= T - ta; ++ta; }
    const int tb = ta + p;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int b = tb * 32 + tx;
    const double ntau_d = (double)g.ntau;
    const long long hfd = g.nfd / 2;
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
                    const double bb = __dadd_rn(__dsub_rn(__dsub_rn(th1, th2), g.fd0), g.half_dfd);
                    const double fqd = floor_div_fast(bb, g.dfd, g.inv_dfd);
                    const long long fq = (fqd == fqd && fabs(fqd) < 9.0e18) ? (long long)fqd : LLONG_MIN;
                    wk[k] = sqrtf((float)fabs(th2 - th1));
                    if (fq < g.nfd && !(fq < -g.nfd)) {     // pnts mask / IndexError (thth_point)
                        const long long fi = fq < 0 ? fq + g.nfd : fq;
                        if (!g.cs_half) col[k] = (int)fi;
                        else if (fi >= hfd) col[k] = (int)(fi - hfd);
                        else if (fi == 0) col[k] = (int)hfd;
                        else { col[k] = (int)(hfd - fi); conj |= 1u << k; }   // CS[-tau,-fd] = conj(CS[tau,fd])
                    }
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
        // ---- phase 2: the gathers, all in flight together (a miss reads CS[0], ignored)
        float2 val[ROWS];
#pragma unroll
        for (int k = 0; k < ROWS; ++k) val[k] = __ldg(g.cs + off[k]);
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
                if (PACK == 1) Mb[(size_t)e * ld * ld + o] = pack_f16x2(make_float2(v.x * hscale, v.y * hscale));
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
// mat-vec).  TMA = true (ld <= 512): every row segment is fetched with one
// cp.async.bulk into a per-warp ring of NST 4 KB shared-memory stages
// (mbarrier complete_tx), so ~NST row fetches per warp are in flight while the
// warp does FMAs.  TMA = false: direct 16-byte loads, any ld, columns in
// chunks of 512.
template <int THREADS, bool TMA, int NST, bool FAST = false>
__global__ void __launch_bounds__(THREADS)
thth_eig_kernel(const float2* __restrict__ Mbase, int ld,
                const int* __restrict__ nred, int eta0,
                double* __restrict__ eigs, int* __restrict__ status,
                int* __restrict__ iters, double tol, double etol, int max_iter, int nb) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int NW = THREADS / 32;
    LanczosShared& S = *reinterpret_cast<LanczosShared*>(smem_raw);
    float2* v = reinterpret_cast<float2*>(smem_raw + sizeof(LanczosShared));
    float2* vp = v + ld;
    float2* w = vp + ld;          // row sums, then the new Lanczos vector
    float2* u = w + ld;           // column sums
    // TMA: [NW][NST][256] float4 stages, re-used as the column-partial scratch
    float4* stages = reinterpret_cast<float4*>(u + ld);
    float2* part = reinterpret_cast<float2*>(stages);   // [NW][512]
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(
        reinterpret_cast<unsigned char*>(stages) +
        (TMA ? (size_t)NW * NST * 4096 : (size_t)NW * 4096));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (TMA) {
        if (tid == 0) {
            for (int i = 0; i < NW * NST; ++i) mbar_init(mbar + i, 1);
            fence_mbarrier_init();
        }
    }
    unsigned gi = 0, gc = 0;             // ring producer / consumer counters
    // grid-stride over the curvatures: gridDim.x == nb (one CTA per eta) or a
    // persistent grid sized so that the matrices in flight stay L2-resident
    for (int e = blockIdx.x; e < nb; e += gridDim.x) {
    __syncthreads();                     // the previous eta is done with the shared buffers
    const int n = nred[eta0 + e];
    const float2* M = Mbase + (size_t)e * ld * ld;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);

    if (status[eta0 + e] & ST_INDEX_ERROR) {
        if (tid == 0) { eigs[eta0 + e] = qnan; iters[eta0 + e] = 0; }
        continue;
    }
    if (n < 3) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= ST_TOO_SMALL;
        }
        continue;
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
        S.done = 0; S.lo = 0.0; S.theta = 0.0; S.res = 0.0; S.m_lo2 = 0; S.lo2 = 0.0;
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
        continue;
    }
    {
        float s = (float)(1.0 / sqrt(nrm2));
        for (int c = tid; c < ld; c += THREADS) { v[c].x *= s; v[c].y *= s; }
    }
    __syncthreads();

    const int ncol4 = (n + 1) >> 1;      // float4 = two complex columns
    const int nchunk = (n + 511) / 512;  // column chunks of 512 (1 when TMA)
    float4* mystage = stages + (size_t)warp * NST * 256;
    unsigned long long* mybar = mbar + warp * NST;
    float beta_prev = 0.f;
    int m = 0;
    for (int it = 0; it < max_iter; ++it) {
        for (int c = tid; c < ld; c += THREADS) w[c] = make_float2(0.f, 0.f);
        __syncthreads();
        if constexpr (TMA) {
            // ---- single column chunk (ld <= 512).  Rows are grouped by JS =
            // number of 32-float4 column groups entirely left of the diagonal,
            // and the row body is specialised on JS (no per-group branches,
            // masks only on the boundary group); row sums use split
            // accumulators and one 5-step shuffle tree for (re, im) together.
            float4 yc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) yc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int K = (n - 2 >= warp) ? (n - 2 - warp) / NW + 1 : 0;
            const bool tail = ncol4 < 256;        // cropped matrix: mask the right edge too
            const float4* v4 = reinterpret_cast<const float4*>(v);
            // prologue: fill the ring
            for (int k = 0; k < NST && k < K; ++k) {
                const int st = gi % NST;
                ++gi;
                if (lane == 0) {
                    const int a = warp + NW * k;
                    const int c_lo = (a + 1) & ~1;
                    const unsigned bytes = (unsigned)(2 * ncol4 - c_lo) * 8u;
                    mbar_expect_tx(mybar + st, bytes);
                    bulk_g2s(reinterpret_cast<float2*>(mystage + st * 256) + c_lo,
                             M + (size_t)a * ld + c_lo, bytes, mybar + st);
                }
            }
            int k = 0;
            auto run_rows = [&](auto JSc) {
                constexpr int JS = decltype(JSc)::value;
                for (; k < K && ((warp + NW * k + 1) >> 6) == JS; ++k) {
                    const int a = warp + NW * k;
                    const int first4 = (a + 1) >> 1;
                    const float2 xa = v[a];
                    const int st = gc % NST;
                    const unsigned par = (gc / NST) & 1u;
                    ++gc;
                    while (!mbar_try_wait(mybar + st, par)) {}
                    const float4* sg = mystage + st * 256;
                    float rxa = 0.f, rxb = 0.f, rya = 0.f, ryb = 0.f;
#pragma unroll
                    for (int j = JS; j < 8; ++j) {
                        const int c4 = lane + 32 * j;
                        float4 q = sg[c4];
                        bool ok = (j > JS) || (c4 >= first4);
                        if (tail) ok = ok && (c4 < ncol4);
                        if (!ok) q = make_float4(0.f, 0.f, 0.f, 0.f);
                        // only the live columns are read: past ld the float4 would alias w / the
                        // other warps' stages (racecheck flags that even though it was discarded)
                        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (ok) x = v4[c4];
                        rxa = fmaf(q.x, x.x, rxa); rxb = fmaf(-q.y, x.y, rxb);
                        rxa = fmaf(q.z, x.z, rxa); rxb = fmaf(-q.w, x.w, rxb);
                        rya = fmaf(q.x, x.y, rya); ryb = fmaf(q.y, x.x, ryb);
                        rya = fmaf(q.z, x.w, rya); ryb = fmaf(q.w, x.z, ryb);
                        // conj(A) * v[a]
                        yc[j].x = fmaf(q.x, xa.x, yc[j].x); yc[j].x = fmaf(q.y, xa.y, yc[j].x);
                        yc[j].y = fmaf(q.x, xa.y, yc[j].y); yc[j].y = fmaf(-q.y, xa.x, yc[j].y);
                        yc[j].z = fmaf(q.z, xa.x, yc[j].z); yc[j].z = fmaf(q.w, xa.y, yc[j].z);
                        yc[j].w = fmaf(q.z, xa.y, yc[j].w); yc[j].w = fmaf(-q.w, xa.x, yc[j].w);
                    }
                    __syncwarp();
                    const bool more = k + NST < K;
                    const int st2 = gi % NST;   // == the stage just consumed
                    if (more) ++gi;
                    if (lane == 0 && more) {
                        const int a2 = warp + NW * (k + NST);
                        const int c_lo = (a2 + 1) & ~1;
                        const unsigned bytes = (unsigned)(2 * ncol4 - c_lo) * 8u;
                        mbar_expect_tx(mybar + st2, bytes);
                        bulk_g2s(reinterpret_cast<float2*>(mystage + st2 * 256) + c_lo,
                                 M + (size_t)a2 * ld + c_lo, bytes, mybar + st2);
                    }
                    // (re, im) reduced together: upper half-warp keeps im, lower re
                    const float rx = rxa + rxb, ry = rya + ryb;
                    const bool hi = lane & 16;
                    float keep = hi ? ry : rx;
                    keep += __shfl_xor_sync(0xffffffffu, hi ? rx : ry, 16);
                    keep += __shfl_xor_sync(0xffffffffu, keep, 8);
                    keep += __shfl_xor_sync(0xffffffffu, keep, 4);
                    keep += __shfl_xor_sync(0xffffffffu, keep, 2);
                    keep += __shfl_xor_sync(0xffffffffu, keep, 1);
                    if (lane == 0) w[a].x += keep;
                    if (lane == 16) w[a].y += keep;
                }
            };
            run_rows(std::integral_constant<int, 0>{});
            run_rows(std::integral_constant<int, 1>{});
            run_rows(std::integral_constant<int, 2>{});
            run_rows(std::integral_constant<int, 3>{});
            run_rows(std::integral_constant<int, 4>{});
            run_rows(std::integral_constant<int, 5>{});
            run_rows(std::integral_constant<int, 6>{});
            run_rows(std::integral_constant<int, 7>{});
            __syncthreads();   // every warp is done with its stages
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float4*>(part + warp * 512 + 2 * (lane + 32 * j)) = yc[j];
            __syncthreads();
            for (int c = tid; c < 512; c += THREADS) {
                float sx = 0.f, sy = 0.f;
#pragma unroll
                for (int kk = 0; kk < NW; ++kk) { sx += part[kk * 512 + c].x; sy += part[kk * 512 + c].y; }
                if (c < ld) u[c] = make_float2(sx, sy);
            }
            fence_proxy_async();
            __syncthreads();
        } else {
        for (int cb = 0; cb < nchunk; ++cb) {
            float4 yc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) yc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int chunk_end = min(n, (cb + 1) * 512);
            // rows a = warp + NW*k with a + 1 < chunk_end
            const int K = (chunk_end - 2 >= warp) ? (chunk_end - 2 - warp) / NW + 1 : 0;
            if (TMA) {
                // prologue: fill the ring
                for (int k = 0; k < NST && k < K; ++k) {
                    const int st = gi % NST;
                    ++gi;
                    if (lane == 0) {
                        const int a = warp + NW * k;
                        const int c_lo = (a + 1) & ~1;
                        const unsigned bytes = (unsigned)(2 * ncol4 - c_lo) * 8u;
                        mbar_expect_tx(mybar + st, bytes);
                        bulk_g2s(reinterpret_cast<float2*>(mystage + st * 256) + c_lo,
                                 M + (size_t)a * ld + c_lo, bytes, mybar + st);
                    }
                }
            }
            for (int k = 0; k < K; ++k) {
                const int a = warp + NW * k;
                const int first4 = (a + 1) >> 1;
                const float2 xa = v[a];
                float4 mm[8];
                if (TMA) {
                    const int st = gc % NST;
                    const unsigned par = (gc / NST) & 1u;
                    ++gc;
                    while (!mbar_try_wait(mybar + st, par)) {}
                    const float4* sg = mystage + st * 256;
                    // lane-local group range [jlo, jhi) that lies inside [first4, ncol4)
                    const int jlo = max(0, (first4 - lane + 31) >> 5);
                    const int jhi = (ncol4 - lane + 31) >> 5;
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        mm[j] = (j >= jlo && j < jhi) ? sg[lane + 32 * j]
                                                      : make_float4(0.f, 0.f, 0.f, 0.f);
                } else {
                    const float4* row = reinterpret_cast<const float4*>(M + (size_t)a * ld);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int c4 = cb * 256 + lane + 32 * j;
                        mm[j] = (c4 >= first4 && c4 < ncol4) ? __ldg(row + c4)
                                                             : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
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
                if (TMA) {
                    __syncwarp();
                    const bool more = k + NST < K;
                    const int st = gi % NST;   // == the stage just consumed
                    if (more) ++gi;
                    if (lane == 0 && more) {
                        const int a2 = warp + NW * (k + NST);
                        const int c_lo = (a2 + 1) & ~1;
                        const unsigned bytes = (unsigned)(2 * ncol4 - c_lo) * 8u;
                        mbar_expect_tx(mybar + st, bytes);
                        bulk_g2s(reinterpret_cast<float2*>(mystage + st * 256) + c_lo,
                                 M + (size_t)a2 * ld + c_lo, bytes, mybar + st);
                    }
                }
                rx = warp_sum(rx);
                ry = warp_sum(ry);
                if (lane == 0) { w[a].x += rx; w[a].y += ry; }
            }
            if (TMA) __syncthreads();   // every warp is done with its stages
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
            if (TMA) fence_proxy_async();
            __syncthreads();
        }
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
        if (warp == 0 && (m >= S.next_check || last || !(beta > 0.0))) {
            if (FAST) lanczos_check_fast(S, m, tol, etol);
            else lanczos_check(S, m, tol, etol);
        }
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
    }   // eta loop
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
// per-launch budget of the curvature-batched work buffers: 3 GiB, or SB_SWEEP_SLAB_MB
// (tests use it to force batching)
unsigned long long sweep_slab_bytes() {
    unsigned long long slab = 3ull << 30;
    if (const char* ev = getenv("SB_SWEEP_SLAB_MB")) {
        const long mb = atol(ev);
        if (mb > 0) slab = (unsigned long long)mb << 20;
    }
    return slab;
}

static bool lower_check_needed(const ThthGeom& g, const double* th_host) {
    // worst case fd argument over all (i, j): min(th) - max(th)
    double tmin = th_host[0], tmax = th_host[0];
    for (int k = 1; k < g.n; ++k) {
        tmin = th_host[k] < tmin ? th_host[k] : tmin;
        tmax = th_host[k] > tmax ? th_host[k] : tmax;
    }
    double worst = floor(((tmin - tmax) - g.fd0 + g.half_dfd) / g.dfd) - 2.0;
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

// fp32 strict upper triangles [nb][ld][ld] of etas e0 .. e0 + nb - 1 (no fp16 copy)
int thth_build_f32(const ThthGeom& g, const double* d_etas, int e0, int nb, int ld,
                   const int* d_idx, const int* d_nred, float2* d_M, cudaStream_t st) {
    const int T = ld / 32;
    dim3 grid((nb + SB_BUILD_EB - 1) / SB_BUILD_EB, T * (T + 1) / 2), block(32, 32 / 4);
    if ((unsigned long long)g.ntau * (unsigned long long)g.cs_pitch < (1ull << 32))
        thth_build_kernel<0, 4, unsigned><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                  d_nred, d_M, nullptr, nullptr, 0.f);
    else
        thth_build_kernel<0, 4, size_t><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx,
                                                                d_nred, d_M, nullptr, nullptr, 0.f);
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
    int* d_idx = (int*)workspace(1, (size_t)neta * ld * sizeof(int));
    if (!d_idx) return SB_ERR_NOMEM;
    int rc = thth_prep(g, th_host, d_etas, neta, ld, d_idx, d_nred, d_status, st);
    if (rc) return rc;
    // batch so that the matrix slab stays <= ~3 GiB
    const size_t per = (size_t)ld * ld * sizeof(float2);
    int batch = (int)(sweep_slab_bytes() / per);
    if (batch < 1) batch = 1;
    if (batch > neta) batch = neta;
    float2* d_M = (float2*)workspace(2, per * batch);
    if (!d_M) return SB_ERR_NOMEM;
    // default solver for ld <= 512 (eig_half.cu): iterates on the bf16 copy written by the
    // build kernel; SB_EIG_FP32=1 selects the fp32 streaming solver below instead
    const bool mixed = (ld <= 512) && !getenv("SB_EIG_FP32") && !getenv("SB_EIG_CLUSTER") &&
                       !getenv("SB_EIG_PERSIST") && !getenv("SB_EIG_NO_TMA");
    unsigned* d_Mb = nullptr;
    if (mixed) {
        d_Mb = (unsigned*)workspace(6, per / 2 * batch);
        if (!d_Mb) return SB_ERR_NOMEM;
    }
    const int T = ld / 32;
    const int npairs = T * (T + 1) / 2;
    // TMA ring variant (ld <= 512): 256 threads, 2 stages -> 2 CTAs per SM so
    // one CTA streams while the other is in its serial Lanczos bookkeeping
    constexpr int TT = 256, TS = 2;      // TMA: threads, stages
    constexpr int DT = 512;              // direct-load variant
    const bool use_tma = (ld <= 512) && !getenv("SB_EIG_NO_TMA");
    const size_t smem = sizeof(LanczosShared) + 4 * (size_t)ld * sizeof(float2) +
                        (use_tma ? (size_t)(TT / 32) * TS * 4096 + 512
                                 : (size_t)(DT / 32) * 4096 + 512);
    // SB_EIG_PERSIST=N: N persistent CTAs (1 per SM, 4-stage ring) walk the curvatures,
    // so that only N matrices (N MB) are in flight and re-reads hit the L2
    int persist = 0;
    if (const char* ev = getenv("SB_EIG_PERSIST")) persist = atoi(ev);
    constexpr int PS = 4;
    const size_t smem_p = sizeof(LanczosShared) + 4 * (size_t)ld * sizeof(float2) +
                          (size_t)(TT / 32) * PS * 4096 + 512;
    if (use_tma && persist > 0)
        SB_CUDA(cudaFuncSetAttribute(thth_eig_kernel<TT, true, PS, true>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_p));
    if (use_tma)
        SB_CUDA(cudaFuncSetAttribute(thth_eig_kernel<TT, true, TS>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    else
        SB_CUDA(cudaFuncSetAttribute(thth_eig_kernel<DT, false, 1>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // scale of the fp16 copy: max |CS| over what the gather can reach, max |theta2 - theta1|
    unsigned* d_absmax = nullptr;
    float span = 0.f;
    if (mixed) {
        d_absmax = (unsigned*)workspace(0, 64 * sizeof(double)) + 32;   // behind the dynspec stats
        if (!d_absmax) return SB_ERR_NOMEM;
        if (g.cs_bound) {       // the caller knows a bound (sb_cs_bound_f32): no scan
            SB_CUDA(cudaMemcpyAsync(d_absmax, g.cs_bound, sizeof(float), cudaMemcpyDeviceToDevice, st));
        } else {
            SB_CUDA(cudaMemsetAsync(d_absmax, 0, sizeof(unsigned), st));
            const long long ncols = g.cs_half ? (g.cs_valid_cols > 0 ? g.cs_valid_cols : g.nfd / 2 + 1)
                                              : g.nfd;
            cs_absmax_kernel<<<num_sms() * 8, 256, 0, st>>>(g.cs, g.ntau, ncols, g.cs_pitch, d_absmax);
            SB_LAUNCH_CHECK();
        }
        double tmin = th_host[0], tmax = th_host[0];
        for (int k = 1; k < g.n; ++k) {
            tmin = th_host[k] < tmin ? th_host[k] : tmin;
            tmax = th_host[k] > tmax ? th_host[k] : tmax;
        }
        span = (float)((tmax - tmin) * 1.0001);
    }
    for (int e0 = 0; e0 < neta; e0 += batch) {
        int nb = neta - e0 < batch ? neta - e0 : batch;
        // rows per thread of thth_build_kernel: 4 (default) or 8 (SB_BUILD_ROWS=8; slower: the
        // gather is bound by random DRAM sector reads, not by the number of loads a thread keeps
        // in flight)
        static const int BR = (getenv("SB_BUILD_ROWS") && atoi(getenv("SB_BUILD_ROWS")) == 8) ? 8 : 4;
        // tensor-core mat-vec of the default solver (block layout of the fp16 copy);
        // SB_EIG_NO_TC=1: the FMA mat-vec on the row-major copy
        const bool tensor = mixed && BR == 4 && !getenv("SB_EIG_NO_TC");
        dim3 grid((nb + SB_BUILD_EB - 1) / SB_BUILD_EB, npairs), block(32, 32 / BR);
        prof_begin(PROF_THTH_BUILD, st);
        // 32-bit CS offsets whenever the spectrum has fewer than 2^32 elements
        const bool small = (unsigned long long)g.ntau * (unsigned long long)g.cs_pitch < (1ull << 32);
#define SB_BUILD_LAUNCH(PACK, ROWS, OFF, MB, AM, SP)                                        \
        thth_build_kernel<PACK, ROWS, OFF><<<grid, block, 0, st>>>(g, d_etas, e0, nb, ld, d_idx, \
                                                                   d_nred, d_M, MB, AM, SP)
        if (BR == 8) {
            if (mixed && small) SB_BUILD_LAUNCH(1, 8, unsigned, d_Mb, d_absmax, span);
            else if (mixed) SB_BUILD_LAUNCH(1, 8, size_t, d_Mb, d_absmax, span);
            else if (small) SB_BUILD_LAUNCH(0, 8, unsigned, nullptr, nullptr, 0.f);
            else SB_BUILD_LAUNCH(0, 8, size_t, nullptr, nullptr, 0.f);
        } else if (tensor) {
            if (small) SB_BUILD_LAUNCH(2, 4, unsigned, d_Mb, d_absmax, span);
            else SB_BUILD_LAUNCH(2, 4, size_t, d_Mb, d_absmax, span);
        } else {
            if (mixed && small) SB_BUILD_LAUNCH(1, 4, unsigned, d_Mb, d_absmax, span);
            else if (mixed) SB_BUILD_LAUNCH(1, 4, size_t, d_Mb, d_absmax, span);
            else if (small) SB_BUILD_LAUNCH(0, 4, unsigned, nullptr, nullptr, 0.f);
            else SB_BUILD_LAUNCH(0, 4, size_t, nullptr, nullptr, 0.f);
        }
#undef SB_BUILD_LAUNCH
        prof_end(PROF_THTH_BUILD, st);
        SB_LAUNCH_CHECK();
        prof_begin(PROF_THTH_EIG, st);
        // experimental solvers, each enabled by its own environment variable
        int rc = mixed ? eig_half_launch(d_M, d_Mb, ld, d_nred, e0, nb, d_eigs, d_status,
                                         d_iters, tol, 2e-7, max_iter, tensor, st)
                       : 0;
        if (rc == 0)
            rc = eig_cluster_launch(d_M, ld, g.n, d_nred, e0, nb, d_eigs, d_status, d_iters,
                                    tol, 2e-7, max_iter, st);
        if (rc < 0) return rc;
        if (rc > 0) {
            // handled by eig_half.cu / eig_cluster.cu
        } else if (use_tma && persist > 0)
            thth_eig_kernel<TT, true, PS, true><<<persist < nb ? persist : nb, TT, smem_p, st>>>(
                d_M, ld, d_nred, e0, d_eigs, d_status, d_iters, tol, 2e-7, max_iter, nb);
        else if (use_tma)
            thth_eig_kernel<TT, true, TS><<<nb, TT, smem, st>>>(
                d_M, ld, d_nred, e0, d_eigs, d_status, d_iters, tol, 2e-7, max_iter, nb);
        else
            thth_eig_kernel<DT, false, 1><<<nb, DT, smem, st>>>(
                d_M, ld, d_nred, e0, d_eigs, d_status, d_iters, tol, 2e-7, max_iter, nb);
        prof_end(PROF_THTH_EIG, st);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
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
