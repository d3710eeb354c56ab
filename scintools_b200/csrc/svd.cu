// Flux-variation correction behind Dynspec.correct_dyn / ththmod.svd_model
// (include/scint_b200.h, sb_svd_* and sb_bandpass_*).
//
// svd=True.  The rank-k model of a real float32 nf x nt matrix A is A V_k V_k^T, V_k the top
// k right singular vectors.  They come from Lanczos on B = A^T A with vectors of length nt in
// float64 and full re-orthogonalisation (classical Gram-Schmidt, twice) against every
// previous Lanczos vector:
//  - one step is one HBM read of A: svd_gram_kernel streams whole rows, forms a_i . x and
//    adds a_i (a_i . x) into CTA-private float64 column partials held in registers; CTA b
//    always takes rows b, b + G, b + 2G, ...; svd_reduce_kernel adds the G partials of each
//    column in CTA order.  No floating-point atomics anywhere, so repeated calls are
//    bit-identical.
//  - the m x m tridiagonal T_m (alpha, beta) is copied to the host at checks and solved
//    there by implicit QL (svd_tridiag_ql) in float64; the host decides when to stop.
//  - svd_apply_kernel is the final pass: per row, one read of a_i gives the k projections
//    p_j = a_i . v_j (u_j s_j is never formed), the model row sum_j p_j v_j and a_i / |model|.
//
// Accuracy.  Narrowing the input to float32 is a perturbation E with ||E||_2 <= u ||A||_F
// (u = 2^-24); by Weyl every singular value moves by at most that.  Past the narrowing all
// arithmetic is float64: a float32 element times a float64 vector entry is one float64
// rounding, so the mat-vec B x carries a relative error of order eps_64 (sqrt(nt) +
// sqrt(nf)) ~ 1e-13 at the envelope's corner.  Squaring the spectrum is harmless for the
// modes the solver returns: an eigenvalue error dl <= rho (the true residual, accepted at
// <= 1e-11 lambda_1) moves s_j by dl / (2 s_j) <= 5e-12 s_1^2 / s_j, which stays below the
// narrowing's u s_1 for every s_j >= 1e-4 s_1.  Modes below that ratio are still returned;
// their share of the model is at most s_j, i.e. of the order of the narrowing itself.
//
// Breakdown and restarts.  When the new Lanczos vector's norm beta_{m+1} falls to <= 1e-12
// max_j alpha_j (<= 1e-12 theta_1) the Krylov space is invariant to round-off.  Eigenvalues
// its start vector never touched -- a second copy of a repeated singular value, say -- are
// not in it, so the iteration does not stop there: beta_{m+1} is recorded as 0 (T_m splits)
// and svd_restart_kernel continues from a fresh pseudo-random vector orthogonal to every
// previous one.  The model is exact (numerical rank <= the Ritz pairs found) once a restart
// vector q itself gives B q ~ 0: two recorded zeros in a row with alpha ~ 0 between them
// (the zero matrix after one step, a constant matrix after two), or when m reaches nt.
//
// Stopping rule (at a check after m steps; theta_1 >= theta_2 >= ... the Ritz values, r_j =
// |beta_{m+1}| |z_{m,j}| the Lanczos residual estimate of pair j, z_j the eigenvector of
// T_m; never right after a restart, which makes every r_j read 0):
//  - values: max_{j<=k} r_j <= 1e-12 theta_1.  By Weyl (Kahan's residual bound) an
//    eigenvalue of B lies within r_j of theta_j; by Cauchy interlacing theta_j <= lambda_j.
//  - next value: r_{k+1} <= 1e-8 theta_1, so that theta_{k+1} + r_{k+1} is an upper
//    estimate of lambda_{k+1} and not of some lower eigenvalue theta_{k+1} is still moving
//    past (the Ritz values interlace from below: theta_{k+1} alone under-states
//    lambda_{k+1} and over-states the gap).  After a restart the earlier blocks' Ritz pairs
//    all read r = 0, so the top Ritz value of the current block must also have r <= 1e-8
//    theta_1: until then a value the restart is still lifting (the second copy of a
//    repeated singular value) may belong above theta_k.
//  - gap: the model is only defined when lambda_k > lambda_{k+1}; the rule's lower bound is
//    delta = theta_k - theta_{k+1} - r_{k+1} > 0.  (Lanczos sees only what its start
//    vectors touch; they have pseudo-random entries in every coordinate, so delta is the
//    bound Lanczos practice uses, not a certificate against an eigenvector orthogonal to
//    all of them.)
//  - model: Davis-Kahan bounds the Ritz subspace's angle by sin(Theta) <= ||R_k||_F / delta
//    <= sqrt(k) 1e-12 theta_1 / delta, and Wedin turns an angle into ||M~ - M||_2 <=
//    sqrt(2) s_1 sin(Theta).  The narrowing alone moves B by up to 2 u s_1 ||A||_F >= 2 u
//    theta_1 and the subspace by up to that over delta, so the solver's share stays below
//    1e-4 sqrt(k) of the narrowing's whatever the gap: delta > 0 is all the rule needs.
//  - tie: when theta_k - theta_{k+1} <= 2 u theta_1 -- a gap the float32 narrowing alone
//    can close -- the truncation is not defined by the data.  Stop and report it (info:
//    tie, not converged); the caller warns.  The exact exits above report ties the same
//    way.  A tail of zeros (theta_{k+1} + r_{k+1} <= 1e-12 theta_1) is the exact model.
//  - at SVD_MAXIT steps: stop, not converged.
// Converged only if the rule stopped on the exact model or on values + gap AND the final
// true-residual pass confirms every returned pair: rho_j = ||B y_j - theta_j y_j||_2, one
// more read of A per mode, <= 1e-11 theta_1.  Numerical trouble (a QL sweep that fails, a
// NaN anywhere) never reads as converged.
//
// svd=False.  bandpass_row_kernel: row NaN-means; bandpass_col_kernel + _reduce: column
// NaN-means of the row quotient; bandpass_divide_kernel: the final division.  Which zeros
// count as NaN is the host's decision (zero_as_nan); the kernels treat NaN as 0 on load.
#include <float.h>
#include <math.h>

#ifndef SB_HOST_EMU
#include <algorithm>
#include <cmath>
#include <vector>
#endif

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int SVD_THREADS = 512;       // gram / apply CTA; a row is at most 32 values per thread
constexpr int SVD_MAX_MODES = 32;
constexpr int SVD_MAXIT = 384;
constexpr int SVD_MAX_NF = 32768;
constexpr int SVD_MAX_NT = 16384;     // = SVD_THREADS * 32 columns per thread
constexpr int SVD_RED_THREADS = 256;
constexpr int BP_THREADS = 256;

__device__ __forceinline__ float svd_load(const float* p) {
    const float v = *p;
    return isnan(v) ? 0.0f : v;
}

// Sum over the block in a fixed order (warp shuffles, then warps 0, 1, ... in turn); every
// thread gets the sum.  red is one half of a [2][32] buffer: callers alternate halves, so
// one barrier per call suffices.
__device__ __forceinline__ double svd_block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    if (lane == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < nw; ++i) s += red[i];
    return s;
}

// Asynchronous 4-byte global -> shared copy (cp.async), its commit and wait; plain copies
// under tests/host_emu.
__device__ __forceinline__ void svd_copy_async(float* dst, const float* src) {
#ifdef SB_HOST_EMU
    *dst = *src;
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(src) : "memory");
#endif
}
__device__ __forceinline__ void svd_copy_commit() {
#ifndef SB_HOST_EMU
    asm volatile("cp.async.commit_group;\n" ::: "memory");
#endif
}
__device__ __forceinline__ void svd_copy_wait_prev() {     // all but the newest group done
#ifndef SB_HOST_EMU
    asm volatile("cp.async.wait_group 1;\n" ::: "memory");
#endif
}

// part[b][j] = sum over rows i = b, b + G, ... of a_ij (a_i . x).  Thread t owns columns
// t + SVD_THREADS c (c < C); x sits in shared memory, the partials in registers, and the
// row in shared memory between its dot product and its update.  A block waits on that row,
// so up to C = 16 the next row is copied into a second buffer (cp.async) while the current
// one is reduced and applied, and up to C = 8 two blocks share an SM.  At C = 32 the
// partials fill the registers and x and one row the shared memory of one block: no
// prefetch.  Every thread copies and reads back only its own entries, so the buffers need
// no barrier.
template <int C>
__global__ void __launch_bounds__(SVD_THREADS, C <= 8 ? 2 : 1)
svd_gram_kernel(const float* __restrict__ A, int nf, int nt, const double* __restrict__ x,
                double* __restrict__ part) {
    constexpr bool PIPE = C <= 16;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* xs = reinterpret_cast<double*>(smem_raw);
    float* as = reinterpret_cast<float*>(xs + C * SVD_THREADS);     // 2 rows (PIPE) or 1
    SB_SHARED double red[2][32];
    const int t = threadIdx.x;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int j = t + SVD_THREADS * c;
        xs[j] = j < nt ? x[j] : 0.0;
    }
    double y[C];
#pragma unroll
    for (int c = 0; c < C; ++c) y[c] = 0.0;
    int par = 0;
    if (PIPE && blockIdx.x < nf) {
        const float* row = A + (long long)blockIdx.x * nt;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int j = t + SVD_THREADS * c;
            if (j < nt) svd_copy_async(as + j, row + j);
        }
    }
    svd_copy_commit();
    for (long long i = blockIdx.x; i < nf; i += gridDim.x) {
        float* cur = as + (PIPE ? par : 0) * C * SVD_THREADS;
        if (PIPE) {
            float* nxt = as + (par ^ 1) * C * SVD_THREADS;
            if (i + gridDim.x < nf) {
                const float* row = A + (i + gridDim.x) * nt;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    const int j = t + SVD_THREADS * c;
                    if (j < nt) svd_copy_async(nxt + j, row + j);
                }
            }
            svd_copy_commit();
            svd_copy_wait_prev();
        }
        const float* row = A + i * nt;
        double d = 0.0;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int j = t + SVD_THREADS * c;
            float v = 0.0f;
            if (j < nt) v = PIPE ? cur[j] : svd_load(row + j);
            if (isnan(v)) v = 0.0f;
            cur[j] = v;
            d += (double)v * xs[j];
        }
        d = svd_block_sum(d, red[par]);
        par ^= 1;
#pragma unroll
        for (int c = 0; c < C; ++c) y[c] += (double)cur[t + SVD_THREADS * c] * d;
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int j = t + SVD_THREADS * c;
        if (j < nt) part[(long long)blockIdx.x * nt + j] = y[c];
    }
}

// y[j] = sum_b part[b][j], b in order
__global__ void svd_reduce_kernel(const double* __restrict__ part, int nparts, int nt,
                                  double* __restrict__ y) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int b = 0; b < nparts; ++b) s += part[(long long)b * nt + j];
        y[j] = s;
    }
}

// h[q] = V[q] . w for q < nq, one block per q
__global__ void svd_dots_kernel(const double* __restrict__ V, int nq, int nt,
                                const double* __restrict__ w, double* __restrict__ h) {
    SB_SHARED double red[2][32];
    int par = 0;
    for (int q = blockIdx.x; q < nq; q += gridDim.x) {
        const double* v = V + (long long)q * nt;
        double s = 0.0;
        for (int j = threadIdx.x; j < nt; j += blockDim.x) s += v[j] * w[j];
        s = svd_block_sum(s, red[par]);
        par ^= 1;
        if (threadIdx.x == 0) h[q] = s;
    }
}

// w[j] -= sum_q h[q] V[q][j], q in order
__global__ void svd_orth_kernel(const double* __restrict__ V, int nq, int nt,
                                const double* __restrict__ h, double* __restrict__ w) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
        double s = w[j];
        for (int q = 0; q < nq; ++q) s -= h[q] * V[(long long)q * nt + j];
        w[j] = s;
    }
}

// One block.  Without h1 (the start vector): *nrm = ||w||_2, *amax = 0.  With h1 (step m):
// alpha[m] = h1[m] + h2[m] (the Rayleigh quotient v_m^T B v_m and its re-orthogonalisation
// correction), *amax = max(*amax, alpha[m]), and *nrm = ||w||_2 unless that is <= 1e-12
// *amax (breakdown, NaN included): then *nrm = 0 and *restart = 1.
__global__ void svd_norm_kernel(const double* __restrict__ w, int nt, double* __restrict__ nrm,
                                int m, const double* __restrict__ h1, const double* __restrict__ h2,
                                double* __restrict__ alpha, double* __restrict__ amax,
                                int* __restrict__ restart) {
    SB_SHARED double red[2][32];
    double s = 0.0;
    for (int j = threadIdx.x; j < nt; j += blockDim.x) s += w[j] * w[j];
    s = svd_block_sum(s, red[0]);
    if (threadIdx.x == 0) {
        s = sqrt(s);
        int r = 0;
        if (h1) {
            const double a = h1[m] + h2[m];
            alpha[m] = a;
            const double am = fmax(*amax, a);
            *amax = am;
            r = !(s > 1e-12 * am);
        } else {
            *amax = 0.0;
        }
        *nrm = r ? 0.0 : s;
        *restart = r;
    }
}

// v = w / nrm, unless a restart is due (svd_restart_kernel writes v then)
__global__ void svd_scale_kernel(const double* __restrict__ w, int nt, const double* __restrict__ nrm,
                                 const int* __restrict__ restart, double* __restrict__ v) {
    if (*restart) return;
    const double b = *nrm;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x)
        v[j] = w[j] / b;
}

// pseudo-random entry j of start vector `seed` in [-0.5, 0.5) (splitmix64): no coordinate
// is left out, and every call starts from the same vectors
__device__ __forceinline__ double svd_random(int seed, int j) {
    unsigned long long z = ((unsigned long long)seed << 32 | (unsigned)j) * 0x9e3779b97f4a7c15ull +
                           0x632be59bd9b4e019ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
}

__global__ void svd_start_kernel(int nt, double* __restrict__ w) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x)
        w[j] = svd_random(0, j);
}

// One block, only when *restart: v = start vector nq, orthogonalised twice against V[0..nq)
// and normalised (0 if nothing is left: nq = nt).  Thread t owns entries t + blockDim c.
__global__ void svd_restart_kernel(const int* __restrict__ restart, const double* __restrict__ V,
                                   int nq, int nt, double* __restrict__ v) {
    if (!*restart) return;
    SB_SHARED double red[2][32];
    int par = 0;
    for (int j = threadIdx.x; j < nt; j += blockDim.x) v[j] = svd_random(nq, j);
    for (int pass = 0; pass < 2; ++pass) {
        for (int q = 0; q < nq; ++q) {
            const double* u = V + (long long)q * nt;
            double s = 0.0;
            for (int j = threadIdx.x; j < nt; j += blockDim.x) s += u[j] * v[j];
            s = svd_block_sum(s, red[par]);
            par ^= 1;
            for (int j = threadIdx.x; j < nt; j += blockDim.x) v[j] -= s * u[j];
        }
    }
    double s = 0.0;
    for (int j = threadIdx.x; j < nt; j += blockDim.x) s += v[j] * v[j];
    s = sqrt(svd_block_sum(s, red[par]));
    const double f = s > 1e-8 ? 1.0 / s : 0.0;       // entries are O(1): 1e-8 is round-off
    for (int j = threadIdx.x; j < nt; j += blockDim.x) v[j] *= f;
}

// Ritz vectors Y[j] = sum_q S[q][j] V[q] for j < kk (S is m x kk), zero for kk <= j < k
__global__ void svd_ritz_kernel(const double* __restrict__ V, int m, int nt,
                                const double* __restrict__ S, int kk, int k,
                                double* __restrict__ Y) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
        for (int r = 0; r < k; ++r) {
            double s = 0.0;
            if (r < kk)
                for (int q = 0; q < m; ++q) s += S[q * kk + r] * V[(long long)q * nt + j];
            Y[(long long)r * nt + j] = s;
        }
    }
}

// One block: *res = ||w - theta y||_2
__global__ void svd_resid_kernel(const double* __restrict__ w, const double* __restrict__ y,
                                 double theta, int nt, double* __restrict__ res) {
    SB_SHARED double red[2][32];
    double s = 0.0;
    for (int j = threadIdx.x; j < nt; j += blockDim.x) {
        const double r = w[j] - theta * y[j];
        s += r * r;
    }
    s = svd_block_sum(s, red[0]);
    if (threadIdx.x == 0) *res = sqrt(s);
}

// Final pass, one row at a time per block: p_q = a_i . Y[q] (q < k), model m_ij = sum_q p_q
// Y[q][j], out_ij = a_ij / |m_ij| (float64, rounded once; 0/0 = NaN and a/0 = inf as in
// numpy); model (float32) when not NULL, out skipped when NULL.
// The row is parked as in svd_gram_kernel.
template <int C>
__global__ void __launch_bounds__(SVD_THREADS, 1)
svd_apply_kernel(const float* __restrict__ A, int nf, int nt, int k, const double* __restrict__ Y,
                 float* __restrict__ out, float* __restrict__ model) {
    constexpr bool STAGE = C > 16;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* as = reinterpret_cast<float*>(smem_raw);                  // STAGE only
    SB_SHARED double red[2][32];
    SB_SHARED double p_s[SVD_MAX_MODES];
    const int t = threadIdx.x;
    int par = 0;
    for (long long i = blockIdx.x; i < nf; i += gridDim.x) {
        const float* row = A + i * nt;
        float a[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int j = t + SVD_THREADS * c;
            const float v = j < nt ? svd_load(row + j) : 0.0f;
            if (STAGE) as[j] = v;
            else a[c] = v;
        }
        for (int q = 0; q < k; ++q) {
            const double* y = Y + (long long)q * nt;
            double d = 0.0;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const int j = t + SVD_THREADS * c;
                if (j < nt) d += (double)(STAGE ? as[j] : a[c]) * y[j];
            }
            d = svd_block_sum(d, red[par]);
            par ^= 1;
            if (t == 0) p_s[q] = d;
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int j = t + SVD_THREADS * c;
            if (j < nt) {
                double mv = 0.0;
                for (int q = 0; q < k; ++q) mv += p_s[q] * Y[(long long)q * nt + j];
                const double av = STAGE ? as[j] : a[c];
                if (out) out[i * nt + j] = (float)(av / fabs(mv));
                if (model) model[i * nt + j] = (float)mv;
            }
        }
    }
}

// ---- bandpass (svd=False) ----------------------------------------------------

__device__ __forceinline__ double bp_value(float v, int zero_as_nan) {
    if (isnan(v)) v = 0.0f;
    return (zero_as_nan && v == 0.0f) ? (double)NAN : (double)v;
}

// mean[i] = numpy nanmean of row i (NaN for a row without values)
__global__ void bandpass_row_kernel(const float* __restrict__ A, int nf, int nt, int zero_as_nan,
                                    double* __restrict__ mean) {
    SB_SHARED double red[2][32];
    int par = 0;
    for (long long i = blockIdx.x; i < nf; i += gridDim.x) {
        const float* row = A + i * nt;
        double s = 0.0, n = 0.0;
        for (int j = threadIdx.x; j < nt; j += blockDim.x) {
            const double v = bp_value(row[j], zero_as_nan);
            if (!isnan(v)) { s += v; n += 1.0; }
        }
        s = svd_block_sum(s, red[par]);
        par ^= 1;
        n = svd_block_sum(n, red[par]);
        par ^= 1;
        if (threadIdx.x == 0) mean[i] = n > 0.0 ? s / n : (double)NAN;
    }
}

// Column partial sums and counts of v_ij = value / rowdiv[i] (rowdiv NULL: value) over the
// rows of chunk blockIdx.y, NaN quotients skipped.
__global__ void bandpass_col_kernel(const float* __restrict__ A, int nf, int nt, int zero_as_nan,
                                    const double* __restrict__ rowdiv, int rows_per,
                                    double* __restrict__ psum, double* __restrict__ pcnt) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nt) return;
    const long long i0 = (long long)blockIdx.y * rows_per;
    const long long i1 = i0 + rows_per < nf ? i0 + rows_per : nf;
    double s = 0.0, n = 0.0;
    for (long long i = i0; i < i1; ++i) {
        double v = bp_value(A[i * nt + j], zero_as_nan);
        if (rowdiv) v = v / rowdiv[i];
        if (!isnan(v)) { s += v; n += 1.0; }
    }
    psum[(long long)blockIdx.y * nt + j] = s;
    pcnt[(long long)blockIdx.y * nt + j] = n;
}

__global__ void bandpass_col_reduce_kernel(const double* __restrict__ psum,
                                           const double* __restrict__ pcnt, int nchunk, int nt,
                                           double* __restrict__ mean) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
        double s = 0.0, n = 0.0;
        for (int b = 0; b < nchunk; ++b) {
            s += psum[(long long)b * nt + j];
            n += pcnt[(long long)b * nt + j];
        }
        mean[j] = n > 0.0 ? s / n : (double)NAN;
    }
}

// out_ij = (value / rowdiv[i]) / coldiv[j] in float64, rounded once (either divisor NULL: skipped)
__global__ void bandpass_divide_kernel(const float* __restrict__ A, int nf, int nt, int zero_as_nan,
                                       const double* __restrict__ rowdiv,
                                       const double* __restrict__ coldiv, float* __restrict__ out) {
    const long long n = (long long)nf * nt;
    for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < n;
         x += (long long)gridDim.x * blockDim.x) {
        const long long i = x / nt;
        const int j = (int)(x - i * nt);
        double v = bp_value(A[x], zero_as_nan);
        if (rowdiv) v = v / rowdiv[i];
        if (coldiv) v = v / coldiv[j];
        out[x] = (float)v;
    }
}

// Eigenvalues d[0..n) of the symmetric tridiagonal with diagonal d and off-diagonal e (e[i]
// couples i and i+1; destroyed) by implicit QL with Wilkinson shifts, and Z <- Z Q for the nz
// rows of Z (row-major, n columns): Z = I gives the eigenvectors as columns, Z = e_{n-1}^T
// their last components.  Returns -1 if an eigenvalue needs more than 64 sweeps.
inline int svd_tridiag_ql(int n, double* d, double* e, double* Z, int nz) {
    if (n > 0) e[n - 1] = 0.0;
    for (int l = 0; l < n; ++l) {
        for (int it = 0;; ++it) {
            int m = l;
            for (; m < n - 1; ++m)
                if (fabs(e[m]) <= DBL_EPSILON * (fabs(d[m]) + fabs(d[m + 1]))) break;
            if (m == l) break;
            if (it == 64) return -1;
            double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
            double r = hypot(g, 1.0);
            g = d[m] - d[l] + e[l] / (g + copysign(r, g));
            double s = 1.0, c = 1.0, p = 0.0;
            bool split = false;
            for (int i = m - 1; i >= l; --i) {
                double f = s * e[i];
                const double b = c * e[i];
                r = hypot(f, g);
                e[i + 1] = r;
                if (r == 0.0) {          // exact deflation inside the sweep
                    d[i + 1] -= p;
                    e[m] = 0.0;
                    split = true;
                    break;
                }
                s = f / r;
                c = g / r;
                g = d[i + 1] - p;
                r = (d[i] - g) * s + 2.0 * c * b;
                p = s * r;
                d[i + 1] = g + p;
                g = c * r - b;
                for (int q = 0; q < nz; ++q) {
                    double* z = Z + (size_t)q * n;
                    f = z[i + 1];
                    z[i + 1] = s * z[i] + c * f;
                    z[i] = c * z[i] - s * f;
                }
            }
            if (split) continue;
            d[l] -= p;
            e[l] = g;
            e[m] = 0.0;
        }
    }
    return 0;
}

#ifndef SB_HOST_EMU

static int svd_shape(const char* who, int nf, int nt) {
    SB_ARG(nf >= 1 && nt >= 1);
    if (nf > SVD_MAX_NF || nt > SVD_MAX_NT) {
        set_error("%s: %d x %d is outside the supported shapes (nf <= %d, nt <= %d)", who, nf, nt,
                  SVD_MAX_NF, SVD_MAX_NT);
        return SB_ERR_UNSUPPORTED;
    }
    return SB_OK;
}

static unsigned svd_grid(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    const long long cap = (long long)num_sms() * 8;
    return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

template <int C>
static size_t svd_gram_smem() {
    return (size_t)C * SVD_THREADS * (sizeof(double) + (C <= 16 ? 2 : 1) * sizeof(float));
}

template <int C>
static int svd_gram_launch(const float* A, int nf, int nt, const double* x, double* part, int G,
                           cudaStream_t st) {
    const size_t smem = svd_gram_smem<C>();
    svd_gram_kernel<C><<<G, SVD_THREADS, smem, st>>>(A, nf, nt, x, part);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

template <int C>
static int svd_gram_blocks(int nf) {
    const size_t smem = svd_gram_smem<C>();
    if (cudaFuncSetAttribute(svd_gram_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem) != cudaSuccess)
        return -1;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, svd_gram_kernel<C>, SVD_THREADS,
                                                      smem) != cudaSuccess || per_sm < 1)
        return -1;
    const long long G = (long long)num_sms() * per_sm;
    return (int)(G < nf ? G : nf);
}

static int svd_cols(int nt) {
    int C = 1;
    while (C * SVD_THREADS < nt) C *= 2;
    return C;
}

#define SVD_DISPATCH(C, call)                                   \
    switch (C) {                                                \
    case 1: call(1); break;                                     \
    case 2: call(2); break;                                     \
    case 4: call(4); break;                                     \
    case 8: call(8); break;                                     \
    case 16: call(16); break;                                   \
    default: call(32); break;                                   \
    }

// grid size of the gram pass: the CTAs the device holds at once, at most one per row
static int svd_gram_grid(int nf, int nt) {
    int G = -1;
#define SVD_G(C) G = svd_gram_blocks<C>(nf)
    SVD_DISPATCH(svd_cols(nt), SVD_G)
#undef SVD_G
    return G;
}

// w = B x = A^T (A x): one read of A
static int svd_matvec(const float* A, int nf, int nt, int G, const double* x, double* part,
                      double* w, cudaStream_t st) {
    ProfScope prof(PROF_SVD_GRAM, st);
    int rc = SB_OK;
#define SVD_L(C) rc = svd_gram_launch<C>(A, nf, nt, x, part, G, st)
    SVD_DISPATCH(svd_cols(nt), SVD_L)
#undef SVD_L
    if (rc) return rc;
    svd_reduce_kernel<<<svd_grid(nt, 256), 256, 0, st>>>(part, G, nt, w);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int svd_topk(const float* A, int nf, int nt, int k, double* Y, double* s_host, double* res_host,
             double* gap_host, int* info_host, cudaStream_t st) {
    int rc = svd_shape("sb_svd_topk", nf, nt);
    if (rc) return rc;
    SB_ARG(A && Y && s_host && res_host && gap_host && info_host);
    SB_ARG(k >= 1 && k <= SVD_MAX_MODES);
    const int maxit = nt < SVD_MAXIT ? nt : SVD_MAXIT;
    const int G = svd_gram_grid(nf, nt);
    if (G < 1) {
        set_error("sb_svd_topk: no launch configuration for nt = %d", nt);
        return SB_ERR_CUDA;
    }
    double* part = (double*)workspace(WS_TABLE, (size_t)G * nt * sizeof(double));
    if (!part) return SB_ERR_NOMEM;
    const size_t nV = (size_t)(maxit + 1) * nt;
    const size_t nsmall = nt + 2 * (size_t)(maxit + 1) + (maxit + 1) + (maxit + 2) +
                          (size_t)maxit * k + k + 2;
    double* V = (double*)workspace(WS_BATCH, (nV + nsmall) * sizeof(double));
    if (!V) return SB_ERR_NOMEM;
    double* w = V + nV;
    double* h1 = w + nt;
    double* h2 = h1 + (maxit + 1);
    double* alpha = h2 + (maxit + 1);
    double* beta = alpha + (maxit + 1);
    double* S = beta + (maxit + 2);
    double* res = S + (size_t)maxit * k;
    double* amax = res + k;
    int* restart = (int*)(amax + 1);
    const unsigned gv = svd_grid(nt, 256);

    svd_start_kernel<<<gv, 256, 0, st>>>(nt, w);
    SB_LAUNCH_CHECK();
    svd_norm_kernel<<<1, SVD_RED_THREADS, 0, st>>>(w, nt, beta, 0, nullptr, nullptr, nullptr,
                                                   amax, restart);
    SB_LAUNCH_CHECK();
    svd_scale_kernel<<<gv, 256, 0, st>>>(w, nt, beta, restart, V);
    SB_LAUNCH_CHECK();

    const double u = 5.9604644775390625e-08;     // 2^-24
    std::vector<double> ah(maxit + 1), bh(maxit + 2), d, e, z;
    int m = 0, next_check = k + 1 < maxit ? k + 1 : maxit;
    bool breakdown = false, tie = false, rule_ok = false;
    double gap = 0.0, theta1 = 0.0;
    std::vector<int> order;
    for (;;) {
        // one Lanczos step on v_m = V[m]
        const double* v = V + (size_t)m * nt;
        rc = svd_matvec(A, nf, nt, G, v, part, w, st);
        if (rc) return rc;
        for (int pass = 0; pass < 2; ++pass) {
            double* h = pass ? h2 : h1;
            svd_dots_kernel<<<m + 1, SVD_RED_THREADS, 0, st>>>(V, m + 1, nt, w, h);
            SB_LAUNCH_CHECK();
            svd_orth_kernel<<<gv, 256, 0, st>>>(V, m + 1, nt, h, w);
            SB_LAUNCH_CHECK();
        }
        svd_norm_kernel<<<1, SVD_RED_THREADS, 0, st>>>(w, nt, beta + m + 1, m, h1, h2, alpha,
                                                       amax, restart);
        SB_LAUNCH_CHECK();
        svd_scale_kernel<<<gv, 256, 0, st>>>(w, nt, beta + m + 1, restart,
                                             V + (size_t)(m + 1) * nt);
        SB_LAUNCH_CHECK();
        if (m + 1 < maxit) {
            svd_restart_kernel<<<1, 1024, 0, st>>>(restart, V, m + 1, nt, V + (size_t)(m + 1) * nt);
            SB_LAUNCH_CHECK();
        }
        ++m;
        if (m < next_check && m < maxit) continue;

        SB_CUDA(cudaMemcpyAsync(ah.data(), alpha, m * sizeof(double), cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaMemcpyAsync(bh.data(), beta, (m + 1) * sizeof(double), cudaMemcpyDeviceToHost,
                                st));
        SB_CUDA(cudaStreamSynchronize(st));
        d.assign(ah.begin(), ah.begin() + m);
        e.assign(m, 0.0);
        for (int i = 0; i + 1 < m; ++i) e[i] = bh[i + 1];
        z.assign(m, 0.0);
        z[m - 1] = 1.0;
        bool finite = true;
        for (int i = 0; i <= m; ++i) finite = finite && std::isfinite(bh[i]);
        for (int i = 0; i < m; ++i) finite = finite && std::isfinite(ah[i]);
        if (!finite || svd_tridiag_ql(m, d.data(), e.data(), z.data(), 1) != 0) {
            rule_ok = false;       // NaN / Inf data or a failed QL: stop, not converged
            break;
        }
        order.resize(m);
        for (int i = 0; i < m; ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return d[a] > d[b]; });
        theta1 = d[order[0]] > 0.0 ? d[order[0]] : 0.0;
        const double bnext = bh[m];
        const bool exhausted = m >= nt;          // T_m is B in the basis V
        const bool null_restart =                // the restart vector found nothing left
            bnext == 0.0 && m >= 2 && bh[m - 1] == 0.0 && ah[m - 1] <= 1e-12 * theta1;
        if (bnext == 0.0 && !exhausted && !null_restart) {
            next_check = m + 1;                  // restart due: never judge r_j = 0 here
            if (m >= maxit) break;
            continue;
        }
        // top Ritz value of the current block (the steps since the last restart): until it
        // has converged, a Ritz value the restart is still lifting may belong above theta_k
        int b0 = m - 1;
        while (b0 > 0 && bh[b0] != 0.0) --b0;
        double rb = 0.0;
        {
            const int nb = m - b0;
            std::vector<double> db(ah.begin() + b0, ah.begin() + m), eb(nb, 0.0), zb(nb, 0.0);
            for (int i = 0; i + 1 < nb; ++i) eb[i] = bh[b0 + i + 1];
            zb[nb - 1] = 1.0;
            if (svd_tridiag_ql(nb, db.data(), eb.data(), zb.data(), 1) != 0) break;
            const int top = (int)(std::max_element(db.begin(), db.end()) - db.begin());
            rb = fabs(bnext * zb[top]);
        }
        double rmax = 0.0, tk = 0.0, tk1 = 0.0, rk1 = 0.0;
        for (int j = 0; j < k && j < m; ++j) rmax = fmax(rmax, fabs(bnext * z[order[j]]));
        if (m > k) {
            tk = d[order[k - 1]];
            tk1 = d[order[k]];
            rk1 = fabs(bnext * z[order[k]]);
            gap = tk - tk1 - rk1;
        }
        const bool ok = rmax <= 1e-12 * theta1 && rk1 <= 1e-8 * theta1 && rb <= 1e-8 * theta1;
        const bool zero_tail = tk1 + rk1 <= 1e-12 * theta1;      // also when m <= k
        const bool exact = exhausted || null_restart || (ok && zero_tail);
        tie = (exact || ok) && !zero_tail && tk - tk1 <= 2.0 * u * theta1;
        if (exact || (ok && (gap > 0.0 || tie))) {
            breakdown = exact;
            rule_ok = !tie;
            break;
        }
        if (m >= maxit) {
            rule_ok = false;
            break;
        }
        next_check = m + (m / 8 > 1 ? m / 8 : 1);
        if (next_check > maxit) next_check = maxit;
    }

    // Ritz vectors of the top kk = min(k, m) values: full QL of T_m once
    const int kk = k < m ? k : m;
    std::vector<double> Z((size_t)m * m, 0.0), Sh((size_t)m * kk);
    d.assign(ah.begin(), ah.begin() + m);
    e.assign(m, 0.0);
    for (int i = 0; i + 1 < m; ++i) e[i] = bh[i + 1];
    for (int i = 0; i < m; ++i) Z[(size_t)i * m + i] = 1.0;
    const bool ql_ok = std::isfinite(theta1) &&
                       svd_tridiag_ql(m, d.data(), e.data(), Z.data(), m) == 0;
    order.resize(m);
    for (int i = 0; i < m; ++i) order[i] = i;
    if (ql_ok)   // NaN values would break the ordering; the result is flagged below anyway
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return d[a] > d[b]; });
    for (int q = 0; q < m; ++q)
        for (int r = 0; r < kk; ++r) Sh[(size_t)q * kk + r] = Z[(size_t)q * m + order[r]];
    SB_CUDA(cudaMemcpyAsync(S, Sh.data(), Sh.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    svd_ritz_kernel<<<gv, 256, 0, st>>>(V, m, nt, S, kk, k, Y);
    SB_LAUNCH_CHECK();
    // true residuals ||B y_j - theta_j y_j||: one read of A per mode
    for (int r = 0; r < kk; ++r) {
        rc = svd_matvec(A, nf, nt, G, Y + (size_t)r * nt, part, w, st);
        if (rc) return rc;
        svd_resid_kernel<<<1, SVD_RED_THREADS, 0, st>>>(w, Y + (size_t)r * nt, d[order[r]], nt,
                                                        res + r);
        SB_LAUNCH_CHECK();
    }
    std::vector<double> rh(k, 0.0);
    if (kk > 0)
        SB_CUDA(cudaMemcpyAsync(rh.data(), res, kk * sizeof(double), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    bool confirmed = ql_ok;
    for (int r = 0; r < k; ++r) {
        const double th = r < kk ? d[order[r]] : 0.0;
        s_host[r] = th > 0.0 ? sqrt(th) : 0.0;
        res_host[r] = rh[r];
        confirmed = confirmed && rh[r] <= 1e-11 * theta1;    // NaN fails
    }
    *gap_host = gap;
    info_host[0] = m;
    info_host[1] = (rule_ok && confirmed) ? 1 : 0;
    info_host[2] = tie ? 1 : 0;
    info_host[3] = breakdown ? 1 : 0;
    return SB_OK;
}

int svd_apply(const float* A, int nf, int nt, int k, const double* Y, float* out, float* model,
              cudaStream_t st) {
    int rc = svd_shape("sb_svd_apply", nf, nt);
    if (rc) return rc;
    SB_ARG(A && Y && (out || model));
    SB_ARG(k >= 1 && k <= SVD_MAX_MODES);
    ProfScope prof(PROF_SVD_APPLY, st);
    const int C = svd_cols(nt);
    const size_t smem = C > 16 ? (size_t)C * SVD_THREADS * sizeof(float) : 0;
    if (smem > 48 * 1024)
        SB_CUDA(cudaFuncSetAttribute(svd_apply_kernel<32>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const unsigned G = (unsigned)(nf < num_sms() * 2 ? nf : num_sms() * 2);
#define SVD_A(C) svd_apply_kernel<C><<<G, SVD_THREADS, smem, st>>>(A, nf, nt, k, Y, out, model)
    SVD_DISPATCH(C, SVD_A)
#undef SVD_A
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int bandpass_rows(const float* A, int nf, int nt, int zero_as_nan, double* mean, cudaStream_t st) {
    int rc = svd_shape("sb_bandpass_rows", nf, nt);
    if (rc) return rc;
    SB_ARG(A && mean);
    const unsigned G = (unsigned)(nf < num_sms() * 8 ? nf : num_sms() * 8);
    bandpass_row_kernel<<<G, BP_THREADS, 0, st>>>(A, nf, nt, zero_as_nan, mean);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int bandpass_cols(const float* A, int nf, int nt, int zero_as_nan, const double* rowdiv,
                  double* mean, cudaStream_t st) {
    int rc = svd_shape("sb_bandpass_cols", nf, nt);
    if (rc) return rc;
    SB_ARG(A && mean);
    const int gx = (nt + BP_THREADS - 1) / BP_THREADS;
    int nchunk = num_sms() * 8 / gx;
    nchunk = nchunk < 1 ? 1 : (nchunk > nf ? nf : nchunk);
    const int rows_per = (nf + nchunk - 1) / nchunk;
    nchunk = (nf + rows_per - 1) / rows_per;
    double* psum = (double*)workspace(WS_TABLE, (size_t)2 * nchunk * nt * sizeof(double));
    if (!psum) return SB_ERR_NOMEM;
    double* pcnt = psum + (size_t)nchunk * nt;
    bandpass_col_kernel<<<dim3(gx, nchunk), BP_THREADS, 0, st>>>(A, nf, nt, zero_as_nan, rowdiv,
                                                                 rows_per, psum, pcnt);
    SB_LAUNCH_CHECK();
    bandpass_col_reduce_kernel<<<svd_grid(nt, 256), 256, 0, st>>>(psum, pcnt, nchunk, nt, mean);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int bandpass_divide(const float* A, int nf, int nt, int zero_as_nan, const double* rowdiv,
                    const double* coldiv, float* out, cudaStream_t st) {
    int rc = svd_shape("sb_bandpass_divide", nf, nt);
    if (rc) return rc;
    SB_ARG(A && out);
    bandpass_divide_kernel<<<svd_grid((long long)nf * nt, 256), 256, 0, st>>>(
        A, nf, nt, zero_as_nan, rowdiv, coldiv, out);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
