// Phase retrieval building blocks (SURVEY section 8f rank 1):
//   rev_map      ththmod.py:176-258   theta-theta -> conjugate spectrum (scatter)
//   herm_eigvec  ththmod.py:300-307   top eigenpair of the reduced theta-theta
//                                     matrix (eigsh(.., 1, which='LA') in modeler)
//   ifft2        ththmod.py:321, 1462 ifft2(ifftshift(recov)), cropped
//   chisq_sweep  ththmod.py:330-368   chisq_calc over a batch of curvatures
//   vlbi_retrieval ththmod.py:1223-1387 VLBI_chunk_retrieval after the spectra, and
//                conj_spectrum_c2c    the conjugate spectrum of its complex visibilities
//   asymmetry_batch ththmod.py:2385-2463 calc_asymmetry over a batch of chunks
// used by the Python mirrors of modeler / single_chunk_retrieval / chisq_calc /
// VLBI_chunk_retrieval / calc_asymmetry.
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>

#ifndef SB_HOST_EMU            // tests/host_emu runs the scatter / eigenpair kernels on the CPU
#include "fft_kernels.cuh"
#endif
#include "../../include/scint_b200.h"   // SB_ETA_* status bits, tests/host_emu too
#include "drivers.cuh"
#include "lanczos.cuh"
#include "thth.cuh"

namespace sb {

// Combinations of the SB_ETA_* status bits of an eigenpair
// no eigenpair: the reference raises (IndexError, eigsh on fewer than 3 centres) or ARPACK
// fails on a zero start vector
constexpr int ETA_NO_EIGENPAIR = SB_ETA_INDEX_ERROR | SB_ETA_ZERO_START | SB_ETA_TOO_SMALL;
// no eigenvector was computed (a zero matrix still yields one)
constexpr int ETA_NO_VECTOR = SB_ETA_INDEX_ERROR | SB_ETA_TOO_SMALL;
// the reference's try/except stores NaN
constexpr int ETA_NAN = ETA_NO_EIGENPAIR | SB_ETA_NOT_CONVERGED;

// --------------------------------------------------------------------------
// rev_map.  np.histogram2d with explicit edges e_k = (k - 0.5) * d + x0
// (k = 0..N, the same two roundings as numpy): bin = #{e_k <= x} - 1, x == e_N
// belongs to the last bin, anything outside is dropped.  Bit-exact bins; the
// weighted sums are fp32 atomics (order-dependent in the last bits).
// --------------------------------------------------------------------------
__device__ __forceinline__ double hist_edge(int k, double x0, double d) {
    return __dadd_rn(__dmul_rn((double)k - 0.5, d), x0);
}
__device__ __forceinline__ int hist_bin(double x, double x0, double d, int N) {
    if (!(x == x)) return -1;
    const double g = (x - x0) / d + 0.5;
    if (!(g > -2.0) || !(g < (double)N + 2.0)) return -1;
    int k = (int)floor(g);
    k = max(0, min(k, N));
    while (k < N && hist_edge(k + 1, x0, d) <= x) ++k;
    while (k >= 0 && hist_edge(k, x0, d) > x) --k;
    if (k < 0) return -1;
    if (k == N) return (x == hist_edge(N, x0, d)) ? N - 1 : -1;
    return k;
}

struct RevGeom {
    const double* th;
    int n;
    double eta, tau0, dtau, fd0, dfd;
    int ntau, nfd;
};

// fd, tau and Jacobian of point (i, j) of the theta-theta matrix:
// fd_map[i][j] = th[j] - th[i];  tau_map = eta * (th[j]^2 - th[i]^2)
struct RevPoint { double x, y, jac; };
__device__ __forceinline__ RevPoint rev_point(const RevGeom& g, int i, int j) {
    const double ti = g.th[i], tj = g.th[j];
    return {__dsub_rn(tj, ti),
            __dmul_rn(g.eta, __dsub_rn(__dmul_rn(tj, tj), __dmul_rn(ti, ti))),
            sqrt(fabs(__dmul_rn(__dmul_rn(2.0, g.eta), __dsub_rn(ti, tj))))};
}
// histogram bin of (fd, tau) = (x, y), or -1 outside
__device__ __forceinline__ long rev_bin(const RevGeom& g, double x, double y) {
    const int bx = hist_bin(x, g.fd0, g.dfd, g.nfd), by = hist_bin(y, g.tau0, g.dtau, g.ntau);
    return (bx >= 0 && by >= 0) ? (long)by * g.nfd + bx : -1;
}

// point (i, j), i != j, of the theta-theta matrix with value v into the histograms
__device__ __forceinline__ void rev_scatter_point(const RevGeom& g, int i, int j, float2 v,
                                                  int hermitian, float2* __restrict__ acc,
                                                  int* __restrict__ cnt) {
    const RevPoint p = rev_point(g, i, j);
    const float wre = (float)((double)v.x / p.jac), wim = (float)((double)v.y / p.jac);
    long o = rev_bin(g, p.x, p.y);
    if (o >= 0) {
        atomicAdd(&acc[o].x, wre);
        atomicAdd(&acc[o].y, wim);
        atomicAdd(&cnt[o], 1);
    }
    if (hermitian) {
        o = rev_bin(g, -p.x, -p.y);
        if (o >= 0) {
            atomicAdd(&acc[o].x, wre);
            atomicAdd(&acc[o].y, -wim);
            atomicAdd(&cnt[o], 1);
        }
    }
}

__global__ void rev_scatter_kernel(RevGeom g, const float2* __restrict__ thth, int hermitian,
                                   float2* __restrict__ acc, int* __restrict__ cnt) {
    const long total = (long)g.n * g.n;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total;
         p += (long)gridDim.x * blockDim.x) {
        const int i = (int)(p / g.n), j = (int)(p - (long)i * g.n);
        if (i == j) continue;   // zero Jacobian: the DC bin is NaN -> 0 (finalise kernel)
        rev_scatter_point(g, i, j, thth[p], hermitian, acc, cnt);
    }
}

// the bin of (fd, tau) = (0, 0) receives the n diagonal points with an infinite / NaN
// weight: NaN after the division, 0 after nan_to_num.  Its index, or -1.
__device__ __forceinline__ long rev_dc_bin(const RevGeom& g) {
    const int bx0 = hist_bin(0.0, g.fd0, g.dfd, g.nfd), by0 = hist_bin(0.0, g.tau0, g.dtau, g.ntau);
    return (bx0 >= 0 && by0 >= 0) ? (long)by0 * g.nfd + bx0 : -1;
}
// bin mean of rev_map (recov /= norm; nan_to_num) from the weighted sum and the count
__device__ __forceinline__ float2 rev_bin_value(float2 v, int c, bool dc) {
    if (c > 0 && !dc) {
        const float s = 1.0f / (float)c;
        v.x *= s;
        v.y *= s;
        // np.nan_to_num(recov): NaN -> 0, +-inf -> +-largest float
        v.x = (v.x != v.x) ? 0.f : fminf(fmaxf(v.x, -FLT_MAX), FLT_MAX);
        v.y = (v.y != v.y) ? 0.f : fminf(fmaxf(v.y, -FLT_MAX), FLT_MAX);
        return v;
    }
    return make_float2(0.f, 0.f);
}

__global__ void rev_finalise_kernel(RevGeom g, float2* __restrict__ acc,
                                    const int* __restrict__ cnt) {
    const long total = (long)g.ntau * g.nfd;
    const long dc = rev_dc_bin(g);
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < total;
         o += (long)gridDim.x * blockDim.x)
        acc[o] = rev_bin_value(acc[o], cnt[o], o == dc);
}

// --------------------------------------------------------------------------
// chisq_sweep: rev_map of the rank-1 model |w| V V^H of every curvature of a batch
// (blockIdx.y), computed on the fly from V; the model matrix is never stored.
// th_red [neta][th_pitch]: the curvature's rev_map centres (theta_centres of its
// edges_red), nred[e] of them.  Curvatures without an eigenpair (ETA_NO_EIGENPAIR)
// scatter nothing: their model is zero.
// --------------------------------------------------------------------------
__global__ void rev_scatter_rank1_kernel(RevGeom g, const double* __restrict__ th_red,
                                         int th_pitch, const double* __restrict__ etas, int e0,
                                         const int* __restrict__ nred,
                                         const int* __restrict__ status,
                                         const double* __restrict__ w,
                                         const float2* __restrict__ V, int ldv,
                                         float2* __restrict__ acc, int* __restrict__ cnt) {
    const int e = blockIdx.y;
    if (status[e0 + e] & ETA_NO_EIGENPAIR) return;
    g.n = nred[e0 + e];
    g.th = th_red + (size_t)(e0 + e) * th_pitch;
    g.eta = etas[e0 + e];
    const float aw = (float)fabs(w[e0 + e]);
    const float2* v = V + (size_t)e * ldv;
    const size_t bins = (size_t)g.ntau * g.nfd;
    acc += e * bins;
    cnt += e * bins;
    const long total = (long)g.n * g.n;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < total;
         p += (long)gridDim.x * blockDim.x) {
        const int i = (int)(p / g.n), j = (int)(p - (long)i * g.n);
        if (i == j) continue;
        const float2 a = v[i], b = v[j];        // |w| V_i conj(V_j)
        const float2 t = make_float2(aw * (a.x * b.x + a.y * b.y), aw * (a.y * b.x - a.x * b.y));
        rev_scatter_point(g, i, j, t, 1, acc, cnt);
    }
}

__global__ void rev_finalise_batch_kernel(RevGeom g, float2* __restrict__ acc,
                                          const int* __restrict__ cnt) {
    const long total = (long)g.ntau * g.nfd;
    const long dc = rev_dc_bin(g);
    acc += blockIdx.y * (size_t)total;
    cnt += blockIdx.y * (size_t)total;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < total;
         o += (long)gridDim.x * blockDim.x)
        acc[o] = rev_bin_value(acc[o], cnt[o], o == dc);
}

#ifndef SB_HOST_EMU
int rev_map(const float2* thth, int n, const double* th_dev, double eta, double tau0,
            double dtau, int ntau, double fd0, double dfd, int nfd, int hermitian,
            float2* recov, cudaStream_t st) {
    if (!(dtau > 0.0) || !(dfd > 0.0)) {
        set_error("rev_map needs ascending tau / fd axes (bins must increase monotonically)");
        return SB_ERR_ARG;
    }
    const size_t bins = (size_t)ntau * nfd;
    int* cnt = (int*)workspace(WS_INDEX, bins * sizeof(int));
    if (!cnt) return SB_ERR_NOMEM;
    SB_CUDA(cudaMemsetAsync(recov, 0, bins * sizeof(float2), st));
    SB_CUDA(cudaMemsetAsync(cnt, 0, bins * sizeof(int), st));
    RevGeom g{th_dev, n, eta, tau0, dtau, fd0, dfd, ntau, nfd};
    const long total = (long)n * n;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    if (blocks < 1) blocks = 1;
    rev_scatter_kernel<<<blocks, 256, 0, st>>>(g, thth, hermitian, recov, cnt);
    SB_LAUNCH_CHECK();
    int fb = (int)((bins + 255) / 256);
    if (fb > num_sms() * 16) fb = num_sms() * 16;
    rev_finalise_kernel<<<fb, 256, 0, st>>>(g, recov, cnt);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

// --------------------------------------------------------------------------
// Top eigenpair (largest algebraic) of one full Hermitian complex matrix:
// Lanczos with the basis kept in global memory and classical Gram-Schmidt
// re-orthogonalisation (twice), Ritz vector from the backward three-term
// recurrence of T_m at theta.  One CTA; used once per chunk.
// --------------------------------------------------------------------------
constexpr int EV_THREADS = 512;
constexpr int EV_NW = EV_THREADS / 32;

// element (a, c) of a full row-major matrix
struct FullMatrix {
    const float2* A;
    int ld;
    __device__ __forceinline__ float2 operator()(int a, int c) const { return A[(size_t)a * ld + c]; }
};
// element (a, c) of a Hermitian matrix with zero diagonal stored as its strict upper
// triangle (thth_build_kernel<PACK = 0>): the lower triangle is the conjugate mirror
struct UpperHermitian {
    const float2* M;
    int ld;
    __device__ __forceinline__ float2 operator()(int a, int c) const {
        if (c > a) return M[(size_t)a * ld + c];
        if (c < a) {
            const float2 x = M[(size_t)c * ld + a];
            return make_float2(x.x, -x.y);
        }
        return make_float2(0.f, 0.f);
    }
};

// The composite of VLBI_chunk_retrieval: n_dish x n_dish blocks of n x n, full row-major
struct CompositeMatrix {
    const float2* A;
    int ld, n_dish, n;
    __device__ __forceinline__ float2 operator()(int a, int c) const { return A[(size_t)a * ld + c]; }
};
// Lanczos start vector, element c: row h of the matrix ...
template <class Mat>
__device__ __forceinline__ float2 start_row(const Mat& A, int h, int c) { return A(h, c); }
// ... except for the composite: the sum of row n//2 of every station's block row.  A
// single row lies in one block row; when the stations do not couple (zero visibilities)
// the composite is block diagonal and Lanczos would never leave that station's block.
__device__ __forceinline__ float2 start_row(const CompositeMatrix& A, int, int c) {
    float2 s = make_float2(0.f, 0.f);
    for (int d = 0; d < A.n_dish; ++d) {
        const float2 x = A(d * A.n + A.n / 2, c);
        s.x += x.x;
        s.y += x.y;
    }
    return s;
}

// Shared body.  Start vector: row n//2 (start_row).  If it is zero, zero_start_fallback == 0
// reports it (w = NaN, info[1] = SB_ETA_ZERO_START); otherwise Lanczos starts from a fixed
// non-zero vector instead, and a start vector that A maps to zero (for a zero-diagonal
// Hermitian matrix: A == 0) gives w = 0 with that vector as V and info[1] = SB_ETA_ZERO_START.
template <class Mat>
__device__ void herm_eigvec_body(Mat A, int n, float2* __restrict__ Q, int max_iter, double tol,
                                 int zero_start_fallback, double* __restrict__ w_out,
                                 float2* __restrict__ V_out, int* __restrict__ info) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    LanczosShared& S = *reinterpret_cast<LanczosShared*>(smem_raw);
    double* red = reinterpret_cast<double*>(smem_raw + sizeof(LanczosShared));   // [EV_NW]
    double2* coef = reinterpret_cast<double2*>(red + 32);                        // [max_iter + 1]
    float2* v = reinterpret_cast<float2*>(coef + SB_LANCZOS_MAXIT + 1);
    float2* w = v + n;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);

    // start vector: row n//2, like Eval_calc (any vector with a component
    // along the top eigenvector would do; eigsh uses a random one)
    const int h = n / 2;
    double p0 = 0.0;
    for (int c = tid; c < n; c += EV_THREADS) {
        const float2 x = start_row(A, h, c);
        v[c] = x;
        p0 += (double)x.x * x.x + (double)x.y * x.y;
    }
    lanczos_reset(S);
    double nrm2 = cta_sum<EV_NW>(p0, red);
    const bool fallback = zero_start_fallback && nrm2 == 0.0 && n >= 2;
    if (fallback) {
        p0 = 0.0;
        for (int c = tid; c < n; c += EV_THREADS) {
            v[c] = make_float2(1.0f + 0.125f * (float)((c * 37) % 11), 0.f);
            p0 += (double)v[c].x * v[c].x;
        }
        __syncthreads();                // every thread has read red
        nrm2 = cta_sum<EV_NW>(p0, red);
    }
    if (!(nrm2 > 0.0) || !isfinite(nrm2) || n < 2) {
        if (tid == 0) { *w_out = qnan; info[0] = 0; info[1] = SB_ETA_ZERO_START; }
        for (int c = tid; c < n; c += EV_THREADS) V_out[c] = make_float2(0.f, 0.f);
        return;
    }
    {
        const float s = (float)(1.0 / sqrt(nrm2));
        for (int c = tid; c < n; c += EV_THREADS) { v[c].x *= s; v[c].y *= s; }
    }
    __syncthreads();
    int m = 0;
    float beta_prev = 0.f;
    for (int it = 0; it < max_iter; ++it) {
        for (int c = tid; c < n; c += EV_THREADS) Q[(size_t)it * n + c] = v[c];
        // w = A v : one warp per row, lanes across the columns
        for (int a = warp; a < n; a += EV_NW) {
            float rx = 0.f, ry = 0.f;
            for (int c = lane; c < n; c += 32) {
                const float2 q = A(a, c), x = v[c];
                rx = fmaf(q.x, x.x, rx); rx = fmaf(-q.y, x.y, rx);
                ry = fmaf(q.x, x.y, ry); ry = fmaf(q.y, x.x, ry);
            }
            rx = warp_sum(rx);
            ry = warp_sum(ry);
            if (lane == 0) w[a] = make_float2(rx, ry);
        }
        __syncthreads();
        double ap = 0.0;
        for (int c = tid; c < n; c += EV_THREADS)
            ap += (double)v[c].x * w[c].x + (double)v[c].y * w[c].y;
        const double alpha = cta_sum<EV_NW>(ap, red);
        {
            const float af = (float)alpha;
            const float2* qp = Q + (size_t)(it > 0 ? it - 1 : 0) * n;
            for (int c = tid; c < n; c += EV_THREADS) {
                float2 x = w[c];
                const float2 pv = it > 0 ? qp[c] : make_float2(0.f, 0.f);
                x.x -= af * v[c].x + beta_prev * pv.x;
                x.y -= af * v[c].y + beta_prev * pv.y;
                w[c] = x;
            }
        }
        __syncthreads();
        // classical Gram-Schmidt against Q[0..it], twice: warp j computes <Q_j, w>
        for (int pass = 0; pass < 2; ++pass) {
            for (int j0 = 0; j0 <= it; j0 += EV_NW) {
                const int j = j0 + warp;
                if (j <= it) {
                    const float2* q = Q + (size_t)j * n;
                    double cx_ = 0.0, cy_ = 0.0;
                    for (int c = lane; c < n; c += 32) {
                        const float2 a = q[c], b = w[c];   // conj(a) * b
                        cx_ += (double)a.x * b.x + (double)a.y * b.y;
                        cy_ += (double)a.x * b.y - (double)a.y * b.x;
                    }
                    cx_ = warp_sum(cx_);
                    cy_ = warp_sum(cy_);
                    if (lane == 0) coef[j] = make_double2(cx_, cy_);
                }
            }
            __syncthreads();
            for (int c = tid; c < n; c += EV_THREADS) {
                double sx = 0.0, sy = 0.0;
                for (int j = 0; j <= it; ++j) {
                    const float2 q = Q[(size_t)j * n + c];
                    const double2 cf = coef[j];
                    sx += cf.x * q.x - cf.y * q.y;
                    sy += cf.x * q.y + cf.y * q.x;
                }
                w[c].x -= (float)sx;
                w[c].y -= (float)sy;
            }
            __syncthreads();
        }
        double bp = 0.0;
        for (int c = tid; c < n; c += EV_THREADS) bp += (double)w[c].x * w[c].x + (double)w[c].y * w[c].y;
        const double b2 = cta_sum<EV_NW>(bp, red);
        const double beta = sqrt(b2);
        m = it + 1;
        if (fallback && it == 0 && alpha == 0.0 && b2 == 0.0) {
            // A v = 0 for the fallback vector: report w = 0, V = v
            for (int c = tid; c < n; c += EV_THREADS) V_out[c] = v[c];
            if (tid == 0) { *w_out = 0.0; info[0] = 1; info[1] = SB_ETA_ZERO_START; }
            return;
        }
        if (tid == 0) { S.alpha[it] = alpha; S.beta[m] = beta; S.beta2[m] = b2; }
        __syncthreads();
        if (warp == 0) lanczos_check(S, m, tol, 0.0);
        __syncthreads();
        if (S.done || !isfinite(alpha) || m == max_iter || m == n) break;
        const float ib = (float)(1.0 / beta);
        for (int c = tid; c < n; c += EV_THREADS) v[c] = make_float2(w[c].x * ib, w[c].y * ib);
        beta_prev = (float)beta;
        __syncthreads();
    }
    // Ritz vector of T_m at theta
    lanczos_ritz(S, m);
    double yp = 0.0;
    for (int c = tid; c < n; c += EV_THREADS) {
        double sx = 0.0, sy = 0.0;
        for (int j = 0; j < m; ++j) {
            const float2 q = Q[(size_t)j * n + c];
            sx += S.piv[j] * q.x;
            sy += S.piv[j] * q.y;
        }
        w[c] = make_float2((float)sx, (float)sy);
        yp += sx * sx + sy * sy;
    }
    const double yn = cta_sum<EV_NW>(yp, red);
    const float ys = (float)(1.0 / sqrt(yn));
    for (int c = tid; c < n; c += EV_THREADS) V_out[c] = make_float2(w[c].x * ys, w[c].y * ys);
    if (tid == 0) {
        *w_out = S.theta;
        info[0] = m;
        // the requested residual (1e-7 by default) is close to the fp32 rounding floor; a
        // residual <= 2e-6 |theta| at the iteration cap is still a converged pair for every
        // consumer (eigenvalue error ~ res^2 / gap), anything worse is flagged
        info[1] = (S.done || S.res <= 2e-6 * fabs(S.theta)) ? 0 : SB_ETA_NOT_CONVERGED;
    }
}

__global__ void __launch_bounds__(EV_THREADS)
herm_eigvec_kernel(const float2* __restrict__ A, int n, int ld, float2* __restrict__ Q,
                   int max_iter, double tol, double* __restrict__ w_out,
                   float2* __restrict__ V_out, int* __restrict__ info) {
    herm_eigvec_body(FullMatrix{A, ld}, n, Q, max_iter, tol, 0, w_out, V_out, info);
}

// chisq_sweep: the top eigenpair of every cropped theta-theta matrix of a batch, one CTA per
// curvature (blockIdx.x), on the strict upper triangles M [nb][ld][ld] of the sweep's gather.
// Q: [nb][max_iter + 1][ld] Lanczos bases; V: [nb][ld].  Writes w (NaN where the reference
// raises), iters and the SB_ETA_* bits of curvatures e0 .. e0 + nb - 1.
__global__ void __launch_bounds__(EV_THREADS)
herm_eigvec_batch_kernel(const float2* __restrict__ M, int ld, const int* __restrict__ nred,
                         int e0, float2* __restrict__ Q, int max_iter, double tol,
                         double* __restrict__ w, float2* __restrict__ V,
                         int* __restrict__ status, int* __restrict__ iters) {
    const int e = blockIdx.x, ge = e0 + e;
    const int n = nred[ge];
    if ((status[ge] & SB_ETA_INDEX_ERROR) || n < 3) {    // IndexError / eigsh raises for n < 3
        if (threadIdx.x == 0) {
            w[ge] = __longlong_as_double(0x7ff8000000000000LL);
            iters[ge] = 0;
            if (n < 3) status[ge] |= SB_ETA_TOO_SMALL;
        }
        return;
    }
    __shared__ int info[2];
    herm_eigvec_body(UpperHermitian{M + (size_t)e * ld * ld, ld}, n, Q + (size_t)e * (max_iter + 1) * ld,
                     max_iter, tol, 1, w + ge, V + (size_t)e * ld, info);
    if (threadIdx.x == 0) {        // info was written by thread 0 of the body
        iters[ge] = info[0];
        status[ge] |= info[1];
    }
}

// --------------------------------------------------------------------------
// calc_asymmetry (ththmod.py:2385-2463) over a batch of chunks, each with its own
// spectrum, axes, theta grid and curvature (geoms[e], etas[e]).
// --------------------------------------------------------------------------
// Strict upper triangle of every cropped matrix of chunks e0 .. e0 + gridDim.y - 1 into
// M [nb][ld][ld] (the layout herm_eigvec_batch_kernel reads): thth_redmap's Hermitian
// fill of the crop idx[e][0 .. nred[e]).
__global__ void asym_gather_kernel(const ThthGeom* __restrict__ geoms,
                                   const double* __restrict__ etas, int e0, int ld,
                                   const int* __restrict__ idx, const int* __restrict__ nred,
                                   float2* __restrict__ M) {
    const int e = blockIdx.y, ge = e0 + e;
    const ThthGeom g = geoms[ge];
    const double eta = etas[ge];
    const int n = nred[ge];
    const int* id = idx + (size_t)ge * ld;
    float2* Me = M + (size_t)e * ld * ld;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < (long)n * n;
         p += (long)gridDim.x * blockDim.x) {
        const int a = (int)(p / n), c = (int)(p - (long)a * n);
        if (c > a) Me[(size_t)a * ld + c] = thth_herm_upper(g, eta, id[a], id[c]);
    }
}

// asymm = (|V[:h]|^2 - |V[h+1:m]|^2) / (|V[:h]|^2 + |V[h+1:m]|^2), h = (m - 1) // 2, in fp64
// from the fp32 eigenvector V [nb][ld] of each chunk (one warp per chunk).  NaN where the
// reference's try/except stores NaN: IndexError, a zero matrix, m < 3, no convergence
// (ETA_NAN); 0 / 0 is NaN as in numpy.  v_out [nchunk][ld] (optional): V, zero-padded, or
// zeros where no eigenvector was computed (ETA_NO_VECTOR).
__global__ void asym_finish_kernel(const float2* __restrict__ V, int ld,
                                   const int* __restrict__ nred, const int* __restrict__ status,
                                   int e0, double* __restrict__ asym, float2* __restrict__ v_out) {
    const int e = blockIdx.x, ge = e0 + e, lane = threadIdx.x;
    const int m = nred[ge], st = status[ge];
    const float2* v = V + (size_t)e * ld;
    const int h = (m - 1) / 2;
    const bool has_v = !(st & ETA_NO_VECTOR);
    double l = 0.0, r = 0.0;
    for (int c = lane; c < ld; c += 32) {
        const float2 x = (has_v && c < m) ? v[c] : make_float2(0.f, 0.f);
        const double p = (double)x.x * x.x + (double)x.y * x.y;
        if (c < h) l += p;
        else if (c > h) r += p;
        if (v_out) v_out[(size_t)ge * ld + c] = x;
    }
    l = warp_sum(l);
    r = warp_sum(r);
    if (lane == 0)
        asym[ge] = (st & ETA_NAN) ? __longlong_as_double(0x7ff8000000000000LL) : (l - r) / (l + r);
}

// --------------------------------------------------------------------------
// VLBI_chunk_retrieval (ththmod.py:1223-1387): the composite theta-theta matrix of
// n_dish stations, its top eigenpair and one wavefield per station.
// Spectra are in reference order [I1, V12, .., V1N, I2, V23, .., IN]; pair (d1, d1 + d2)
// sits at index N(N+1)/2 - (N-d1)(N-d1+1)/2 + d2, autos at d2 = 0.
// --------------------------------------------------------------------------
__host__ __device__ __forceinline__ int vlbi_pair_index(int n_dish, int d1, int d2) {
    return n_dish * (n_dish + 1) / 2 - (n_dish - d1) * (n_dish - d1 + 1) / 2 + d2;
}

// Composite [n_dish n][n_dish n], row-major, written whole: block (b, b + d2) is
// conj(T_k).T and block (b + d2, b) is T_k, k = pair (b, d2); the diagonal blocks are
// the autos' T.  T_k is thth_redmap of spectrum k on the crop idx[0..n): autos with the
// Hermitian fill of thth_map (upper triangle mirrored, diagonal and anti-diagonal of the
// full grid zeroed, nan_to_num), visibilities the raw Jacobian-weighted gather.
// cs: [n_dish (n_dish + 1) / 2] full-plane spectra of the geometry g.
__global__ void vlbi_composite_kernel(ThthGeom g, const double* __restrict__ eta_p,
                                      const float2* const* __restrict__ cs, int n_dish,
                                      const int* __restrict__ idx, int n,
                                      float2* __restrict__ A) {
    const double eta = *eta_p;
    const long N = (long)n_dish * n;
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < N * N;
         p += (long)gridDim.x * blockDim.x) {
        const int R = (int)(p / N), C = (int)(p - (long)R * N);
        const int bi = R / n, a = R - bi * n, bj = C / n, c = C - bj * n;
        // element (r, s) of T_k; the upper blocks read it transposed and conjugate it
        const bool upper = bi < bj;
        const int d1 = upper ? bi : bj, d2 = upper ? bj - bi : bi - bj;
        const int r = upper ? c : a, s = upper ? a : c;
        ThthGeom gk = g;
        gk.cs = cs[vlbi_pair_index(n_dish, d1, d2)];
        const int i = idx[r], j = idx[s];            // rows / columns of the full grid
        const double thi = g.th[i], thj = g.th[j];
        float2 v;
        if (d2 != 0) {
            v = thth_value(gk, eta, thj, thi, thth_point(gk, eta, thj, thi));
        } else if (i == j) {
            v = make_float2(0.f, 0.f);
        } else if (j > i) {
            v = thth_herm_upper(gk, eta, i, j);
        } else {                                     // conj of the upper element (j, i)
            v = thth_herm_upper(gk, eta, j, i);
            v.y = -v.y;
        }
        if (upper) v.y = -v.y;
        A[p] = v;
    }
}

// Top eigenpair of the composite (N = n_dish n), started from the sum of the stations'
// rows n//2 or, if that is zero, from the fixed start vector.  info = {Lanczos steps,
// SB_ETA_* status, nred}; SB_ETA_INDEX_ERROR comes from thth_prep.  A matrix smaller than
// 3 x 3 is reported as SB_ETA_TOO_SMALL (eigsh raises).
__global__ void __launch_bounds__(EV_THREADS)
vlbi_eigvec_kernel(const float2* __restrict__ A, int n_dish, int n, float2* __restrict__ Q,
                   int max_iter, double tol, double* __restrict__ w, float2* __restrict__ V,
                   int* __restrict__ info) {
    const int N = n_dish * n;
    if ((info[1] & SB_ETA_INDEX_ERROR) || N < 3) {
        for (int c = threadIdx.x; c < N; c += EV_THREADS) V[c] = make_float2(0.f, 0.f);
        if (threadIdx.x == 0) {
            *w = __longlong_as_double(0x7ff8000000000000LL);
            info[0] = 0;
            if (N < 3) info[1] |= SB_ETA_TOO_SMALL;
        }
        return;
    }
    __shared__ int sh_info[2];
    herm_eigvec_body(CompositeMatrix{A, N, n_dish, n}, N, Q, max_iter, tol, 1, w, V, sh_info);
    if (threadIdx.x == 0) {        // sh_info was written by thread 0 of the body
        info[0] = sh_info[0];
        info[1] |= sh_info[1];
    }
}

// rev_map(hermetian=False) of every station's model, whose only non-zero row is row n//2,
// conj(V[d n : (d + 1) n]) sqrt(w) (the zero rows still count in the bin means).
// blockIdx.y < n_dish: station blockIdx.y adds the values of row n//2 to acc[d];
// blockIdx.y == n_dish: the counts of all n^2 - n off-diagonal points, shared by every
// station.  A failed eigenpair (ETA_NO_EIGENPAIR) scatters nothing.
__global__ void vlbi_scatter_kernel(RevGeom g, int n_dish, const int* __restrict__ info,
                                    const double* __restrict__ w,
                                    const float2* __restrict__ V, float2* __restrict__ acc,
                                    int* __restrict__ cnt) {
    if (info[1] & ETA_NO_EIGENPAIR) return;
    const int n = g.n, h = n / 2, d = blockIdx.y;
    if (d == n_dish) {
        for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < (long)n * n;
             p += (long)gridDim.x * blockDim.x) {
            const int i = (int)(p / n), j = (int)(p - (long)i * n);
            if (i == j) continue;
            const RevPoint q = rev_point(g, i, j);
            const long o = rev_bin(g, q.x, q.y);
            if (o >= 0) atomicAdd(&cnt[o], 1);
        }
        return;
    }
    const double sw = sqrt(*w);
    float2* out = acc + (size_t)d * g.ntau * g.nfd;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        if (j == h) continue;          // zero Jacobian: the DC bin, zeroed by the finalise step
        const RevPoint pt = rev_point(g, h, j);
        const long o = rev_bin(g, pt.x, pt.y);
        if (o < 0) continue;
        const float2 q = V[(size_t)d * n + j];
        // the model element, rounded to fp32 as an uploaded complex128 matrix would be
        const float tre = (float)((double)q.x * sw), tim = (float)(-(double)q.y * sw);
        atomicAdd(&out[o].x, (float)((double)tre / pt.jac));
        atomicAdd(&out[o].y, (float)((double)tim / pt.jac));
    }
}

__global__ void vlbi_finalise_kernel(RevGeom g, float2* __restrict__ acc,
                                     const int* __restrict__ cnt) {
    const long total = (long)g.ntau * g.nfd;
    const long dc = rev_dc_bin(g);
    acc += blockIdx.y * (size_t)total;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < total;
         o += (long)gridDim.x * blockDim.x)
        acc[o] = rev_bin_value(acc[o], cnt[o], o == dc);
}

#ifndef SB_HOST_EMU
// Launch setup of a top-eigenpair kernel on matrices of order n (herm_eigvec_body): tol <= 0
// becomes 1e-7, max_iter outside 1..SB_LANCZOS_MAXIT becomes 96 and is then held to n, and
// *smem, the body's dynamic shared memory, is set as the kernel's limit.
template <class Kernel>
static int eigvec_setup(Kernel kern, int n, double* tol, int* max_iter, size_t* smem) {
    if (!(*tol > 0.0)) *tol = 1e-7;
    if (*max_iter <= 0 || *max_iter > SB_LANCZOS_MAXIT) *max_iter = 96;
    if (*max_iter > n) *max_iter = n;
    *smem = sizeof(LanczosShared) + 32 * sizeof(double) + (SB_LANCZOS_MAXIT + 1) * sizeof(double2) +
            2 * (size_t)n * sizeof(float2);
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem));
    return SB_OK;
}

int herm_eigvec(const float2* A, int n, int ld, double tol, int max_iter, double* w_dev,
                float2* V_dev, int* info_dev, cudaStream_t st) {
    if (n < 1 || n > 8192) {
        set_error("herm_eigvec: n = %d outside 1..8192", n);
        return SB_ERR_UNSUPPORTED;
    }
    size_t smem;
    int rc = eigvec_setup(herm_eigvec_kernel, n, &tol, &max_iter, &smem);
    if (rc) return rc;
    float2* Q = (float2*)workspace(WS_BATCH, (size_t)(max_iter + 1) * n * sizeof(float2));
    if (!Q) return SB_ERR_NOMEM;
    herm_eigvec_kernel<<<1, EV_THREADS, smem, st>>>(A, n, ld, Q, max_iter, tol, w_dev, V_dev,
                                                    info_dev);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// --------------------------------------------------------------------------
// Inverse 2-D transforms of the conjugate spectra: ifft2(ifftshift(.)) of the rev_map
// planes, cropped, into a wavefield / model or into the chi-square residual.
// --------------------------------------------------------------------------
// The sizes they take: powers of two 8..65536 x 8..16384 (the rows run in one
// shared-memory row transform), other sizes 3..32768 x 3..8192 (chirp-z)
static int ifft2_size_check(const char* who, int n0, int n1) {
    const bool pow2 = is_pow2(n0) && is_pow2(n1);
    if (pow2 ? (n0 < 8 || n1 < 8 || n0 > 65536 || n1 > 16384)
             : (n0 < 3 || n1 < 3 || n0 > 32768 || n1 > 8192)) {
        set_error("%s: conjugate spectrum %d x %d outside 8..65536 x 8..16384 (powers of two) / "
                  "3..32768 x 3..8192 (other sizes)", who, n0, n1);
        return SB_ERR_UNSUPPORTED;
    }
    return SB_OK;
}

// row r of plane p of ifftshift(in[p]), or of in[p] when not centred, for row = p n0 + r;
// n0 and n1 are powers of two
struct ShiftedRowLoad {
    const float2* in;
    int n0, n1, centred;
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        const long p0 = row & ~(long)(n0 - 1);          // p n0
        int r = (int)(row & (n0 - 1)), c = n;
        if (centred) {
            r = (r + n0 / 2) & (n0 - 1);
            c = (n + n1 / 2) & (n1 - 1);
        }
        return in[(size_t)(p0 + r) * n1 + c];
    }
};

// Chirp-z inverse of one [n0][n1] plane of any size, ifftshifted first when centred:
// ifft2(X) = conj(fft2(conj X)) / (n0 n1).  conj_in != 0 transforms conj(in) instead, so
// that the result is conj(fft2(in)) / (n0 n1).  The output rows x cols go to the base store
// mk(den), den = the normalisation of the unnormalised inverse it receives.
template <class MakeBase>
static int ifft2_chirp(const float2* in, int n0, int n1, int centred, int conj_in, int rows,
                       int cols, MakeBase mk, cudaStream_t st) {
    return chirp_fft2(ChirpRowLoadC{in, n0, n1, centred, conj_in, nullptr}, n0, n1, n0, cols,
                      [&](int R1, const float2* wF, int MF) {
                          const double den = (double)MF * (double)n0 * (double)n1;
                          return ChirpStore<decltype(mk(den))>{R1, rows, cols, wF, mk(den)};
                      }, "ifft2 (chirp-z):", st);
}

// ifft2 of the nplanes planes of in [nplanes][n0][n1], each ifftshifted first when centred;
// the output rows x cols of plane p go to the base store mk(p, den) (CropStore or
// ResidualSink), den = the normalisation of the unnormalised inverse it receives.  Powers of
// two: the rows of every plane in one launch, then the kept columns plane by plane; other
// sizes: ifft2_chirp per plane.  Sizes as ifft2_size_check.
template <class MakeBase>
static int ifft2_planes(const float2* in, int nplanes, int n0, int n1, int centred, int rows,
                        int cols, MakeBase mk, cudaStream_t st) {
    const size_t bins = (size_t)n0 * n1;
    if (!is_pow2(n0) || !is_pow2(n1)) {
        for (int p = 0; p < nplanes; ++p) {
            const int rc = ifft2_chirp(in + bins * p, n0, n1, centred, 0, rows, cols,
                                       [&](double den) { return mk(p, den); }, st);
            if (rc) return rc;
        }
        return SB_OK;
    }
    float2* B1 = (float2*)workspace(WS_PLANE0, nplanes * bins * sizeof(float2));
    float2* B2 = (float2*)workspace(WS_PLANE1, bins * sizeof(float2));
    if (!B1 || !B2) return SB_ERR_NOMEM;
    ShiftedRowLoad ld{in, n0, n1, centred};
    PlainRowStore<float2> rs{B1, n1};
    int rc = SB_OK;
    SB_ROW_DISPATCH(n1, rc = (launch_row_c2c<float, N1, N2, +1>(ld, rs, (long)nplanes * n0, st)));
    if (rc) return rc;
    int R1, R2;
    split_len(n0, &R1, &R2);
    const double den = (double)n0 * (double)n1;
    for (int p = 0; p < nplanes; ++p) {
        StrideALoad<float2> la{B1 + bins * p, n1, R2};
        const auto base = mk(p, den);
        rc = cols_generic<float, +1>(la, B2, n1, n0, cols,
                                     RadixStore<decltype(base)>{R1, rows, cols, base}, st);
        if (rc) return rc;
    }
    return SB_OK;
}

// scale * ifft2(conj(in)) = scale * conj(fft2(in)) / (n0 n1) of one plane of any size: the
// forward transform of the Gerchberg-Saxton loop and of conj_spectrum_c2c
static int ifft2_conj_any(const float2* in, int n0, int n1, double scale, float2* out,
                          cudaStream_t st) {
    return ifft2_chirp(in, n0, n1, 0, 1, n0, n1, [&](double den) {
        return CropStore{out, nullptr, n1, (float)(scale / den)};
    }, st);
}

// out[:crop0, :crop1] = scale * ifft2(ifftshift(in)) (centred) or scale * ifft2(in)
int ifft2_c2c(const float2* in, int n0, int n1, int centred, int crop0, int crop1,
              double scale, int real_only, void* out, cudaStream_t st) {
    const int rc = ifft2_size_check("ifft2", n0, n1);
    if (rc) return rc;
    if (crop0 <= 0 || crop0 > n0) crop0 = n0;
    if (crop1 <= 0 || crop1 > n1) crop1 = n1;
    return ifft2_planes(in, 1, n0, n1, centred, crop0, crop1, [&](int, double den) {
        return CropStore{real_only ? nullptr : (float2*)out, real_only ? (float*)out : nullptr,
                         crop1, (float)(scale / den)};
    }, st);
}

// --------------------------------------------------------------------------
// ththmod.chisq_calc over a grid of curvatures (ththmod.py:330-368 with modeler
// :261-327): per curvature the cropped theta-theta matrix, its top eigenpair, the
// rank-1 model scattered back into the conjugate spectrum, ifft2(ifftshift(.)) and
// sum over the mask of (model[:nf, :nt] - dspec)^2.  One launch sequence per batch of
// curvatures, no host synchronisation.
// --------------------------------------------------------------------------
// fp64 partial sums per curvature; consecutive columns go to different slots so that the
// atomics of one warp never meet on one address
constexpr int CHISQ_SLOTS = 64;

// base store of ifft2_planes: adds (scale re(v) - dspec)^2 to the partial sums where the
// mask is set (mask == nullptr: where dspec is finite), so the model is never written
struct ResidualSink {
    const float* dspec;            // [nf][nt]
    const unsigned char* mask;     // [nf][nt] or null
    int nf, nt;
    double* part;                  // [CHISQ_SLOTS]
    float scale;
    __device__ __forceinline__ void operator()(int row, int c, float2 v) const {
        const size_t o = (size_t)row * nt + c;
        const float d = dspec[o];
        if (mask ? !mask[o] : !isfinite(d)) return;
        const double r = (double)(v.x * scale) - (double)d;
        atomicAdd(part + (o % CHISQ_SLOTS), r * r);
    }
};
__global__ void chisq_finish_kernel(const double* __restrict__ part, int e0, int nb,
                                    const int* __restrict__ status, double* __restrict__ ssq) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nb) return;
    double s = 0.0;
    for (int k = 0; k < CHISQ_SLOTS; ++k) s += part[(size_t)e * CHISQ_SLOTS + k];
    // the reference raises for these curvatures (IndexError, ARPACK error, n < 3)
    ssq[e0 + e] = (status[e0 + e] & ETA_NO_EIGENPAIR) ? __longlong_as_double(0x7ff8000000000000LL) : s;
}

int chisq_sweep(const ThthGeom& g, const double* th_host, const double* d_etas, int neta,
                const double* d_th_red, double dtau_bin, double dfd_bin, const float* dspec,
                const unsigned char* mask, int nf, int nt, double tol, int max_iter,
                double* d_ssq, double* d_w, int* d_status, int* d_nred, int* d_iters,
                cudaStream_t st) {
    if (g.n > 4096) {
        set_error("chisq_sweep: theta-theta grid of %d centres exceeds the supported 4096", g.n);
        return SB_ERR_UNSUPPORTED;
    }
    const int n0 = (int)g.ntau, n1 = (int)g.nfd;
    if (nf < 1 || nt < 1 || nf > n0 || nt > n1) {
        set_error("chisq_sweep: dynamic spectrum %d x %d is empty or larger than the conjugate "
                  "spectrum %d x %d", nf, nt, n0, n1);
        return SB_ERR_ARG;
    }
    if (!(dtau_bin > 0.0) || !(dfd_bin > 0.0)) {
        set_error("chisq_sweep needs ascending tau / fd axes (bins must increase monotonically)");
        return SB_ERR_ARG;
    }
    int rc = ifft2_size_check("chisq_sweep", n0, n1);
    if (rc) return rc;
    if (neta <= 0) return SB_OK;
    const int ld = (g.n + 31) / 32 * 32;
    size_t smem;
    rc = eigvec_setup(herm_eigvec_batch_kernel, ld, &tol, &max_iter, &smem);
    if (rc) return rc;
    int* d_idx = (int*)workspace(WS_INDEX, (size_t)neta * ld * sizeof(int));
    if (!d_idx) return SB_ERR_NOMEM;
    rc = thth_prep(g, th_host, d_etas, neta, ld, d_idx, d_nred, d_status, st);
    if (rc) return rc;
    ThthCopy copy;
    rc = thth_gather_source(g, th_host, neta, &copy, st);
    if (rc) return rc;
    // per curvature: matrix, Lanczos basis, eigenvector, bin sums, partial sums, counts
    // (+ the row-transformed spectrum on the radix path), all under the sweep's slab budget
    const bool pow2 = is_pow2(n0) && is_pow2(n1);
    const size_t bins = (size_t)n0 * n1;
    const size_t mat = (size_t)ld * ld, qn = (size_t)(max_iter + 1) * ld;
    const size_t per = (mat + qn + ld + bins) * sizeof(float2) + CHISQ_SLOTS * sizeof(double) +
                       bins * sizeof(int) + (pow2 ? bins * sizeof(float2) : 0);
    const int batch = sweep_batch(per, neta, 65535);
    unsigned char* ws = (unsigned char*)workspace(WS_BATCH, per * batch);
    if (!ws) return SB_ERR_NOMEM;
    float2* M = (float2*)ws;
    float2* Q = M + mat * batch;
    float2* V = Q + qn * batch;
    float2* acc = V + (size_t)ld * batch;
    double* part = (double*)(acc + bins * batch);
    int* cnt = (int*)(part + (size_t)CHISQ_SLOTS * batch);
    // rev_map bins: tau[0], tau[1] - tau[0], fd[0], fd[1] - fd[0] (ththmod.py:210-215)
    const RevGeom rg{nullptr, 0, 0.0, g.tau0, dtau_bin, g.fd0, dfd_bin, n0, n1};
    int sb_ = (int)((mat + 255) / 256), fb = (int)((bins + 255) / 256);
    sb_ = sb_ > 256 ? 256 : sb_;
    fb = fb > 1024 ? 1024 : fb;
    for (int e0 = 0; e0 < neta; e0 += batch) {
        const int nb = neta - e0 < batch ? neta - e0 : batch;
        rc = thth_build_f32(g, copy, d_etas, e0, nb, ld, d_idx, d_nred, M, st);
        if (rc) return rc;
        herm_eigvec_batch_kernel<<<nb, EV_THREADS, smem, st>>>(M, ld, d_nred, e0, Q, max_iter, tol,
                                                              d_w, V, d_status, d_iters);
        SB_LAUNCH_CHECK();
        SB_CUDA(cudaMemsetAsync(acc, 0, bins * nb * sizeof(float2), st));
        SB_CUDA(cudaMemsetAsync(cnt, 0, bins * nb * sizeof(int), st));
        SB_CUDA(cudaMemsetAsync(part, 0, (size_t)CHISQ_SLOTS * nb * sizeof(double), st));
        rev_scatter_rank1_kernel<<<dim3(sb_, nb), 256, 0, st>>>(rg, d_th_red, g.n, d_etas, e0, d_nred,
                                                               d_status, d_w, V, ld, acc, cnt);
        SB_LAUNCH_CHECK();
        rev_finalise_batch_kernel<<<dim3(fb, nb), 256, 0, st>>>(rg, acc, cnt);
        SB_LAUNCH_CHECK();
        rc = ifft2_planes(acc, nb, n0, n1, 1, nf, nt, [&](int e, double den) {
            return ResidualSink{dspec, mask, nf, nt, part + (size_t)CHISQ_SLOTS * e,
                                (float)(1.0 / den)};
        }, st);
        if (rc) return rc;
        chisq_finish_kernel<<<(nb + 127) / 128, 128, 0, st>>>(part, e0, nb, d_status, d_ssq);
        SB_LAUNCH_CHECK();
    }
    return thth_gather_check(copy, st);
}

// --------------------------------------------------------------------------
// Gerchberg-Saxton iterations on a wavefield (Dynspec.gerchberg_saxton,
// dynspec.py:1883-1896): fft2 -> zero the tau < 0 rows -> ifft2 -> put the
// measured amplitude back where it is known.  fftshift / ifftshift cancel, so
// the causality mask is applied to the unshifted rows; mask and amplitude are
// fused into the final stores of the two column passes.
// --------------------------------------------------------------------------
template <typename C> struct RowMaskStore {     // out[k][c] = rowmask[k] ? 0 : v,  k = k1 + R1 k2
    C* out;
    long pitch;
    int R1;
    const unsigned char* rowmask;
    __device__ __forceinline__ void operator()(int y, int k, int c, C v) const {
        const int row = y + R1 * k;
        if (rowmask[row]) v.x = v.y = 0;
        out[(size_t)row * pitch + c] = v;
    }
};
__device__ __forceinline__ float gs_hypot(float x, float y) { return hypotf(x, y); }
__device__ __forceinline__ double gs_hypot(double x, double y) { return hypot(x, y); }
// w = v / (n0 n1); where amp is not NaN: amp * exp(i angle(w))
template <typename T> struct AmplitudeStore {
    cx<T>* out;
    long pitch;
    int R1;
    const float* amp;
    T scale;
    __device__ __forceinline__ void operator()(int y, int k, int c, cx<T> v) const {
        const int row = y + R1 * k;
        const size_t o = (size_t)row * pitch + c;
        cx<T> w = mkc<T>(v.x * scale, v.y * scale);
        const T a = amp[o];
        if (a == a) {
            const T m = gs_hypot(w.x, w.y);
            w = (m > (T)0) ? mkc<T>(a * (w.x / m), a * (w.y / m)) : mkc<T>(a, (T)0);
        }
        out[o] = w;
    }
};

// ---- any-size variant on the chirp-z inverse (fp32; tests/test_gpu_fft_lengths.py holds
// one iteration to a float64 loop at sizes up to 32768 x 8192):
//   T = ifft2(conj W) = conj(fft2 W) / N;  zero the masked rows of T;
//   W = N * ifft2(conj T) = ifft2(masked fft2 W);  amplitude step.
__global__ void gs_rowmask_kernel(float2* T, const unsigned char* __restrict__ rowmask,
                                  long n0, long n1) {
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < n0 * n1;
         o += (long)gridDim.x * blockDim.x)
        if (rowmask[o / n1]) T[o] = make_float2(0.f, 0.f);
}
__global__ void gs_amplitude_kernel(float2* W, const float* __restrict__ amp, long count) {
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < count;
         o += (long)gridDim.x * blockDim.x) {
        const float a = amp[o];
        if (a == a) {
            const float2 w = W[o];
            const float m = hypotf(w.x, w.y);
            W[o] = (m > 0.f) ? make_float2(a * (w.x / m), a * (w.y / m)) : make_float2(a, 0.f);
        }
    }
}
static int gerchberg_saxton_any(float2* W, const float* amp, const unsigned char* rowmask,
                                int n0, int n1, int niter, cudaStream_t st) {
    // the limits of ifft2_conj_any, checked before the workspace is allocated
    if (n0 < 3 || n1 < 3 || n0 > 32768 || n1 > 8192) {
        set_error("gerchberg_saxton (chirp-z): wavefield %d x %d outside 3..32768 x 3..8192",
                  n0, n1);
        return SB_ERR_UNSUPPORTED;
    }
    const long count = (long)n0 * n1;
    float2* T = (float2*)workspace(WS_BATCH, (size_t)count * sizeof(float2));
    if (!T) return SB_ERR_NOMEM;
    int blocks = (int)((count + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    for (int it = 0; it < niter; ++it) {
        int rc = ifft2_conj_any(W, n0, n1, 1.0, T, st);
        if (rc) return rc;
        gs_rowmask_kernel<<<blocks, 256, 0, st>>>(T, rowmask, n0, n1);
        SB_LAUNCH_CHECK();
        rc = ifft2_conj_any(T, n0, n1, (double)count, W, st);
        if (rc) return rc;
        gs_amplitude_kernel<<<blocks, 256, 0, st>>>(W, amp, count);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

template <typename A, typename B>
__global__ void gs_convert_kernel(const A* __restrict__ a, B* __restrict__ b, long n) {
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < n; o += (long)gridDim.x * blockDim.x)
        b[o] = (B)a[o];
}
// niter iterations on a power-of-two wavefield W in precision T; B: three scratch arrays
template <typename T>
static int gs_pow2(cx<T>* W, const float* amp, const unsigned char* rowmask, int n0, int n1,
                   int niter, cx<T>* const* B, cudaStream_t st) {
    using C = cx<T>;
    int R1, R2;
    split_len(n0, &R1, &R2);
    for (int it = 0; it < niter; ++it) {
        int rc = SB_OK;
        PitchRowLoad<C> l0{W, n1};
        PlainRowStore<C> s1{B[0], n1};
        SB_ROW_DISPATCH(n1, rc = (launch_row_c2c<T, N1, N2, -1>(l0, s1, n0, st)));
        if (rc) return rc;
        StrideALoad<C> la{B[0], n1, R2};
        RowMaskStore<C> ms{B[2], n1, R1, rowmask};
        rc = cols_generic<T, -1>(la, B[1], n1, n0, n1, ms, st);
        if (rc) return rc;
        PitchRowLoad<C> l3{B[2], n1};
        SB_ROW_DISPATCH(n1, rc = (launch_row_c2c<T, N1, N2, +1>(l3, s1, n0, st)));
        if (rc) return rc;
        AmplitudeStore<T> as{W, n1, R1, amp, (T)(1.0 / ((double)n0 * (double)n1))};
        rc = cols_generic<T, +1>(la, B[1], n1, n0, n1, as, st);
        if (rc) return rc;
    }
    return SB_OK;
}

int gerchberg_saxton(float2* W, const float* amp, const unsigned char* rowmask, int n0, int n1,
                     int niter, cudaStream_t st) {
    if ((n0 & (n0 - 1)) || (n1 & (n1 - 1)))
        return gerchberg_saxton_any(W, amp, rowmask, n0, n1, niter, st);
    // checked before any workspace is allocated; rows as in ifft2_c2c (8..16384 points)
    if (n0 < 8 || n1 < 8 || n0 > 65536 || n1 > 16384) {
        set_error("gerchberg_saxton: power-of-two wavefield %d x %d outside 8..65536 x 8..16384",
                  n0, n1);
        return SB_ERR_UNSUPPORTED;
    }
    if (n1 > 8192) {                  // fp64 rows of this length do not fit shared memory
        const WsSlot slot[3] = {WS_PLANE0, WS_PLANE1, WS_PLANE2};
        float2* B[3];
        for (int i = 0; i < 3; ++i)
            if (!(B[i] = (float2*)workspace(slot[i], (size_t)n0 * n1 * sizeof(float2)))) return SB_ERR_NOMEM;
        return gs_pow2<float>(W, amp, rowmask, n0, n1, niter, B, st);
    }
    // fp64 iterations: the phase step divides by |w|, so where |w| is small it amplifies the
    // rounding of the transforms; with fp32 transforms that reaches 1e-5 of the wavefield's
    // scale within three iterations on random input
    const WsSlot slot[4] = {WS_BATCH, WS_PLANE0, WS_PLANE1, WS_PLANE2};
    double2* B[4];
    for (int i = 0; i < 4; ++i)
        if (!(B[i] = (double2*)workspace(slot[i], (size_t)n0 * n1 * sizeof(double2)))) return SB_ERR_NOMEM;
    const long count = 2L * n0 * n1;
    int blocks = (int)((count + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    gs_convert_kernel<<<blocks, 256, 0, st>>>((const float*)W, (double*)B[3], count);
    SB_LAUNCH_CHECK();
    const int rc = gs_pow2<double>(B[3], amp, rowmask, n0, n1, niter, B, st);
    if (rc) return rc;
    gs_convert_kernel<<<blocks, 256, 0, st>>>((const double*)B[3], (float*)W, count);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// --------------------------------------------------------------------------
// Conjugate spectrum of a complex chunk (the visibilities of VLBI_chunk_retrieval,
// ththmod.py:1313-1325): pad to NF x NT, fft2, fftshift, zero the masked tau rows.
// The padded chunk is materialised; power-of-two sizes run the radix rows and columns
// forwards, other sizes the chirp-z inverse on the conjugate (fft2(x) = conj(N ifft2(conj x))).
// --------------------------------------------------------------------------
__global__ void c2c_sum_kernel(const float2* __restrict__ in, long count, double* __restrict__ sum) {
    double sx = 0.0, sy = 0.0;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < count;
         o += (long)gridDim.x * blockDim.x) {
        sx += in[o].x;
        sy += in[o].y;
    }
    sx = warp_sum(sx);
    sy = warp_sum(sy);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(sum, sx);
        atomicAdd(sum + 1, sy);
    }
}
// P [NF][NT]: the chunk in the first nf x nt corner, pad elsewhere (sum != null: the mean)
__global__ void c2c_pad_kernel(const float2* __restrict__ in, int nf, int nt, int NF, int NT,
                               float2 pad, const double* __restrict__ sum, float2* __restrict__ P) {
    if (sum) {
        const double cnt = (double)nf * (double)nt;
        pad = make_float2((float)(sum[0] / cnt), (float)(sum[1] / cnt));
    }
    const long total = (long)NF * NT;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < total;
         o += (long)gridDim.x * blockDim.x) {
        const int r = (int)(o / NT), c = (int)(o - (long)r * NT);
        P[o] = (r < nf && c < nt) ? in[(size_t)r * nt + c] : pad;
    }
}
struct CsShiftStore {     // CS[fftshift(k)][fftshift(c)] = v, masked rows zero (powers of two)
    float2* CS;
    int NF, NT, R1;
    const unsigned char* rowmask;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int rs = (y + R1 * k + NF / 2) & (NF - 1), cs = (c + NT / 2) & (NT - 1);
        CS[(size_t)rs * NT + cs] = (rowmask && rowmask[rs]) ? make_float2(0.f, 0.f) : v;
    }
};
// CS = fftshift(conj(T)), masked rows zero (any size)
__global__ void c2c_shift_conj_kernel(const float2* __restrict__ T, int NF, int NT,
                                      const unsigned char* __restrict__ rowmask,
                                      float2* __restrict__ CS) {
    const long total = (long)NF * NT;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < total;
         o += (long)gridDim.x * blockDim.x) {
        const int r = (int)(o / NT), c = (int)(o - (long)r * NT);
        const int rs = (r + NF / 2) % NF, cs = (c + NT / 2) % NT;
        const float2 t = T[o];
        CS[(size_t)rs * NT + cs] =
            (rowmask && rowmask[rs]) ? make_float2(0.f, 0.f) : make_float2(t.x, -t.y);
    }
}

int conj_spectrum_c2c(const float2* in, int nf, int nt, int npad, float pad_re, float pad_im,
                      const unsigned char* rowmask, float2* CS, cudaStream_t st) {
    const long NFl = (long)(npad + 1) * nf, NTl = (long)(npad + 1) * nt;
    // a complex row is one row transform of NT points (8..16384), unlike the real input's
    // half-length rows; the chirp-z path has the limits of ifft2_conj_any
    const bool radix = is_pow2(NFl) && is_pow2(NTl) && NFl >= 8 && NTl >= 8 && NFl <= 65536 &&
                       NTl <= 16384;
    if (!radix && (NFl < 3 || NTl < 3 || NFl > 32768 || NTl > 8192)) {
        set_error("conjugate spectrum (complex input): padded size %ldx%ld outside 8..65536 x "
                  "8..16384 (powers of two) / 3..32768 x 3..8192 (other sizes)", NFl, NTl);
        return SB_ERR_UNSUPPORTED;
    }
    const int NF = (int)NFl, NT = (int)NTl;
    const size_t count = (size_t)NF * NT;
    ScalarBlock* sc = scalar_block();
    if (!sc) return SB_ERR_NOMEM;
    double* sum = sc->c2c_sum;
    float2* P = (float2*)workspace(WS_BATCH, count * sizeof(float2));
    if (!P) return SB_ERR_NOMEM;
    int blocks = (int)((count + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    const bool dev_mean = pad_re != pad_re;
    if (dev_mean) {
        SB_CUDA(cudaMemsetAsync(sum, 0, sizeof(sc->c2c_sum), st));
        c2c_sum_kernel<<<num_sms() * 4, 256, 0, st>>>(in, (long)nf * nt, sum);
        SB_LAUNCH_CHECK();
    }
    c2c_pad_kernel<<<blocks, 256, 0, st>>>(in, nf, nt, NF, NT, make_float2(pad_re, pad_im),
                                           dev_mean ? sum : nullptr, P);
    SB_LAUNCH_CHECK();
    if (radix) {
        float2* B1 = (float2*)workspace(WS_PLANE0, count * sizeof(float2));
        float2* B2 = (float2*)workspace(WS_PLANE1, count * sizeof(float2));
        if (!B1 || !B2) return SB_ERR_NOMEM;
        int rc = SB_OK;
        PitchRowLoad<float2> lr{P, NT};
        PlainRowStore<float2> rs{B1, NT};
        SB_ROW_DISPATCH(NT, rc = (launch_row_c2c<float, N1, N2, -1>(lr, rs, NF, st)));
        if (rc) return rc;
        int R1, R2;
        split_len(NF, &R1, &R2);
        StrideALoad<float2> la{B1, NT, R2};
        return cols_generic<float, -1>(la, B2, NT, NF, NT, CsShiftStore{CS, NF, NT, R1, rowmask},
                                       st);
    }
    float2* T = (float2*)workspace(WS_INDEX, count * sizeof(float2));
    if (!T) return SB_ERR_NOMEM;
    const int rc = ifft2_conj_any(P, NF, NT, (double)count, T, st);
    if (rc) return rc;
    c2c_shift_conj_kernel<<<blocks, 256, 0, st>>>(T, NF, NT, rowmask, CS);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// --------------------------------------------------------------------------
// VLBI_chunk_retrieval for one chunk, steps 3-6 (ththmod.py:1310-1383): crop, composite
// gather, eigenpair, per-station rev_map of row n//2, ifft2(ifftshift(.)) cropped to
// nf x nt and scaled by nf nt / 4.  No host synchronisation.
// --------------------------------------------------------------------------
constexpr int VLBI_PTRS = 64;
struct VlbiArgs {          // device copies of eta and of a run of spectrum pointers
    const float2* cs[VLBI_PTRS];
    int base, count;
    double eta;
};
__global__ void vlbi_args_kernel(VlbiArgs a, const float2** cs, double* eta) {
    if ((int)threadIdx.x < a.count) cs[a.base + threadIdx.x] = a.cs[threadIdx.x];
    if (threadIdx.x == 0 && a.base == 0) *eta = a.eta;
}

int vlbi_retrieval(const ThthGeom& geom, const double* th_host, const float2* const* cs_host,
                   int n_dish, double eta, const double* d_th_red, double dtau_bin,
                   double dfd_bin, int nf, int nt, double tol, int max_iter, float2* d_model,
                   double* d_w, float2* d_v, int* d_info, cudaStream_t st) {
    // every spectrum is a dense, complex, full-plane [ntau][nfd] array: the layout and
    // mode fields of the caller's geometry do not apply
    ThthGeom g = geom;
    g.cs = nullptr;
    g.cs_pitch = g.nfd;
    g.cs_valid_cols = 0;
    g.cs_bound = nullptr;
    g.coherent = 1;
    const int n0 = (int)g.ntau, n1 = (int)g.nfd;
    if (n_dish < 1) {
        set_error("vlbi_retrieval: n_dish = %d, needs at least one station", n_dish);
        return SB_ERR_ARG;
    }
    if (nf < 1 || nt < 1 || nf > n0 || nt > n1) {
        set_error("vlbi_retrieval: chunk %d x %d is empty or larger than the conjugate "
                  "spectrum %d x %d", nf, nt, n0, n1);
        return SB_ERR_ARG;
    }
    if (!(dtau_bin > 0.0) || !(dfd_bin > 0.0)) {
        set_error("vlbi_retrieval needs ascending tau / fd axes (bins must increase monotonically)");
        return SB_ERR_ARG;
    }
    if (g.cs_half) {
        set_error("vlbi_retrieval needs full-plane conjugate spectra");
        return SB_ERR_ARG;
    }
    const int npairs = n_dish * (n_dish + 1) / 2;
    for (int k = 0; k < npairs; ++k)
        if (!cs_host[k]) {
            set_error("vlbi_retrieval: conjugate spectrum %d is null", k);
            return SB_ERR_ARG;
        }
    // cropped size: the mask of thth_prep_kernel with the same (exactly rounded) expressions
    int n = 0;
    for (int k = 0; k < g.n; ++k) {
        const double t = th_host[k];
        if ((t * t) * eta < g.tau_absmax && fabs(t) < g.fd_half) ++n;
    }
    const long N = (long)n_dish * n;
    if (N > 8192) {
        set_error("vlbi_retrieval: composite theta-theta matrix of %d stations x %d centres = %ld "
                  "exceeds the eigen solver's limit of 8192", n_dish, n, N);
        return SB_ERR_UNSUPPORTED;
    }
    int rc = ifft2_size_check("vlbi_retrieval", n0, n1);
    if (rc) return rc;
    size_t smem;
    rc = eigvec_setup(vlbi_eigvec_kernel, (int)N, &tol, &max_iter, &smem);
    if (rc) return rc;
    const size_t bins = (size_t)n0 * n1;
    const size_t qn = (size_t)(max_iter + 1) * (N > 0 ? N : 1);
    // s1: eta, spectrum pointers, crop indices; s2: composite, Lanczos basis, per-station bin
    // sums, shared bin counts
    unsigned char* s1 = (unsigned char*)workspace(
        WS_INDEX, sizeof(double) + (size_t)npairs * sizeof(float2*) + (size_t)g.n * sizeof(int));
    unsigned char* s2 = (unsigned char*)workspace(
        WS_BATCH, ((size_t)N * N + qn + (size_t)n_dish * bins) * sizeof(float2) + bins * sizeof(int));
    if (!s1 || !s2) return SB_ERR_NOMEM;
    double* d_eta = (double*)s1;
    const float2** d_cs = (const float2**)(d_eta + 1);
    int* d_idx = (int*)(d_cs + npairs);
    float2* A = (float2*)s2;
    float2* Q = A + (size_t)N * N;
    float2* acc = Q + qn;
    int* cnt = (int*)(acc + (size_t)n_dish * bins);
    for (int b = 0; b < npairs; b += VLBI_PTRS) {
        VlbiArgs a;
        a.base = b;
        a.count = npairs - b < VLBI_PTRS ? npairs - b : VLBI_PTRS;
        a.eta = eta;
        for (int k = 0; k < a.count; ++k) a.cs[k] = cs_host[b + k];
        vlbi_args_kernel<<<1, VLBI_PTRS, 0, st>>>(a, d_cs, d_eta);
        SB_LAUNCH_CHECK();
    }
    rc = thth_prep(g, th_host, d_eta, 1, g.n, d_idx, d_info + 2, d_info + 1, st);
    if (rc) return rc;
    if (N > 0) {
        int blocks = (int)((N * N + 255) / 256);
        if (blocks > num_sms() * 16) blocks = num_sms() * 16;
        vlbi_composite_kernel<<<blocks, 256, 0, st>>>(g, d_eta, d_cs, n_dish, d_idx, n, A);
        SB_LAUNCH_CHECK();
    }
    vlbi_eigvec_kernel<<<1, EV_THREADS, smem, st>>>(A, n_dish, n, Q, max_iter, tol, d_w, d_v,
                                                    d_info);
    SB_LAUNCH_CHECK();
    SB_CUDA(cudaMemsetAsync(acc, 0, (size_t)n_dish * bins * sizeof(float2), st));
    SB_CUDA(cudaMemsetAsync(cnt, 0, bins * sizeof(int), st));
    // rev_map bins: tau[0], tau[1] - tau[0], fd[0], fd[1] - fd[0] (ththmod.py:210-215)
    const RevGeom rg{d_th_red, n, eta, g.tau0, dtau_bin, g.fd0, dfd_bin, n0, n1};
    if (n > 0) {
        int sb_ = (int)(((size_t)n * n + 255) / 256);
        sb_ = sb_ > 256 ? 256 : sb_;
        vlbi_scatter_kernel<<<dim3(sb_, n_dish + 1), 256, 0, st>>>(rg, n_dish, d_info, d_w, d_v,
                                                                   acc, cnt);
        SB_LAUNCH_CHECK();
    }
    int fb = (int)((bins + 255) / 256);
    fb = fb > 1024 ? 1024 : fb;
    vlbi_finalise_kernel<<<dim3(fb, n_dish), 256, 0, st>>>(rg, acc, cnt);
    SB_LAUNCH_CHECK();
    const double scale = (double)nf * (double)nt / 4.0;
    return ifft2_planes(acc, n_dish, n0, n1, 1, nf, nt, [&](int d, double den) {
        return CropStore{d_model + (size_t)nf * nt * d, nullptr, nt, (float)(scale / den)};
    }, st);
}

// --------------------------------------------------------------------------
// calc_asymmetry over nchunk chunks after their spectra (ththmod.py:2385-2463): crop and
// gather, top eigenpair, asymmetry of V.  Chunks run in batches under the sweep's slab
// budget; one launch sequence, no host synchronisation, nchunk numbers per output.
// --------------------------------------------------------------------------
int asymmetry_batch(const ThthGeom* geoms, const double* const* th_host, int nchunk,
                    const double* d_etas, double tol, int max_iter, double* d_asym, double* d_w,
                    int* d_status, int* d_nred, int* d_iters, float2* d_v, cudaStream_t st) {
    if (nchunk <= 0) return SB_OK;
    const ThthGeom& g0 = geoms[0];
    for (int k = 0; k < nchunk; ++k) {
        const ThthGeom& g = geoms[k];
        if (!g.cs) {
            set_error("asymmetry_batch: conjugate spectrum of chunk %d is null", k);
            return SB_ERR_ARG;
        }
        if (g.ntau != g0.ntau || g.nfd != g0.nfd || g.n != g0.n || g.cs_half != g0.cs_half ||
            g.cs_pitch != g0.cs_pitch || g.cs_valid_cols != g0.cs_valid_cols ||
            g.coherent != g0.coherent) {
            set_error("asymmetry_batch: chunk %d differs from chunk 0 in spectrum size, theta "
                      "grid size or spectrum layout", k);
            return SB_ERR_ARG;
        }
    }
    if (g0.n > 4096) {
        set_error("asymmetry_batch: theta-theta grid of %d centres exceeds the supported 4096",
                  g0.n);
        return SB_ERR_UNSUPPORTED;
    }
    // the spectra sb_cs_f32 makes: powers of two up to 65536 x 32768 (radix path, full or
    // half plane), any other size in 3..32768 x 3..8192 (chirp-z path, full plane)
    const long long n0 = g0.ntau, n1 = g0.nfd;
    const bool radix = is_pow2(n0) && is_pow2(n1) && n0 >= 4 && n1 >= 16;
    if (radix ? (n0 > 65536 || n1 > 32768)
              : (g0.cs_half || n0 < 3 || n1 < 3 || n0 > 32768 || n1 > 8192)) {
        set_error("asymmetry_batch: conjugate spectrum %lld x %lld outside 4..65536 x 16..32768 "
                  "(powers of two) / 3..32768 x 3..8192 (other sizes, full plane)", n0, n1);
        return SB_ERR_UNSUPPORTED;
    }
    const int ld = (g0.n + 31) / 32 * 32;
    size_t smem;
    int rc = eigvec_setup(herm_eigvec_batch_kernel, ld, &tol, &max_iter, &smem);
    if (rc) return rc;
    // per chunk: matrix, Lanczos basis, eigenvector, under the sweep's slab budget
    const size_t mat = (size_t)ld * ld, qn = (size_t)(max_iter + 1) * ld;
    const size_t per = (mat + qn + ld) * sizeof(float2);
    const int batch = sweep_batch(per, nchunk, 65535);
    // s1: geometry table and crop indices; s2: the batch's matrices, bases, vectors
    const size_t tab = ((size_t)nchunk * sizeof(ThthGeom) + 255) / 256 * 256;
    unsigned char* s1 = (unsigned char*)workspace(WS_INDEX, tab + (size_t)nchunk * ld * sizeof(int));
    unsigned char* s2 = (unsigned char*)workspace(WS_BATCH, per * batch);
    if (!s1 || !s2) return SB_ERR_NOMEM;
    ThthGeom* d_geoms = (ThthGeom*)s1;
    int* d_idx = (int*)(s1 + tab);
    float2* M = (float2*)s2;
    float2* Q = M + mat * batch;
    float2* V = Q + qn * batch;
    SB_CUDA(cudaMemcpyAsync(d_geoms, geoms, (size_t)nchunk * sizeof(ThthGeom),
                            cudaMemcpyHostToDevice, st));
    rc = thth_prep_table(geoms, th_host, d_geoms, d_etas, nchunk, ld, d_idx, d_nred, d_status, st);
    if (rc) return rc;
    int gb = (int)((mat + 255) / 256);
    gb = gb > 32 ? 32 : gb;
    for (int e0 = 0; e0 < nchunk; e0 += batch) {
        const int nb = nchunk - e0 < batch ? nchunk - e0 : batch;
        asym_gather_kernel<<<dim3(gb, nb), 256, 0, st>>>(d_geoms, d_etas, e0, ld, d_idx, d_nred, M);
        SB_LAUNCH_CHECK();
        herm_eigvec_batch_kernel<<<nb, EV_THREADS, smem, st>>>(M, ld, d_nred, e0, Q, max_iter, tol,
                                                              d_w, V, d_status, d_iters);
        SB_LAUNCH_CHECK();
        asym_finish_kernel<<<nb, 32, 0, st>>>(V, ld, d_nred, d_status, e0, d_asym, d_v);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
