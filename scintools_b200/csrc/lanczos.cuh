// Lanczos pieces shared by the fp32 Lanczos solvers (thth_eig_kernel in thth.cu,
// thth_eig_half_kernel in eig_half.cu, thin_sv_kernel in thin.cu, herm_eigvec_body in
// retrieval.cu): tridiagonal storage and its reset, the CTA sum, the three-term step and
// the rotation, division-free Sturm counts, warp multisection for the top Ritz values, the
// residual / gap stopping rule and the Ritz coefficients.
#pragma once
#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace sb {

#define SB_LANCZOS_MAXIT 256

// The reserved members are unused.  They keep the size the struct had when a second
// check routine needed them: 2 KB less lets thin_sv_kernel (128 registers, 256 threads)
// fit two CTAs per SM instead of one at 3008 .. 3072 theta1 columns, which is not measured.
struct alignas(16) LanczosShared {
    double alpha[SB_LANCZOS_MAXIT];
    double beta[SB_LANCZOS_MAXIT + 1];
    double beta2[SB_LANCZOS_MAXIT + 1];
    double piv[SB_LANCZOS_MAXIT];
    double reserved0[SB_LANCZOS_MAXIT];
    double red[2][32];
    double theta, lo, res;
    double reserved1;
    int done, next_check;
    int reserved2;
    int m_last;              // lanczos_check: step of the previous check (0: none)
};

// State of a new run: not converged, first check after step 1.  Written by thread 0; the
// caller's next barrier publishes it.
__device__ __forceinline__ void lanczos_reset(LanczosShared& S) {
    if (threadIdx.x == 0) {
        S.done = 0; S.lo = 0.0; S.theta = 0.0; S.res = 0.0;
        S.next_check = 1; S.m_last = 0; S.beta2[0] = 0.0;
    }
}

// First index of this thread in a loop strided over the threads of the first NW warps.
// Threads past them (eig_half.cu's check warp) start beyond every bound: their loops are empty.
template <int NW>
__device__ __forceinline__ int lanczos_first() {
    return threadIdx.x < NW * 32 ? (int)threadIdx.x : INT_MAX;
}

// fp64 sum of x over the first NW warps of the CTA, in a fixed order: warp_sum, then the
// warps 0 .. NW-1 through red[warp].  Every thread calls it (it holds a barrier) and gets
// the sum.  A barrier must separate it from the last read of red by an earlier sum.
template <int NW>
__device__ __forceinline__ double cta_sum(double x, double* red) {
    x = warp_sum(x);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
    __syncthreads();
    double s = 0.0;
    for (int k = 0; k < NW; ++k) s += red[k];
    return s;
}

// Step `it` of the three-term recurrence on fp32 vectors of length n, sums in fp64, once the
// mat-vec has left A v in w -- plus the column sums u of the triangle solvers, added first
// (null: none): alpha = Re <v, A v>, w = A v - alpha v - beta_prev vp, beta = ||w||, all
// three recorded in S.  Ends with a barrier.
template <int NW>
__device__ __forceinline__ void lanczos_step(LanczosShared& S, int it, int n, const float2* v,
                                             const float2* vp, float2* w, const float2* u,
                                             float beta_prev, double& alpha, double& beta) {
    const int c0 = lanczos_first<NW>();
    double apart = 0.0;
    for (int c = c0; c < n; c += NW * 32) {
        float2 x = w[c];
        if (u) {
            x.x += u[c].x;
            x.y += u[c].y;
            w[c] = x;
        }
        apart += (double)(v[c].x * x.x + v[c].y * x.y);
    }
    alpha = cta_sum<NW>(apart, S.red[0]);
    const float af = (float)alpha;
    double bpart = 0.0;
    for (int c = c0; c < n; c += NW * 32) {
        float2 x = w[c];
        x.x -= af * v[c].x + beta_prev * vp[c].x;
        x.y -= af * v[c].y + beta_prev * vp[c].y;
        w[c] = x;
        bpart += (double)x.x * x.x + (double)x.y * x.y;
    }
    const double b2 = cta_sum<NW>(bpart, S.red[1]);
    beta = sqrt(b2);
    if (threadIdx.x == 0) { S.alpha[it] = alpha; S.beta[it + 1] = beta; S.beta2[it + 1] = b2; }
    __syncthreads();
}

// vp = v, v = w / beta (elements 0 .. n-1).  Ends with a barrier.
template <int NW>
__device__ __forceinline__ void lanczos_rotate(float2* v, float2* vp, const float2* w, int n,
                                               double beta) {
    const float ib = (float)(1.0 / beta);
    for (int c = lanczos_first<NW>(); c < n; c += NW * 32) {
        const float2 x = w[c];
        vp[c] = v[c];
        v[c] = make_float2(x.x * ib, x.y * ib);
    }
    __syncthreads();
}

// Number of eigenvalues of the m x m tridiagonal (alpha[0..m), beta[1..m))
// below sigma = sign changes of the Sturm sequence q_0 = 1, q_1 = alpha_0 -
// sigma, q_{i+1} = (alpha_i - sigma) q_i - beta_i^2 q_{i-1}.  Division free;
// q is rescaled by powers of two when it drifts out of range.
__device__ __forceinline__ int sturm_count(const LanczosShared& S, int m, double sig) {
    double q0 = 1.0, q1 = S.alpha[0] - sig;
    bool neg = !(q1 > 0.0);          // a zero counts as a sign change
    int cnt = neg ? 1 : 0;
    for (int i = 1; i < m; ++i) {
        double q2 = (S.alpha[i] - sig) * q1 - S.beta2[i] * q0;
        const double aq = fabs(q2);
        if (aq > 1e140) { q2 *= 1e-140; q1 *= 1e-140; }
        else if (aq < 1e-140 && fabs(q1) < 1e-140) { q2 *= 1e140; q1 *= 1e140; }
        const bool neg2 = (q2 == 0.0) ? !neg : (q2 < 0.0);
        cnt += (neg2 != neg);
        neg = neg2;
        q0 = q1;
        q1 = q2;
    }
    return cnt;
}

// warp multisection: smallest sigma in (lo, hi] with count(sigma) >= want
__device__ __forceinline__ void sturm_multisect(const LanczosShared& S, int m,
                                                int want, double& lo, double& hi,
                                                int rounds) {
    const int lane = threadIdx.x & 31;
    for (int round = 0; round < rounds; ++round) {
        const double sig = lo + (hi - lo) * (double)(lane + 1) / 33.0;
        const int cnt = sturm_count(S, m, sig);
        const unsigned ok = __ballot_sync(0xffffffffu, cnt >= want);
        const int f = ok ? __ffs(ok) - 1 : 32;
        const double nhi = f < 32 ? __shfl_sync(0xffffffffu, sig, f & 31) : hi;
        const double nlo = f > 0 ? __shfl_sync(0xffffffffu, sig, (f - 1) & 31) : lo;
        hi = nhi;
        lo = nlo;
    }
}

// Largest Ritz value theta of T_m, residual bound beta[m]*|s_m| (last
// component of the Ritz vector through the ratios l_i = beta_{i+1} q_i /
// q_{i+1} of the Sturm sequence at theta), and -- once the residual is small
// -- the second Ritz value for the error estimate res^2/gap.  Converged when
// res <= tol*theta or res^2 <= etol*theta*gap.  Called by warp 0.
__device__ inline void lanczos_check(LanczosShared& S, int m, double tol, double etol) {
    const int lane = threadIdx.x & 31;
    __syncwarp();   // every lane has read S.next_check before lane 0 rewrites it below
    const double bnew = S.beta[m];
    double gh = -DBL_MAX, gl = DBL_MAX;
    for (int i = lane; i < m; i += 32) {
        double b0 = i > 0 ? fabs(S.beta[i]) : 0.0;
        double b1 = i + 1 < m ? fabs(S.beta[i + 1]) : 0.0;
        gh = fmax(gh, S.alpha[i] + b0 + b1);
        gl = fmin(gl, S.alpha[i] - b0 - b1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        gh = fmax(gh, __shfl_xor_sync(0xffffffffu, gh, o));
        gl = fmin(gl, __shfl_xor_sync(0xffffffffu, gl, o));
    }
    double hi = gh + 1e-9 * fabs(gh) + 1e-290;
    double lo = (m == 1) ? S.alpha[0] - fabs(S.alpha[0]) * 1e-9 - 1e-290 : S.lo;
    if (lo > hi) lo = hi - fabs(hi) - 1.0;
    sturm_multisect(S, m, m, lo, hi, 6);
    // Polish the upper bracket end to fp64 accuracy: Newton on p_m(x) = det(T_m - x) from
    // above the largest root converges monotonically and quadratically (two steps from a
    // 1e-9 bracket).  The residual estimate below is only as good as the shift is close to
    // the Ritz value: with the raw 1e-9 offset it bottoms out near 3e-5 |theta| (and grows
    // with m), which starved every caller that asks for less (herm_eigvec: 1e-7).
    double theta = hi;
    if (lane == 0 && m >= 2) {
        double x = hi;
        for (int nit = 0; nit < 3; ++nit) {
            double p0 = 1.0, p1 = S.alpha[0] - x, d0 = 0.0, d1 = -1.0;
            for (int i = 1; i < m; ++i) {
                const double a = S.alpha[i] - x, b2 = S.beta2[i];
                const double p2 = a * p1 - b2 * p0;
                const double d2 = a * d1 - p1 - b2 * d0;
                p0 = p1; p1 = p2; d0 = d1; d1 = d2;
                const double aq = fmax(fabs(p1), fabs(d1));
                if (aq > 1e140) { p0 *= 1e-140; p1 *= 1e-140; d0 *= 1e-140; d1 *= 1e-140; }
                else if (aq < 1e-140 && aq > 0.0) { p0 *= 1e140; p1 *= 1e140; d0 *= 1e140; d1 *= 1e140; }
            }
            const double step = (d1 != 0.0) ? p1 / d1 : 0.0;
            if (!(step > 0.0) || !(x - step >= lo)) break;     // not above the root any more
            x -= step;
        }
        theta = x;
    }
    theta = __shfl_sync(0xffffffffu, theta, 0);
    // ratios l_i at sigma = theta: lanes in parallel, then a product chain
    double res = 0.0;
    if (lane == 0) {
        double q0 = 1.0, q1 = S.alpha[0] - theta;
        for (int i = 1; i < m; ++i) {
            double q2 = (S.alpha[i] - theta) * q1 - S.beta2[i] * q0;
            // l_{i-1} = beta_i * q_{i-1}/q_i in pivot terms: beta_i / d_{i-1}, d = q1/q0.
            // Taken BEFORE the range rescaling below, which scales (q1, q2) but not q0:
            // with the ratio formed afterwards the first rescale (|q| > 1e140, i.e. step
            // ~20 for eigenvalues ~3e7) blew piv up by 1e140, the norm overflowed and the
            // residual came out as 0 -- a silent stop at m = 21 with an unconverged value
            // (round 1: up to 4e-3 off on 2.5 % of the 4096x8192 curvatures).
            S.piv[i - 1] = (q1 != 0.0) ? S.beta[i] * q0 / q1 : 1e300;
            const double aq = fabs(q2);
            if (aq > 1e140) { q2 *= 1e-140; q1 *= 1e-140; }
            else if (aq < 1e-140 && fabs(q1) < 1e-140) { q2 *= 1e140; q1 *= 1e140; }
            q0 = q1;
            q1 = q2;
        }
        double z = 1.0, nrm = 1.0;
        bool bad = false;
        for (int i = m - 2; i >= 0; --i) {
            z = -S.piv[i] * z;
            nrm += z * z;
            if (!(nrm < 1e200)) { bad = true; break; }
        }
        // numerical trouble must never read as "converged": no estimate -> keep iterating
        res = bad ? DBL_MAX : bnew * rsqrt(nrm);
    }
    res = __shfl_sync(0xffffffffu, res, 0);
    bool done = (res <= tol * fabs(theta)) || !(bnew > 1e-30 * fabs(theta));
    double gap_est = 0.0;
    if (!done && m >= 3 && res <= 3e-2 * fabs(theta)) {
        double lo2 = gl - 1e-9 * fabs(gl) - 1e-290, hi2 = theta;
        sturm_multisect(S, m, m - 1, lo2, hi2, 4);
        const double gap = theta - hi2;
        done = gap > 0.0 && res * res <= etol * fabs(theta) * gap;
        gap_est = gap;
    }
    // When is the next check worth its ~10 Sturm sweeps (the other warps idle
    // meanwhile)?  The residual decays roughly geometrically: extrapolate the rate
    // seen since the previous check to the residual the stopping rule needs and skip
    // half of the predicted remaining steps (at most 4).
    int skip = (res > 0.3 * fabs(theta)) ? 2 : 1;
    if (!done && S.m_last > 0 && m > S.m_last && S.res > 0.0 && res > 0.0 && res < S.res) {
        const double rate = log(res / S.res) / (double)(m - S.m_last);      // < 0 per step
        double target = tol * fabs(theta);
        if (gap_est > 0.0) target = fmax(target, sqrt(etol * fabs(theta) * gap_est));
        else target = fmax(target, sqrt(etol * 0.02) * fabs(theta));        // gap unknown yet
        if (res > target) {
            const double remaining = log(target / res) / rate;
            int sk = (int)(0.5 * remaining);
            sk = sk > 4 ? 4 : sk;
            skip = sk > skip ? sk : skip;
        }
    }
    __syncwarp();   // all lanes are done reading S.lo / S.next_check
    if (lane == 0) {
        S.theta = theta;
        S.lo = lo;
        S.res = res;
        S.done = done ? 1 : 0;
        S.m_last = m;
        S.next_check = m + skip;
    }
}

// Coefficients s_0 .. s_{m-1} of the unit Ritz vector of T_m at S.theta (y = sum_j s_j q_j)
// into S.piv: the backward recurrence from s_{m-1} = 1, which grows towards s_0 and is
// rescaled by 1e-150 whenever it passes 1e150.  Thread 0 computes; ends with a barrier.
__device__ __forceinline__ void lanczos_ritz(LanczosShared& S, int m) {
    if (threadIdx.x == 0) {
        const double theta = S.theta;
        double* s = S.piv;
        s[m - 1] = 1.0;
        if (m >= 2) s[m - 2] = (S.beta[m - 1] != 0.0) ? (theta - S.alpha[m - 1]) / S.beta[m - 1] : 0.0;
        for (int i = m - 2; i >= 1; --i) {
            const double t = (theta - S.alpha[i]) * s[i] - S.beta[i + 1] * s[i + 1];
            s[i - 1] = (S.beta[i] != 0.0) ? t / S.beta[i] : 0.0;
            if (fabs(s[i - 1]) > 1e150)
                for (int k = i - 1; k < m; ++k) s[k] *= 1e-150;
        }
        double nn = 0.0;
        for (int i = 0; i < m; ++i) nn += s[i] * s[i];
        nn = 1.0 / sqrt(nn);
        for (int i = 0; i < m; ++i) s[i] *= nn;
    }
    __syncthreads();
}

}  // namespace sb
