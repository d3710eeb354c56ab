// Lanczos bookkeeping shared by the square (thth.cu) and the thin (thin.cu)
// theta-theta solvers: tridiagonal storage, division-free Sturm counts, warp
// multisection for the top Ritz values and the residual / gap stopping rule.
#pragma once
#include <float.h>

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

}  // namespace sb
