// Dynspec.norm_sspec (scintools/dynspec.py:2076-2183): every delay row of the
// secondary spectrum is resampled with numpy.interp onto the normalised
// Doppler axis fdop / sqrt(tdel / eta), then scrunched over delay with weights.
// This is the per-row gather + linear interpolation that feeds fit_arc's
// power-vs-curvature profile (:1156-1180).
//
//   row ii :  s = sqrt(tdel[ii] / eta);  sel = |fdop| <= maxnormfac * s
//             normline = np.interp(fdopnew, fdop[sel] / s, sspec[ii, sel])
//             mask     = |fdopnew| > max|fdop[sel] / s|   (or NaN result)
//   powerspectrum[ii] = masked mean of 10^(normline / 10), finite samples only (:2127)
//   normsspecavg[j]   = masked weighted average over the rows         (:2166)
//
// All axis arithmetic is fp64 with numpy's own expressions (same selections,
// same interval search results as np.interp); the samples are fp32 (dB).
// HBM-bound gather: nr * nq outputs of 4 B, each from two neighbouring samples
// of an L1/L2-resident row.
#include <math.h>

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

// np.interp of one point on the selected, scaled row: xp[k] = fdop[lo + k] / s
__device__ __forceinline__ double interp_one(const float* __restrict__ row,
                                             const double* __restrict__ fdop, int lo, int len,
                                             double s, double dfd, double x) {
    // one sample: numpy returns it for every x, NaN included (its one-point branch makes
    // no NaN check); longer rows map NaN to NaN
    if (len == 1) return (double)row[lo];
    if (x != x) return x;
    const double x0 = __ddiv_rn(fdop[lo], s), xl = __ddiv_rn(fdop[lo + len - 1], s);
    if (x < x0) return (double)row[lo];
    if (x > xl) return (double)row[lo + len - 1];
    // interval j with xp[j] <= x < xp[j+1]: guess from the uniform step, then settle
    // with exactly the comparisons a search over xp would make
    int j = (int)floor((x * s - fdop[lo]) / dfd);
    j = j < 0 ? 0 : (j > len - 1 ? len - 1 : j);
    while (j > 0 && __ddiv_rn(fdop[lo + j], s) > x) --j;
    while (j < len - 1 && __ddiv_rn(fdop[lo + j + 1], s) <= x) ++j;
    const double xj = __ddiv_rn(fdop[lo + j], s), yj = (double)row[lo + j];
    if (j == len - 1 || xj == x) return yj;
    const double xk = __ddiv_rn(fdop[lo + j + 1], s), yk = (double)row[lo + j + 1];
    const double slope = __ddiv_rn(__dsub_rn(yk, yj), __dsub_rn(xk, xj));
    double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xj)), yj);
    if (r != r) {                      // numpy's NaN fallbacks (compiled_base.c:arr_interp)
        r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xk)), yk);
        if (r != r && yj == yk) r = yj;
    }
    return r;
}

// one CTA per delay row
__global__ void __launch_bounds__(256)
norm_sspec_rows_kernel(const float* __restrict__ sspec, int nc, const double* __restrict__ fdop,
                       const double* __restrict__ tdel, double eta, double maxnormfac,
                       const double* __restrict__ fdopnew, int nq, float* __restrict__ out,
                       double* __restrict__ power) {
    __shared__ int s_lo, s_hi;
    __shared__ double s_sum[8];
    __shared__ int s_cnt[8];
    const int ii = blockIdx.x, tid = threadIdx.x;
    const float* row = sspec + (size_t)ii * nc;
    const double s = sqrt(__ddiv_rn(tdel[ii], eta));
    const double imax = __dmul_rn(maxnormfac, s);
    if (tid == 0) { s_lo = nc; s_hi = -1; }
    __syncthreads();
    int lo = nc, hi = -1;
    for (int k = tid; k < nc; k += blockDim.x)
        if (fabs(fdop[k]) <= imax) { lo = k < lo ? k : lo; hi = k > hi ? k : hi; }
    if (lo < nc) { atomicMin(&s_lo, lo); atomicMax(&s_hi, hi); }
    __syncthreads();
    lo = s_lo;
    hi = s_hi;
    const float qnan = __int_as_float(0x7fc00000);
    double psum = 0.0;
    int pcnt = 0;
    if (hi >= lo) {
        const int len = hi - lo + 1;
        const double dfd = nc > 1 ? fdop[1] - fdop[0] : 1.0;
        const double amax = fmax(fabs(__ddiv_rn(fdop[lo], s)), fabs(__ddiv_rn(fdop[hi], s)));
        for (int j = tid; j < nq; j += blockDim.x) {
            const double x = fdopnew[j];
            double r = interp_one(row, fdop, lo, len, s, dfd, x);
            const bool masked = (fabs(x) > amax) || (r != r);
            out[(size_t)ii * nq + j] = masked ? qnan : (float)r;
            // the reference's np.power(10, normSspec / 10) divides with numpy.ma's safe
            // division, which masks +-inf samples: their terms are left out of the mean
            if (!masked && isfinite(r)) { psum += pow(10.0, r / 10.0); ++pcnt; }
        }
    } else {
        for (int j = tid; j < nq; j += blockDim.x) out[(size_t)ii * nq + j] = qnan;
    }
    psum = warp_sum(psum);
    for (int o = 16; o > 0; o >>= 1) pcnt += __shfl_xor_sync(0xffffffffu, pcnt, o);
    if ((tid & 31) == 0) { s_sum[tid >> 5] = psum; s_cnt[tid >> 5] = pcnt; }
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        int c = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { t += s_sum[k]; c += s_cnt[k]; }
        power[ii] = c > 0 ? t / (double)c : __longlong_as_double(0x7ff8000000000000LL);
    }
}

// masked weighted average over the rows: one thread per column, coalesced over j
__global__ void norm_sspec_avg_kernel(const float* __restrict__ norm, int nr, int nq,
                                      const double* __restrict__ weights,
                                      double* __restrict__ avg) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nq) return;
    double num = 0.0, den = 0.0;
    for (int ii = 0; ii < nr; ++ii) {
        const float v = norm[(size_t)ii * nq + j];
        if (v == v) {
            const double w = weights[ii];
            num += w * (double)v;
            den += w;
        }
    }
    avg[j] = den != 0.0 ? num / den : __longlong_as_double(0x7ff8000000000000LL);
}

int norm_sspec_rows(const float* sspec, int nr, int nc, const double* fdop, const double* tdel,
                    double eta, double maxnormfac, const double* fdopnew, int nq, float* out,
                    double* power, cudaStream_t st) {
    norm_sspec_rows_kernel<<<nr, 256, 0, st>>>(sspec, nc, fdop, tdel, eta, maxnormfac, fdopnew,
                                               nq, out, power);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int norm_sspec_avg(const float* norm, int nr, int nq, const double* weights, double* avg,
                   cudaStream_t st) {
    norm_sspec_avg_kernel<<<(nq + 127) / 128, 128, 0, st>>>(norm, nr, nq, weights, avg);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

}  // namespace sb
