// Scintillation-scale fits behind Dynspec.get_scint_params (include/scint_b200.h,
// sb_scint_fit_1d and sb_scint_fit_2d).  Everything is float64.
//
// One batched Levenberg-Marquardt driver, templated on the model.  A fit has at most five
// parameters in fixed slots (tau, dnu, amp, alpha, phasegrad); `vary` and `bounded` are bit
// masks over the slots.  Varying bounded slots (min 0, max inf) are fitted in lmfit's
// internal variable, p = -1 + sqrt(x^2 + 1); varying unbounded ones directly, and fixed
// slots keep their value untransformed.  The models give the residual and
// its analytic derivative by every slot at one point; the ACF is read in place from a
// device stack through a row pitch.
//
// An iteration is two launches:
//   eval   one block per (fit, chunk) of a host-built table: the points
//          [first, first + SF_CHUNK) of the fit at its trial vector; partials of J^T J (upper
//          triangle over the varying slots), J^T r and r^T r into part[chunk][SF_NPART]
//   solve  one thread per fit: sums its chunks' partials in chunk order, then the Marquardt
//          step: accept the trial if r^T r fell, else raise lambda; test the stop rule; solve
//          (A + lambda diag(d)) dx = -g by Cholesky, d the running maximum of diag(A).
// Every sum runs in a fixed order inside a fixed chunk shape and nothing is atomic, so a
// fit's result is bit-identical alone, in any batch, in any order and on any repeat.  The
// host reads the number of finished fits every SF_CHECK iterations.
//
// A trial is accepted when r^T r falls, or when it stays within SF_LEVEL (float64 rounding
// of the sum) and the relative gradient falls.
// Stop rule: max_i |g_i| / sqrt(A_ii r^T r) <= SF_GTOL at an accepted point (stationary),
// or lambda > SF_LAMBDA_MAX after rejected trials (no decrease left at float64 precision),
// or r^T r == 0.  A fit that reaches max_nfev evaluations stops with SF_CAP and no errors; a
// non-finite r^T r at any evaluated point stops it with SF_NONFINITE.
//
// Standard errors as lmfit computes them: C = inv(A) at the result in the internal variables
// (NaN if A is not positive definite), C_ij g_i g_j redchi with g the transform's gradient,
// redchi = r^T r / max(1, ndata - nvarys).
#include <math.h>

#ifndef SB_HOST_EMU
#include <vector>
#endif

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int SF_NP = 5;                        // slots: tau dnu amp alpha phasegrad
constexpr int SF_NTRI = SF_NP * (SF_NP + 1) / 2;
constexpr int SF_NPART = SF_NTRI + SF_NP + 1;   // J^T J, J^T r, r^T r
constexpr int SF_NOUT = 2 * SF_NP + 1;         // params, stderr, chisqr
constexpr int SF_THREADS = 256;
constexpr int SF_CHUNK = 1024;                  // points per eval block
constexpr int SF_CHECK = 32;                    // iterations per host check
constexpr double SF_GTOL = 1e-10;
constexpr double SF_LAMBDA0 = 1e-3;
constexpr double SF_LAMBDA_MIN = 1e-15;
constexpr double SF_LAMBDA_MAX = 1e16;
constexpr double SF_LEVEL = 1e-14;             // r^T r changes below this are rounding
constexpr double SF_LN2 = 0.6931471805599453;  // np.log(2)

enum { SF_RUNNING = 0, SF_CONVERGED = 1, SF_STALLED = 2, SF_CAP = -1, SF_NONFINITE = -2 };

// one fit as the driver sees it (the public struct, include/scint_b200.h)
using FitDesc = sb_scint_fit;

struct FitState {
    double x[SF_NP];        // accepted point, internal variables (fixed slots: their value)
    double xt[SF_NP];       // trial point
    double A[SF_NTRI];      // J^T J at x, over the varying slots, upper triangle row-major
    double g[SF_NP];        // J^T r at x
    double d[SF_NP];        // Marquardt scaling
    double chi2, lam;
    int nfev, status;
};

__device__ __forceinline__ int sf_tri(int i, int j, int n) {   // i <= j < n
    return i * n - i * (i - 1) / 2 + (j - i);
}

__device__ __forceinline__ double sf_ext(double x, bool bounded) {
    return bounded ? -1.0 + sqrt(x * x + 1.0) : x;
}
__device__ __forceinline__ double sf_dext(double x, bool bounded) {
    return bounded ? x / sqrt(x * x + 1.0) : 1.0;
}

// 1-D: the time cut amp exp(-(x/tau)^alpha) and the frequency cut amp exp(-x ln2/dnu), each
// times the triangle 1 - x / max(x) of its cropped axis, weight of lag 0 zeroed
// (scint_models.py:62-120).  Points [0, n0) are the time cut, [n0, n0 + n1) the frequency cut.
struct Model1D {
    __host__ __device__ static long long npoints(const FitDesc& f) { return (long long)f.n0 + f.n1; }
    __device__ static double eval(const FitDesc& f, const double* p, long long k,
                                  double* dr) {
        const bool time = k < f.n0;
        const int i = time ? (int)k : (int)(k - f.n0);
        const int n = time ? f.n0 : f.n1;
        const double step = time ? f.s0 : f.s1;
        const double y = time ? f.acf[(long long)f.r0 * f.pitch + f.c0 + i]
                              : f.acf[(long long)(f.r1 + i) * f.pitch + f.c1];
        const double w = i == 0 ? 0.0 : f.aux[k];
        const double x = step * (double)i;
        const double tri = 1.0 - x / (step * (double)(n - 1));
        const double amp = p[2];
        for (int s = 0; s < SF_NP; ++s) dr[s] = 0.0;
        double m;
        if (time) {
            const double q = x / p[0];
            const double u = pow(q, p[3]);
            const double e = exp(-u);
            m = amp * e * tri;
            dr[2] = -w * e * tri;
            dr[0] = -w * m * p[3] * u / p[0];
            dr[3] = x > 0.0 ? w * m * u * log(q) : 0.0;
        } else {
            const double e = exp(-(x / (p[1] / SF_LN2)));
            m = amp * e * tri;
            dr[2] = -w * e * tri;
            dr[1] = -w * m * x * SF_LN2 / (p[1] * p[1]);
        }
        return (y - m) * w;
    }
};

// 2-D: scint_acf_model_2d_approx (scint_models.py:123-161) on the crop box [n0 rows of
// frequency lag][n1 columns of time lag].  The weight of point (i, j) is the reference's:
// 0 at (zf, zt) (the model's white-noise spike), 1e10 at (pf, pt), else the formula weight
// of point ((i + shf) mod n0, (j + sht) mod n1): the two fftshifts of an odd axis move the
// weights by one.  Formula: w = 1 / (1 / sqrt((c at_b) af_a)) (0 where that is not finite),
// or 1 unweighted, then 0 where y - 1 / w < 0, all at that point.
struct Model2D {
    __host__ __device__ static long long npoints(const FitDesc& f) { return (long long)f.n0 * f.n1; }
    __device__ static double weight(const FitDesc& f, int i, int j) {
        if (i == f.zf && j == f.zt) return 0.0;
        if (i == f.pf && j == f.pt) return 1e10;
        int a = i + f.shf, b = j + f.sht;
        if (a >= f.n0) a -= f.n0;
        if (b >= f.n1) b -= f.n1;
        double w = 1.0;
        if (f.weighted) {
            const double N = __dmul_rn(__dmul_rn(f.c, f.aux[f.n1 + f.n0 + b]),
                                       f.aux[2 * f.n1 + f.n0 + a]);
            double e = __ddiv_rn(1.0, __dsqrt_rn(N));
            if (!isfinite(e)) e = INFINITY;
            w = __ddiv_rn(1.0, e);
        }
        const double ya = f.acf[(long long)(f.r0 + a) * f.pitch + f.c0 + b];
        if (__dsub_rn(ya, __ddiv_rn(1.0, w)) < 0.0) w = 0.0;
        return w;
    }
    __device__ static double eval(const FitDesc& f, const double* p, long long k, double* dr) {
        const int i = (int)(k / f.n1), j = (int)(k - (long long)i * f.n1);
        const double t = f.aux[j], fr = f.aux[f.n1 + i];
        const double y = f.acf[(long long)(f.r0 + i) * f.pitch + f.c0 + j];
        const double w = weight(f, i, j);
        const double tau = p[0], dnu = p[1], amp = p[2], alpha = p[3];
        const double mu = p[4] * 60.0;
        const double a = (t - mu * fr) / tau;
        const double pw = 3.0 * alpha / 2.0;
        const double A = pow(fabs(a), pw);
        const double b = fabs(fr / (dnu / SF_LN2));
        const double B = pow(b, 1.5);
        const double S = A + B;
        const double Q = pow(S, 2.0 / 3.0);
        const double tri = (1.0 - fabs(t) / f.s0) * (1.0 - fabs(fr) / f.s1);
        const double e = exp(-Q);
        const double m = amp * e * tri;
        // dr/ds = -w dm/ds = w m dQ/dS dS/ds, dQ/dS = (2/3) Q / S; amp is linear
        const double h = S > 0.0 ? w * m * (2.0 / 3.0) * Q / S : 0.0;
        const double dAda = a != 0.0 ? pw * A / a : 0.0;
        dr[0] = h * (-pw * A / tau);
        dr[1] = h * (-1.5 * B / dnu);
        dr[2] = -w * e * tri;
        dr[3] = a != 0.0 ? h * 1.5 * A * log(fabs(a)) : 0.0;
        dr[4] = h * dAda * (-60.0 * fr / tau);
        return (y - m) * w;
    }
};

__device__ __forceinline__ void sf_params(const FitDesc& f, const double* x, double* p) {
    for (int s = 0; s < SF_NP; ++s) p[s] = sf_ext(x[s], ((f.bounded & f.vary) >> s) & 1);
}

// one block per row of `table`: (fit, first point) of a chunk of SF_CHUNK points
template <class M>
__global__ void __launch_bounds__(SF_THREADS)
sf_eval_kernel(const FitDesc* __restrict__ fits, const int2* __restrict__ table,
               const FitState* __restrict__ st, double* __restrict__ part) {
    SB_SHARED double red[SF_THREADS / 32][SF_NPART];
    const int2 tc = table[blockIdx.x];
    const FitState& S = st[tc.x];
    if (S.status != SF_RUNNING) return;
    const FitDesc f = fits[tc.x];
    double p[SF_NP], dp[SF_NP];
    sf_params(f, S.xt, p);
    int idx[SF_NP], nv = 0;
    for (int s = 0; s < SF_NP; ++s)
        if ((f.vary >> s) & 1) {
            dp[nv] = sf_dext(S.xt[s], ((f.bounded & f.vary) >> s) & 1);
            idx[nv++] = s;
        }
    double acc[SF_NPART];
    for (int q = 0; q < SF_NPART; ++q) acc[q] = 0.0;
    const long long n = M::npoints(f);
    const long long end = min((long long)tc.y + SF_CHUNK, n);
    for (long long k = tc.y + threadIdx.x; k < end; k += SF_THREADS) {
        double dr[SF_NP], J[SF_NP];
        const double r = M::eval(f, p, k, dr);
        for (int a = 0; a < nv; ++a) J[a] = dr[idx[a]] * dp[a];
        int e = 0;
        for (int a = 0; a < nv; ++a)
            for (int b = a; b < nv; ++b) acc[e++] += J[a] * J[b];
        for (int a = 0; a < nv; ++a) acc[SF_NTRI + a] += J[a] * r;
        acc[SF_NPART - 1] += r * r;
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int q = 0; q < SF_NPART; ++q) {
        const double v = warp_sum(acc[q]);
        if (lane == 0) red[w][q] = v;
    }
    __syncthreads();
    if (threadIdx.x < SF_NPART) {
        double s = 0.0;
        for (int i = 0; i < SF_THREADS / 32; ++i) s += red[i][threadIdx.x];
        part[(long long)blockIdx.x * SF_NPART + threadIdx.x] = s;
    }
}

// max_a |g_a| / sqrt(A_aa chi2): the relative gradient (MINPACK's gtol measure)
__device__ __forceinline__ double sf_cos(const double* A, const double* g, double chi2, int nv) {
    double cmax = 0.0;
    for (int a = 0; a < nv; ++a) {
        const double den = sqrt(A[sf_tri(a, a, nv)] * chi2);
        const double c = den > 0.0 ? fabs(g[a]) / den : (g[a] != 0.0 ? INFINITY : 0.0);
        cmax = fmax(cmax, c);
    }
    return cmax;
}

// Cholesky of the n x n upper-triangle matrix T (row-major packed) into L (full n x n);
// false if a pivot is not positive, not finite, or below rel of its diagonal
__device__ __forceinline__ bool sf_chol(const double* T, int n, double* L, double rel) {
    for (int i = 0; i < n; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = T[sf_tri(j, i, n)];
            for (int k = 0; k < j; ++k) s -= L[i * SF_NP + k] * L[j * SF_NP + k];
            if (i == j) {
                if (!(s > rel * T[sf_tri(i, i, n)]) || !isfinite(s)) return false;
                L[i * SF_NP + i] = sqrt(s);
            } else {
                L[i * SF_NP + j] = s / L[j * SF_NP + j];
            }
        }
    return true;
}

__device__ __forceinline__ void sf_chol_solve(const double* L, int n, double* v) {
    for (int i = 0; i < n; ++i) {
        double s = v[i];
        for (int k = 0; k < i; ++k) s -= L[i * SF_NP + k] * v[k];
        v[i] = s / L[i * SF_NP + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = v[i];
        for (int k = i + 1; k < n; ++k) s -= L[k * SF_NP + i] * v[k];
        v[i] = s / L[i * SF_NP + i];
    }
}

// results of a finished fit: params, stderr (NaN if not estimated), chisqr; info nfev, status
__device__ void sf_finish(const FitDesc& f, const FitState& S, int nv, const int* idx,
                          long long ndata, double* out, int* info) {
    sf_params(f, S.x, out);
    for (int s = 0; s < SF_NP; ++s) out[SF_NP + s] = NAN;
    out[2 * SF_NP] = S.chi2;
    info[0] = S.nfev;
    info[1] = S.status;
    if (S.status <= 0) return;
    double L[SF_NP * SF_NP];
    if (!sf_chol(S.A, nv, L, 1e-14)) return;
    const long long nfree = ndata - nv;
    const double redchi = S.chi2 / (double)(nfree > 1 ? nfree : 1);
    for (int a = 0; a < nv; ++a) {
        double e[SF_NP] = {0.0, 0.0, 0.0, 0.0, 0.0};
        e[a] = 1.0;
        sf_chol_solve(L, nv, e);        // column a of inv(A); e[a] = C_aa
        const int s = idx[a];
        const double g = sf_dext(S.x[s], ((f.bounded & f.vary) >> s) & 1);
        out[SF_NP + s] = sqrt(e[a] * g * g * redchi);
    }
}

template <class M>
__global__ void sf_solve_kernel(const FitDesc* __restrict__ fits, const int2* __restrict__ range,
                                int nfit, const double* __restrict__ part, FitState* __restrict__ st,
                                double* __restrict__ out, int* __restrict__ info) {
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= nfit) return;
    FitState S = st[fi];
    if (S.status != SF_RUNNING) return;
    const FitDesc f = fits[fi];
    int idx[SF_NP], nv = 0;
    for (int s = 0; s < SF_NP; ++s)
        if ((f.vary >> s) & 1) idx[nv++] = s;
    const int ntri = nv * (nv + 1) / 2;
    double P[SF_NPART];
    for (int q = 0; q < SF_NPART; ++q) P[q] = 0.0;
    const int2 rg = range[fi];      // first chunk, number of chunks
    for (int c = 0; c < rg.y; ++c) {
        const double* pc = part + (long long)(rg.x + c) * SF_NPART;
        for (int q = 0; q < SF_NPART; ++q) P[q] += pc[q];
    }
    ++S.nfev;
    const double rr = P[SF_NPART - 1];
    bool jfin = true;
    for (int q = 0; q < ntri; ++q) jfin = jfin && isfinite(P[q]);
    for (int a = 0; a < nv; ++a) jfin = jfin && isfinite(P[SF_NTRI + a]);
    // at the float64 floor of r^T r a step that does not raise it but lowers the gradient
    // is taken too, so the stop rule can still be met
    const bool level = jfin && rr <= S.chi2 * (1.0 + SF_LEVEL) &&
                       sf_cos(P, P + SF_NTRI, rr, nv) < sf_cos(S.A, S.g, S.chi2, nv);
    bool accepted = false;
    if (!isfinite(rr) || (S.nfev == 1 && !jfin)) {
        S.status = SF_NONFINITE;
    } else if (S.nfev == 1 || (rr < S.chi2 && jfin) || level) {
        for (int s = 0; s < SF_NP; ++s) S.x[s] = S.xt[s];
        for (int q = 0; q < ntri; ++q) S.A[q] = P[q];
        for (int a = 0; a < nv; ++a) S.g[a] = P[SF_NTRI + a];
        S.lam = S.nfev == 1 ? SF_LAMBDA0 : fmax(S.lam * 0.1, SF_LAMBDA_MIN);
        S.chi2 = rr;
        accepted = true;
    } else {
        S.lam *= 10.0;
    }
    if (S.status == SF_RUNNING && accepted) {
        if (sf_cos(S.A, S.g, S.chi2, nv) <= SF_GTOL || S.chi2 == 0.0 || nv == 0) S.status = SF_CONVERGED;
    }
    if (S.status == SF_RUNNING && S.lam > SF_LAMBDA_MAX) S.status = SF_STALLED;
    if (S.status == SF_RUNNING && S.nfev >= f.max_nfev) S.status = SF_CAP;
    if (S.status == SF_RUNNING) {
        // next trial: (A + lam diag(d)) dx = -g, raising lam until the factorisation holds
        for (int a = 0; a < nv; ++a) S.d[a] = fmax(S.d[a], S.A[sf_tri(a, a, nv)]);
        double L[SF_NP * SF_NP], v[SF_NP];
        for (;;) {
            double T[SF_NTRI];
            for (int q = 0; q < ntri; ++q) T[q] = S.A[q];
            for (int a = 0; a < nv; ++a) T[sf_tri(a, a, nv)] += S.lam * S.d[a];
            if (sf_chol(T, nv, L, 0.0)) break;
            S.lam *= 10.0;
            if (S.lam > SF_LAMBDA_MAX) {
                S.status = SF_STALLED;
                break;
            }
        }
        if (S.status == SF_RUNNING) {
            for (int a = 0; a < nv; ++a) v[a] = -S.g[a];
            sf_chol_solve(L, nv, v);
            for (int s = 0; s < SF_NP; ++s) S.xt[s] = S.x[s];
            for (int a = 0; a < nv; ++a) S.xt[idx[a]] = S.x[idx[a]] + v[a];
        }
    }
    if (S.status != SF_RUNNING)
        sf_finish(f, S, nv, idx, M::npoints(f), out + (long long)fi * SF_NOUT, info + 2 * fi);
    st[fi] = S;
}

// internal starting point, nfev 0
__global__ void sf_init_kernel(const FitDesc* __restrict__ fits, int nfit, FitState* __restrict__ st) {
    const int fi = blockIdx.x * blockDim.x + threadIdx.x;
    if (fi >= nfit) return;
    const FitDesc f = fits[fi];
    FitState S;
    for (int s = 0; s < SF_NP; ++s) {
        const double v = f.p0[s];
        // lmfit: _val = sqrt((val - min + 1)^2 - 1) for min 0, max inf
        S.x[s] = (((f.bounded & f.vary) >> s) & 1) ? sqrt((v + 1.0) * (v + 1.0) - 1.0) : v;
        S.xt[s] = S.x[s];
        S.g[s] = S.d[s] = 0.0;
    }
    for (int q = 0; q < SF_NTRI; ++q) S.A[q] = 0.0;
    S.chi2 = INFINITY;
    S.lam = SF_LAMBDA0;
    S.nfev = 0;
    S.status = SF_RUNNING;
    st[fi] = S;
}

// number of finished fits, summed in a fixed order by one block
__global__ void sf_count_kernel(const FitState* __restrict__ st, int nfit, int* __restrict__ done) {
    SB_SHARED double red[32];
    int c = 0;
    for (int i = threadIdx.x; i < nfit; i += blockDim.x) c += st[i].status != SF_RUNNING;
    double v = warp_sum((double)c);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
        *done = (int)s;
    }
}

#ifndef SB_HOST_EMU

template <class M>
static int scint_fit(const char* who, const FitDesc* fits_host, int nfit, double* out,
                     int* info, cudaStream_t st) {
    SB_ARG(fits_host && out && info && nfit >= 1);
    // the chunk table and each fit's chunk range
    std::vector<int2> table, range(nfit);
    int max_nfev = 0;
    for (int i = 0; i < nfit; ++i) {
        const FitDesc& f = fits_host[i];
        SB_ARG(f.acf && f.aux && f.pitch >= 1 && f.n0 >= 1 && f.n1 >= 1 && f.max_nfev >= 1);
        SB_ARG((f.vary & ~31) == 0 && (f.bounded & ~31) == 0);
        const long long n = M::npoints(f);
        if (n > (1ll << 31) - SF_CHUNK) {
            set_error("%s: fit %d has %lld points", who, i, n);
            return SB_ERR_UNSUPPORTED;
        }
        const int nc = (int)((n + SF_CHUNK - 1) / SF_CHUNK);
        if ((long long)table.size() + nc > (1ll << 31) - 1) {
            set_error("%s: more than 2^31 - 1 chunks", who);
            return SB_ERR_UNSUPPORTED;
        }
        range[i] = make_int2((int)table.size(), nc);
        for (int c = 0; c < nc; ++c) table.push_back(make_int2(i, c * SF_CHUNK));
        max_nfev = f.max_nfev > max_nfev ? f.max_nfev : max_nfev;
    }
    const size_t nch = table.size();
    const size_t bytes = nfit * (sizeof(FitDesc) + sizeof(int2) + sizeof(FitState)) +
                         nch * (sizeof(int2) + SF_NPART * sizeof(double)) + 6 * 16 + sizeof(int);
    char* w = (char*)workspace(WS_PLANE0, bytes);
    if (!w) return SB_ERR_NOMEM;
    auto take = [&](size_t b) { char* p = w; w += (b + 15) & ~size_t(15); return p; };
    FitDesc* d_fits = (FitDesc*)take(nfit * sizeof(FitDesc));
    int2* d_range = (int2*)take(nfit * sizeof(int2));
    int2* d_table = (int2*)take(nch * sizeof(int2));
    FitState* d_st = (FitState*)take(nfit * sizeof(FitState));
    double* d_part = (double*)take(nch * SF_NPART * sizeof(double));
    int* d_done = (int*)take(sizeof(int));
    SB_CUDA(cudaMemcpyAsync(d_fits, fits_host, nfit * sizeof(FitDesc), cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_range, range.data(), nfit * sizeof(int2), cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_table, table.data(), nch * sizeof(int2), cudaMemcpyHostToDevice, st));
    const unsigned gs = (unsigned)((nfit + 127) / 128);
    sf_init_kernel<<<gs, 128, 0, st>>>(d_fits, nfit, d_st);
    SB_LAUNCH_CHECK();
    int done = 0;
    for (int it = 0; it < max_nfev && done < nfit;) {
        const int stop = it + SF_CHECK < max_nfev ? it + SF_CHECK : max_nfev;
        for (; it < stop; ++it) {
            sf_eval_kernel<M><<<(unsigned)nch, SF_THREADS, 0, st>>>(d_fits, d_table, d_st, d_part);
            SB_LAUNCH_CHECK();
            sf_solve_kernel<M><<<gs, 128, 0, st>>>(d_fits, d_range, nfit, d_part, d_st, out, info);
            SB_LAUNCH_CHECK();
        }
        sf_count_kernel<<<1, 1024, 0, st>>>(d_st, nfit, d_done);
        SB_LAUNCH_CHECK();
        SB_CUDA(cudaMemcpyAsync(&done, d_done, sizeof(int), cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
    }
    return SB_OK;
}

int scint_fit_1d(const sb_scint_fit* fits, int nfit, double* out, int* info, cudaStream_t st) {
    return scint_fit<Model1D>("sb_scint_fit_1d", fits, nfit, out, info, st);
}

int scint_fit_2d(const sb_scint_fit* fits, int nfit, double* out, int* info, cudaStream_t st) {
    return scint_fit<Model2D>("sb_scint_fit_2d", fits, nfit, out, info, st);
}

#endif  // SB_HOST_EMU

}  // namespace sb
