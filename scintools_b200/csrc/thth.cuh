// theta-theta geometry shared by the gather / eigen kernels.
#pragma once
#include <limits.h>

#include "common.cuh"

namespace sb {

// Everything the per-point index math of thth_map needs
// (reference: scintools/ththmod.py:83-107).  Scalars are computed on the
// host with the reference's own numpy expressions so they are bit-identical.
struct ThthGeom {
    const float2* cs;      // conjugate spectrum, fftshifted rows
    long long ntau, nfd;   // logical size
    long long cs_pitch;    // elements per stored row
    int cs_valid_cols;     // half layout: stored columns that hold data (0 = all nfd/2+1)
    const float* cs_bound; // device: upper bound of max |CS| or null (the sweep scans)
    int cs_half;           // 0: full [ntau][nfd]; 1: Hermitian half [ntau][nfd/2+1]
                           //    holding the UNSHIFTED columns k = 0..nfd/2 (fd >= 0)
    double tau0, dtau, half_dtau, tau_absmax;  // tau[0], mean diff, /2, |tau.max()|
    double fd0, dfd, half_dfd, fd_half;        // fd[0], mean diff, /2, |fd.max()|/2
    double inv_dtau, inv_dfd;                  // reciprocals for the fast exact floor
    const double* th;      // theta bin centres (recentred), length n
    int n;
    int coherent;          // 1: complex CS, 0: |CS| (incoherent theta-theta)
};

struct ThthPoint {
    long long tq, fq;  // tau_inv, fd_inv (ththmod.py:94-97)
    bool pnt;          // pnts mask (ththmod.py:100)
    bool index_error;  // numpy would raise IndexError (fd_inv < -nfd)
};

// th1 = theta of the COLUMN, th2 = theta of the ROW (ththmod.py:86-87).
__device__ __forceinline__ ThthPoint thth_point(const ThthGeom& g, double eta,
                                                double th1, double th2) {
    ThthPoint p;
    double d = __dsub_rn(__dmul_rn(th1, th1), __dmul_rn(th2, th2));
    double a = __dadd_rn(__dsub_rn(__dmul_rn(eta, d), g.tau0), g.half_dtau);
    double b = __dadd_rn(__dsub_rn(__dsub_rn(th1, th2), g.fd0), g.half_dfd);
    double tqd = floor_div_fast(a, g.dtau, g.inv_dtau);
    double fqd = floor_div_fast(b, g.dfd, g.inv_dfd);
    // .astype(int): NaN / out-of-range -> INT64_MIN like numpy on x86
    p.tq = (tqd == tqd && fabs(tqd) < 9.0e18) ? (long long)tqd : LLONG_MIN;
    p.fq = (fqd == fqd && fabs(fqd) < 9.0e18) ? (long long)fqd : LLONG_MIN;
    p.pnt = (p.tq > 0) && (p.tq < g.ntau) && (p.fq < g.nfd);
    p.index_error = p.pnt && (p.fq < -g.nfd);
    return p;
}

// Stored CS columns a gather can address: every column of the full layout, the fd >= 0
// half (k = 0..nfd/2, all inside cs_pitch) of the half layout.
__device__ __forceinline__ int thth_ncols(const ThthGeom& g) {
    return (int)(g.cs_half ? g.nfd / 2 + 1 : g.nfd);
}

// Stored CS column of the pair (th1 = theta of the column, th2 = theta of the row): the fd
// bin of thth_point with python's wrap of a negative index, then, in the half layout, the
// stored column of that bin; *mirrored is set when the bin lies in the fd < 0 half
// (CS[-tau, -fd] = conj(CS[tau, fd]): the row is mirrored and the value conjugated).
// Returns -1 where the pnts mask / IndexError rule out the point for every curvature,
// otherwise a column in [0, thth_ncols(g)).  The curvature-sweep gather and the table of
// reached columns (thth_colmark_kernel) both call this, so they cannot disagree.
__device__ __forceinline__ int thth_pair_column(const ThthGeom& g, double th1, double th2,
                                                bool* mirrored) {
    *mirrored = false;
    const double bb = __dadd_rn(__dsub_rn(__dsub_rn(th1, th2), g.fd0), g.half_dfd);
    const double fqd = floor_div_fast(bb, g.dfd, g.inv_dfd);
    const long long fq = (fqd == fqd && fabs(fqd) < 9.0e18) ? (long long)fqd : LLONG_MIN;
    if (!(fq < g.nfd && !(fq < -g.nfd))) return -1;     // pnts mask / IndexError (thth_point)
    const long long fi = fq < 0 ? fq + g.nfd : fq;
    if (!g.cs_half) return (int)fi;
    const long long hfd = g.nfd / 2;
    if (fi >= hfd) return (int)(fi - hfd);
    if (fi == 0) return (int)hfd;
    *mirrored = true;
    return (int)(hfd - fi);
}

// Compact copy of the spectrum columns a theta grid reaches, delay axis contiguous:
// element (row r, stored column c) of the spectrum is base[slot_of_col[c] * tau_pitch + r];
// slot_of_col[c] < 0 marks a column the copy does not hold.  base == null: no copy was
// made, the sweep gathers from the spectrum itself (thth_gather_source, thth.cu).
struct ThthCopy {
    const float2* base;
    long long tau_pitch;
    int nslots;
    const int* slot_of_col;
    int* err;              // device word, set non-zero by a gather that meets slot < 0
};

// Gathered, Jacobian-weighted value before the Hermitian fill
// (ththmod.py:104,107).  Negative fd_inv wraps like python indexing.
__device__ __forceinline__ float2 thth_value(const ThthGeom& g, double eta,
                                             double th1, double th2,
                                             const ThthPoint& p) {
    float2 v = make_float2(0.f, 0.f);
    if (p.pnt && !p.index_error) {
        long long fi = p.fq < 0 ? p.fq + g.nfd : p.fq;
        if (!g.cs_half) {
            v = __ldg(g.cs + (size_t)p.tq * (size_t)g.cs_pitch + (size_t)fi);
        } else {
            // CS of a real dynamic spectrum: CS[-tau, -fd] = conj(CS[tau, fd])
            const long long h = g.nfd / 2;
            long long r = p.tq, c;
            bool cj = false;
            if (fi >= h) c = fi - h;
            else if (fi == 0) c = h;
            else { c = h - fi; r = (g.ntau - p.tq) % g.ntau; cj = true; }
            v = __ldg(g.cs + (size_t)r * (size_t)g.cs_pitch + (size_t)c);
            if (cj) v.y = -v.y;
        }
        if (!g.coherent) v = make_float2(hypotf(v.x, v.y), 0.f);
    }
    // Jacobian sqrt|2 eta (th2 - th1)| (ththmod.py:107); fp32 sqrt is ample
    float wf = sqrtf((float)fabs(2.0 * eta * (th2 - th1)));
    v.x *= wf;
    v.y *= wf;
    return v;
}

// np.nan_to_num on one float component (NaN -> 0, +-inf -> +-FLT_MAX).
__device__ __forceinline__ float nan_to_num(float x) {
    if (x != x) return 0.f;
    if (isinf(x)) return x > 0 ? 3.402823466e+38f : -3.402823466e+38f;
    return x;
}

// Element (i, j), i < j, of thth_map(hermetian=True) on the full grid (ththmod.py:108-114):
// the gathered value with nan_to_num, zero on the anti-diagonal i + j == n - 1.
__device__ __forceinline__ float2 thth_herm_upper(const ThthGeom& g, double eta, int i, int j) {
    if (i + j == g.n - 1) return make_float2(0.f, 0.f);
    const double thi = g.th[i], thj = g.th[j];
    float2 v = thth_value(g, eta, thj, thi, thth_point(g, eta, thj, thi));
    v.x = nan_to_num(v.x);
    v.y = nan_to_num(v.y);
    return v;
}

}  // namespace sb
