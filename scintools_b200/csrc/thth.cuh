// theta-theta geometry shared by the gather / eigen kernels, and the Lanczos pieces of the
// two solvers on its strict upper triangles (thth_eig_kernel, thth_eig_half_kernel).
#pragma once
#include <limits.h>

#include "common.cuh"
#include "lanczos.cuh"

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

// ---- Lanczos on a Hermitian matrix with zero diagonal stored as its strict upper triangle
// M [ld][ld] (thth_build_kernel), run by the first NW warps of the CTA --------------------

// Start vector of Eval_calc (ththmod.py:398-399): v = row n//2 of the Hermitian matrix,
// normalised, vp = 0.  False (v left unnormalised) when that row is zero or not finite.
// Starts with a barrier, so that a solve can restart from it, and ends with one.
template <int NW>
__device__ __forceinline__ bool thth_start_vector(const float2* M, int ld, int n, float2* v,
                                                  float2* vp, double* red) {
    __syncthreads();
    const int c0 = lanczos_first<NW>(), h = n / 2;
    double part0 = 0.0;
    for (int c = c0; c < ld; c += NW * 32) {
        float2 x = make_float2(0.f, 0.f);
        if (c < n && c > h) x = M[(size_t)h * ld + c];
        else if (c < h) { x = M[(size_t)c * ld + h]; x.y = -x.y; }
        v[c] = x;
        vp[c] = make_float2(0.f, 0.f);
        part0 += (double)x.x * x.x + (double)x.y * x.y;
    }
    const double nrm2 = cta_sum<NW>(part0, red);
    if (!(nrm2 > 0.0) || !isfinite(nrm2)) return false;
    const float s = (float)(1.0 / sqrt(nrm2));
    for (int c = c0; c < ld; c += NW * 32) { v[c].x *= s; v[c].y *= s; }
    __syncthreads();
    return true;
}

// Row a of the mat-vec over the column groups c4 = c4_0 + lane + 32 j, j = jskip .. 7 (a
// float4 holds columns 2 c4, 2 c4 + 1): q(j, c4) is the stored element pair, zero outside
// the row's part of the triangle.  Adds A[a][.] v to the row sums (rx, ry) and
// conj(A[a][.]) v[a] to the column partials yc[j], so that every stored element is read once
// per step (16 FFMA per pair).
template <class Row>
__device__ __forceinline__ void thth_row_fma(const Row& q, const float2* v, int ld, int c4_0,
                                             int jskip, float2 xa, float& rx, float& ry,
                                             float4 (&yc)[8]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j < jskip) continue;
        const int c4 = c4_0 + lane + 32 * j;
        const float4 p = q(j, c4);
        const float4 x = (2 * c4 < ld) ? *reinterpret_cast<const float4*>(v + 2 * c4)
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        // explicit FMA chains
        rx = fmaf(p.x, x.x, rx); rx = fmaf(-p.y, x.y, rx);
        rx = fmaf(p.z, x.z, rx); rx = fmaf(-p.w, x.w, rx);
        ry = fmaf(p.x, x.y, ry); ry = fmaf(p.y, x.x, ry);
        ry = fmaf(p.z, x.w, ry); ry = fmaf(p.w, x.z, ry);
        // conj(A) * v[a]
        yc[j].x = fmaf(p.x, xa.x, yc[j].x); yc[j].x = fmaf(p.y, xa.y, yc[j].x);
        yc[j].y = fmaf(p.x, xa.y, yc[j].y); yc[j].y = fmaf(-p.y, xa.x, yc[j].y);
        yc[j].z = fmaf(p.z, xa.x, yc[j].z); yc[j].z = fmaf(p.w, xa.y, yc[j].z);
        yc[j].w = fmaf(p.z, xa.y, yc[j].w); yc[j].w = fmaf(-p.w, xa.x, yc[j].w);
    }
}

// Column sums of a 512-column chunk from per-lane partials (thth_row_fma; thin.cu's A^H A
// pass): yc[j] of warp k holds columns 2 (lane + 32 j), +1 and goes through part [NW][512];
// out[col0 + c] = the sum over warps 0 .. NW-1, for c < 512 and col0 + c < ld.  A barrier
// before the sums and one after.
template <int NW>
__device__ __forceinline__ void thth_fold_columns(const float4 (&yc)[8], float2* part, float2* out,
                                                  int col0, int ld) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp < NW) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(part + warp * 512 + 2 * (lane + 32 * j)) = yc[j];
    }
    __syncthreads();
    for (int c = lanczos_first<NW>(); c < 512; c += NW * 32) {
        float sx = 0.f, sy = 0.f;
#pragma unroll
        for (int k = 0; k < NW; ++k) { sx += part[k * 512 + c].x; sy += part[k * 512 + c].y; }
        if (col0 + c < ld) out[col0 + c] = make_float2(sx, sy);
    }
    __syncthreads();
}

// Plain Lanczos, no re-orthogonalisation (only the top Ritz value is wanted), from the
// normalised vector in v with vp = 0.  matvec() leaves the row sums of A v in w and the
// column sums in u; warp 0 checks T_m whenever lanczos_check scheduled it.  Returns the
// steps taken; S.theta / S.done give the outcome.
template <int NW, class MatVec>
__device__ __forceinline__ int thth_lanczos(LanczosShared& S, const MatVec& matvec, float2* v,
                                            float2* vp, float2* w, const float2* u, int n,
                                            int max_iter, double tol, double etol) {
    lanczos_reset(S);
    __syncthreads();
    float beta_prev = 0.f;
    int m = 0;
    for (int it = 0; it < max_iter; ++it) {
        matvec();
        double alpha, beta;
        lanczos_step<NW>(S, it, n, v, vp, w, u, beta_prev, alpha, beta);
        m = it + 1;
        const bool last = (it + 1 == max_iter);
        if (threadIdx.x < 32 && (m >= S.next_check || last || !(beta > 0.0)))
            lanczos_check(S, m, tol, etol);
        __syncthreads();
        if (S.done || !isfinite(alpha)) break;
        lanczos_rotate<NW>(v, vp, w, n, beta);
        beta_prev = (float)beta;
    }
    return m;
}

#ifndef SB_HOST_EMU
// host drivers of thth.cu that the other sweeps and retrieval.cu share
int sweep_batch(size_t per_item, int count, int cap);
int thth_prep(const ThthGeom& g, const double* th_host, const double* d_etas, int neta, int ld,
              int* d_idx, int* d_nred, int* d_status, cudaStream_t st);
int thth_prep_table(const ThthGeom* geoms, const double* const* th_host, const ThthGeom* d_geoms,
                    const double* d_etas, int n, int ld, int* d_idx, int* d_nred, int* d_status,
                    cudaStream_t st);
int thth_gather_source(const ThthGeom& g, const double* th_host, int neta, ThthCopy* copy,
                       cudaStream_t st);
int thth_gather_check(const ThthCopy& copy, cudaStream_t st);
int thth_build_f32(const ThthGeom& g, const ThthCopy& copy, const double* d_etas, int e0, int nb,
                   int ld, const int* d_idx, const int* d_nred, float2* d_M, cudaStream_t st);
#endif

}  // namespace sb
