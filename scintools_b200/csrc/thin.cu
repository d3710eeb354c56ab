// "thin" theta-theta (arclet) curvature search: two-curvature rectangular map
// + largest singular value.  Reference: scintools/ththmod.py:1557-1636
// (two_curve_map), :496-512 (singularvalue_calc), :589-627 (eta loop of
// single_search_thin).  SURVEY.md section 8(f) rank 4.
//
//   rows  = theta2 bins (arclet grid, curvature eta2), cols = theta1 bins
//   tau_inv = floor((eta1 th1^2 - eta2 th2^2 - tau[1] + dtau/2) / dtau)
//   fd_inv  = floor((th1 - th2 - fd[1] + dfd/2) / dfd)
//   pnts    = 0 < tau_inv < ntau-1  and  fd_inv < nfd-1        (note tau[1], n-1)
//   value   = CS[tau_inv, fd_inv] * sqrt|2 eta1 th1 - 2 eta2 th2|
//   crop    = |th1| < sqrt(tau.max()/eta1), |th2| < sqrt(tau.max()/eta2)
//   columns with |th1| < centerCut are zeroed, result = sigma_max.
// sigma_max^2 is the largest eigenvalue of A^H A: the Lanczos machinery of the
// square sweep runs on the operator x -> A^H (A x); one pass over A per step
// (a warp holds a row in registers: row dot product, then the conjugate
// accumulation into per-lane column sums).
#include <float.h>
#include <limits.h>
#include <math.h>

#include "lanczos.cuh"
#include "thth.cuh"

namespace sb {

enum { TST_OK = 0, TST_INDEX_ERROR = 1, TST_ZERO_START = 2, TST_TOO_SMALL = 4,
       TST_NOT_CONVERGED = 8 };

struct ThinGeom {
    ThthGeom g;          // cs, ntau, nfd, dtau, dfd ...; tau0 := tau[1], fd0 := fd[1];
                         // g.th / g.n = theta1 centres (columns)
    const double* th2;   // theta2 centres (rows)
    int n2;
    double tau_max;      // tau.max() (not abs)
    double center_cut;
    int power;           // 0: CS as is, 1: |CS|^2 (incoherent thin, ththmod.py:609)
};

// crop masks + compaction for both axes, one warp per eta
__global__ void thin_prep_kernel(ThinGeom t, const double* __restrict__ eta1,
                                 const double* __restrict__ eta2, int neta, int ld1,
                                 int ld2, int* __restrict__ idx1, int* __restrict__ idx2,
                                 int* __restrict__ n1r, int* __restrict__ n2r) {
    const int e = blockIdx.x;
    if (e >= neta) return;
    const int lane = threadIdx.x;
    const double m1 = __dsqrt_rn(__ddiv_rn(t.tau_max, eta1[e]));
    const double m2 = __dsqrt_rn(__ddiv_rn(t.tau_max, eta2[e]));
    for (int axis = 0; axis < 2; ++axis) {
        const double* th = axis ? t.th2 : t.g.th;
        const int n = axis ? t.n2 : t.g.n;
        const double lim = axis ? m2 : m1;
        int* out = (axis ? idx2 + (size_t)e * ld2 : idx1 + (size_t)e * ld1);
        int base = 0;
        for (int k0 = 0; k0 < n; k0 += 32) {
            const int k = k0 + lane;
            const bool keep = k < n && fabs(th[k]) < lim;
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (keep) out[base + __popc(m & ((1u << lane) - 1u))] = k;
            base += __popc(m);
        }
        if (lane == 0) (axis ? n2r : n1r)[e] = base;
    }
}

struct ThinPoint { long long tq, fq; bool pnt, index_error; };

__device__ __forceinline__ ThinPoint thin_point(const ThinGeom& t, double e1, double e2,
                                                double th1, double th2) {
    const ThthGeom& g = t.g;
    ThinPoint p;
    const double d = __dsub_rn(__dmul_rn(e1, __dmul_rn(th1, th1)),
                               __dmul_rn(e2, __dmul_rn(th2, th2)));
    const double a = __dadd_rn(__dsub_rn(d, g.tau0), g.half_dtau);
    const double b = __dadd_rn(__dsub_rn(__dsub_rn(th1, th2), g.fd0), g.half_dfd);
    const double tqd = floor_div_fast(a, g.dtau, g.inv_dtau);
    const double fqd = floor_div_fast(b, g.dfd, g.inv_dfd);
    p.tq = (tqd == tqd && fabs(tqd) < 9.0e18) ? (long long)tqd : LLONG_MIN;
    p.fq = (fqd == fqd && fabs(fqd) < 9.0e18) ? (long long)fqd : LLONG_MIN;
    p.pnt = (p.tq > 0) && (p.tq < g.ntau - 1) && (p.fq < g.nfd - 1);
    p.index_error = p.pnt && (p.fq < -g.nfd);
    return p;
}

__device__ __forceinline__ float2 thin_value(const ThinGeom& t, double e1, double e2,
                                             double th1, double th2, const ThinPoint& p) {
    const ThthGeom& g = t.g;
    float2 v = make_float2(0.f, 0.f);
    if (p.pnt && !p.index_error) {
        const long long fi = p.fq < 0 ? p.fq + g.nfd : p.fq;
        if (!g.cs_half) {
            v = __ldg(g.cs + (size_t)p.tq * (size_t)g.cs_pitch + (size_t)fi);
        } else {
            const long long h = g.nfd / 2;
            long long r = p.tq, c;
            bool cj = false;
            if (fi >= h) c = fi - h;
            else if (fi == 0) c = h;
            else { c = h - fi; r = (g.ntau - p.tq) % g.ntau; cj = true; }
            v = __ldg(g.cs + (size_t)r * (size_t)g.cs_pitch + (size_t)c);
            if (cj) v.y = -v.y;
        }
        if (t.power) v = make_float2(v.x * v.x + v.y * v.y, 0.f);
    }
    const double w = __dsub_rn(__dmul_rn(__dmul_rn(2.0, e1), th1),
                               __dmul_rn(__dmul_rn(2.0, e2), th2));
    const float wf = sqrtf((float)fabs(w));
    v.x *= wf;
    v.y *= wf;
    return v;
}

// cropped rectangular map M[e] = [ld2][ld1]; grid (eta, row tiles, col tiles)
__global__ void __launch_bounds__(256)
thin_build_kernel(ThinGeom t, const double* __restrict__ eta1,
                  const double* __restrict__ eta2, int eta0, int ld1, int ld2,
                  const int* __restrict__ idx1, const int* __restrict__ idx2,
                  const int* __restrict__ n1r, const int* __restrict__ n2r,
                  float2* __restrict__ M, int* __restrict__ status) {
    const int e = blockIdx.x;
    const int n1 = n1r[eta0 + e], n2 = n2r[eta0 + e];
    const int ta = blockIdx.y, tb = blockIdx.z;       // row tile, column tile
    if (ta * 32 >= n2 || tb * 32 >= n1) return;
    const double e1 = eta1[eta0 + e], e2 = eta2[eta0 + e];
    const int* id1 = idx1 + (size_t)(eta0 + e) * ld1;
    const int* id2 = idx2 + (size_t)(eta0 + e) * ld2;
    float2* Me = M + (size_t)e * ld1 * ld2;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int b = tb * 32 + tx;
    const int j = b < n1 ? id1[b] : -1;
    const double th1 = j >= 0 ? t.g.th[j] : 0.0;
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int a = ta * 32 + ty + 8 * k;
        float2 v = make_float2(0.f, 0.f);
        if (a < n2 && j >= 0) {
            const double th2 = t.th2[id2[a]];
            const ThinPoint p = thin_point(t, e1, e2, th1, th2);
            bad |= p.index_error;
            if (!(fabs(th1) < t.center_cut)) v = thin_value(t, e1, e2, th1, th2, p);
        }
        if (a < ld2) Me[(size_t)a * ld1 + b] = v;
    }
    if (bad) atomicOr(status + eta0 + e, TST_INDEX_ERROR);
}

// the index error may also sit on a point that the crop removes: scan all
__global__ void thin_indexerr_kernel(ThinGeom t, const double* __restrict__ eta1,
                                     const double* __restrict__ eta2,
                                     int* __restrict__ status) {
    const int e = blockIdx.y;
    const long long total = (long long)t.g.n * t.n2;
    bool bad = false;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(p / t.g.n), j = (int)(p % t.g.n);
        bad |= thin_point(t, eta1[e], eta2[e], t.g.th[j], t.th2[i]).index_error;
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0)
        atomicOr(status + e, TST_INDEX_ERROR);
}

// ---- Lanczos on A^H A (bookkeeping in lanczos.cuh) ---------------------------
// one CTA per eta: sigma_max(A) with A = M[e] (n2 x n1, row pitch ld1)
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
thin_sv_kernel(const float2* __restrict__ Mbase, int ld1, int ld2,
               const int* __restrict__ n1r, const int* __restrict__ n2r, int eta0,
               double* __restrict__ svals, int* __restrict__ status,
               int* __restrict__ iters, double tol, double etol, int max_iter) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NW = THREADS / 32;
    LanczosShared& S = *reinterpret_cast<LanczosShared*>(smem_raw);
    float2* v = reinterpret_cast<float2*>(smem_raw + sizeof(LanczosShared));
    float2* vp = v + ld1;
    float2* w = vp + ld1;
    float2* part = w + ld1;        // [NW][512] per-warp column partials
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int e = blockIdx.x;
    const int n1 = n1r[eta0 + e], n2 = n2r[eta0 + e];
    const float2* M = Mbase + (size_t)e * ld1 * ld2;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    if ((status[eta0 + e] & TST_INDEX_ERROR) || n1 < 1 || n2 < 1) {
        if (tid == 0) {
            svals[eta0 + e] = qnan; iters[eta0 + e] = 0;
            if (n1 < 1 || n2 < 1) status[eta0 + e] |= TST_TOO_SMALL;
        }
        return;
    }
    // start vector: column sums of |A|^2 are positive where A has support;
    // v0 = conj of the row with the largest index that is non-zero, plus ones
    for (int c = tid; c < ld1; c += THREADS) {
        v[c] = c < n1 ? make_float2(1.f, 0.f) : make_float2(0.f, 0.f);
        vp[c] = make_float2(0.f, 0.f);
    }
    if (tid == 0) { S.done = 0; S.lo = 0.0; S.theta = 0.0; S.next_check = 1; S.m_last = 0; S.beta2[0] = 0.0; }
    __syncthreads();
    {
        const float s = rsqrtf((float)n1);
        for (int c = tid; c < n1; c += THREADS) v[c].x *= s;
    }
    __syncthreads();
    const int ncol4 = (n1 + 1) >> 1;
    const int nchunk = (n1 + 511) / 512;
    float beta_prev = 0.f;
    int m = 0;
    bool nonfinite = false;
    for (int it = 0; it < max_iter; ++it) {
        for (int c = tid; c < ld1; c += THREADS) w[c] = make_float2(0.f, 0.f);
        __syncthreads();
        // z = A^H (A v): per row, y = <row, v> over all chunks, then the conjugate
        // accumulation chunk by chunk
        for (int cb = 0; cb < nchunk; ++cb) {
            float4 zc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) zc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int a = warp; a < n2; a += NW) {
                const float4* row = reinterpret_cast<const float4*>(M + (size_t)a * ld1);
                float yx = 0.f, yy = 0.f;
                float4 mm[8];
                for (int c2 = 0; c2 < nchunk; ++c2) {       // full row dot product
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int c4 = c2 * 256 + lane + 32 * j;
                        const float4 q = c4 < ncol4 ? __ldg(row + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (c2 == cb) mm[j] = q;
                        const float4 x = (2 * c4 < ld1) ? *reinterpret_cast<const float4*>(v + 2 * c4)
                                                        : make_float4(0.f, 0.f, 0.f, 0.f);
                        yx = fmaf(q.x, x.x, yx); yx = fmaf(-q.y, x.y, yx);
                        yx = fmaf(q.z, x.z, yx); yx = fmaf(-q.w, x.w, yx);
                        yy = fmaf(q.x, x.y, yy); yy = fmaf(q.y, x.x, yy);
                        yy = fmaf(q.z, x.w, yy); yy = fmaf(q.w, x.z, yy);
                    }
                }
                yx = warp_sum(yx);
                yy = warp_sum(yy);
#pragma unroll
                for (int j = 0; j < 8; ++j) {      // conj(A[a][b]) * y_a
                    const float4 q = mm[j];
                    zc[j].x = fmaf(q.x, yx, zc[j].x); zc[j].x = fmaf(q.y, yy, zc[j].x);
                    zc[j].y = fmaf(q.x, yy, zc[j].y); zc[j].y = fmaf(-q.y, yx, zc[j].y);
                    zc[j].z = fmaf(q.z, yx, zc[j].z); zc[j].z = fmaf(q.w, yy, zc[j].z);
                    zc[j].w = fmaf(q.z, yy, zc[j].w); zc[j].w = fmaf(-q.w, yx, zc[j].w);
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j)
                *reinterpret_cast<float4*>(part + warp * 512 + 2 * (lane + 32 * j)) = zc[j];
            __syncthreads();
            for (int c = tid; c < 512; c += THREADS) {
                float sx = 0.f, sy = 0.f;
#pragma unroll
                for (int k = 0; k < NW; ++k) { sx += part[k * 512 + c].x; sy += part[k * 512 + c].y; }
                if (cb * 512 + c < ld1) w[cb * 512 + c] = make_float2(sx, sy);
            }
            __syncthreads();
        }
        double apart = 0.0;
        for (int c = tid; c < n1; c += THREADS)
            apart += (double)(v[c].x * w[c].x + v[c].y * w[c].y);
        apart = warp_sum(apart);
        if (lane == 0) S.red[0][warp] = apart;
        __syncthreads();
        double alpha = 0.0;
        for (int k = 0; k < NW; ++k) alpha += S.red[0][k];
        const float af = (float)alpha;
        double bpart = 0.0;
        for (int c = tid; c < n1; c += THREADS) {
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
        if (!isfinite(alpha) || !isfinite(beta)) { nonfinite = true; break; }
        if (warp == 0 && (m >= S.next_check || last || !(beta > 0.0))) lanczos_check(S, m, tol, etol);
        __syncthreads();
        if (S.done) break;
        const float ib = (float)(1.0 / beta);
        for (int c = tid; c < n1; c += THREADS) {
            const float2 x = w[c];
            vp[c] = v[c];
            v[c] = make_float2(x.x * ib, x.y * ib);
        }
        beta_prev = (float)beta;
        __syncthreads();
    }
    if (tid == 0) {
        // an all-zero map has sigma_max = 0 (numpy returns 0, no exception)
        const double th = S.theta > 0.0 ? S.theta : 0.0;
        svals[eta0 + e] = nonfinite ? qnan : sqrt(th);
        iters[eta0 + e] = m;
        if (!S.done && !nonfinite) status[eta0 + e] |= TST_NOT_CONVERGED;
    }
}

// full (uncropped) n2 x n1 map for the two_curve_map API / parity tests
__global__ void thin_map_kernel(ThinGeom t, double e1, double e2, float2* __restrict__ out,
                                int* __restrict__ err) {
    const long long total = (long long)t.g.n * t.n2;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(p / t.g.n), j = (int)(p % t.g.n);
        const ThinPoint pt = thin_point(t, e1, e2, t.g.th[j], t.th2[i]);
        if (pt.index_error) atomicOr(err, TST_INDEX_ERROR);
        out[p] = thin_value(t, e1, e2, t.g.th[j], t.th2[i], pt);
    }
}

#ifndef SB_HOST_EMU
int thin_map(const ThinGeom& t, double e1, double e2, float2* d_out, int* d_err,
             cudaStream_t st) {
    SB_CUDA(cudaMemsetAsync(d_err, 0, sizeof(int), st));
    const long long total = (long long)t.g.n * t.n2;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    thin_map_kernel<<<blocks, 256, 0, st>>>(t, e1, e2, d_out, d_err);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int thin_sweep(const ThinGeom& t, const double* d_eta1, const double* d_eta2, int neta,
               double tol, int max_iter, double* d_sv, int* d_status, int* d_n1, int* d_n2,
               int* d_iters, cudaStream_t st) {
    if (neta <= 0) return SB_OK;
    if (max_iter <= 0 || max_iter > SB_LANCZOS_MAXIT) max_iter = SB_LANCZOS_MAXIT;
    const int ld1 = (t.g.n + 31) / 32 * 32, ld2 = (t.n2 + 31) / 32 * 32;
    if (ld1 > 4096 || ld2 > 4096) {
        set_error("thin theta-theta grid %dx%d exceeds the supported 4096", t.n2, t.g.n);
        return SB_ERR_UNSUPPORTED;
    }
    int* d_idx = (int*)workspace(1, (size_t)neta * (ld1 + ld2) * sizeof(int));
    if (!d_idx) return SB_ERR_NOMEM;
    int* d_idx1 = d_idx;
    int* d_idx2 = d_idx + (size_t)neta * ld1;
    SB_CUDA(cudaMemsetAsync(d_status, 0, neta * sizeof(int), st));
    thin_prep_kernel<<<neta, 32, 0, st>>>(t, d_eta1, d_eta2, neta, ld1, ld2, d_idx1, d_idx2,
                                          d_n1, d_n2);
    SB_LAUNCH_CHECK();
    // one pair per gridDim.y row, which CUDA caps at 65535: launches of at most 65535
    for (int e0 = 0; e0 < neta; e0 += 65535) {
        const int nb = neta - e0 < 65535 ? neta - e0 : 65535;
        thin_indexerr_kernel<<<dim3(64, nb), 256, 0, st>>>(t, d_eta1 + e0, d_eta2 + e0,
                                                           d_status + e0);
        SB_LAUNCH_CHECK();
    }
    const size_t per = (size_t)ld1 * ld2 * sizeof(float2);
    const int batch = sweep_batch(per, neta, INT_MAX);
    float2* d_M = (float2*)workspace(2, per * batch);
    if (!d_M) return SB_ERR_NOMEM;
    constexpr int TH = 256;
    const size_t smem = sizeof(LanczosShared) + 3 * (size_t)ld1 * sizeof(float2) +
                        (size_t)(TH / 32) * 4096;
    SB_CUDA(cudaFuncSetAttribute(thin_sv_kernel<TH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
    for (int e0 = 0; e0 < neta; e0 += batch) {
        const int nb = neta - e0 < batch ? neta - e0 : batch;
        dim3 grid(nb, ld2 / 32, ld1 / 32), block(32, 8);
        thin_build_kernel<<<grid, block, 0, st>>>(t, d_eta1, d_eta2, e0, ld1, ld2, d_idx1, d_idx2,
                                                  d_n1, d_n2, d_M, d_status);
        SB_LAUNCH_CHECK();
        thin_sv_kernel<TH><<<nb, TH, smem, st>>>(d_M, ld1, ld2, d_n1, d_n2, e0, d_sv, d_status,
                                                 d_iters, tol, 2e-7, max_iter);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
