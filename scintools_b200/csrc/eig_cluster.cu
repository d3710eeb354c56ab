// Shared-memory-resident Lanczos for the theta-theta eigenvalue
// (ththmod.Eval_calc, scintools/ththmod.py:371-401; eta loops :789-799).
//
// The streaming solver in thth.cu re-reads the 1 MB strict upper triangle from
// HBM on every Lanczos step (~18 steps -> 19 GB per 1024-eta launch).  Here a
// thread-block CLUSTER of C CTAs keeps the triangle on chip for the whole
// solve: every CTA copies its share of the rows into shared memory ONCE
// (cp.async.bulk, one copy per row, packed back to back), and each Lanczos
// step is
//   1. every CTA: partial  y_r = (its rows of U) v + (its rows of U)^H v
//      (row sums by warp shuffle, column sums in per-lane registers, as in
//      thth.cu, v held in registers),
//   2. cluster barrier, every CTA reads the C partial vectors over DSMEM in
//      rank order (deterministic, bit-identical in all CTAs) -> full A v,
//   3. alpha / beta / vector update redundantly in every CTA (thread t owns
//      columns 2t, 2t+1 in registers), so no scalar has to be exchanged.
// Rows are dealt to the CTAs (and, inside a CTA, to the warps) in snake order
// so that the triangle is balanced to within one row.
//
// The serial tridiagonal bookkeeping (Sturm multisection + residual, a few
// thousand cycles per step) runs on a dedicated CHECKER warp concurrently with
// the next step's mat-vec; its verdict is consumed one step late (costs one
// extra mat-vec per eta, removes the bookkeeping from the critical path).
//
// HBM traffic: each matrix element is read exactly once.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "lanczos.cuh"
#include "tma.cuh"

namespace sb {

enum { EC_ST_INDEX_ERROR = 1, EC_ST_ZERO_START = 2, EC_ST_TOO_SMALL = 4,
       EC_ST_NOT_CONVERGED = 8 };

constexpr int EC_NW = 8;                 // mat-vec warps
constexpr int EC_MAIN = EC_NW * 32;      // 256 threads: thread t owns columns 2t, 2t+1
constexpr int EC_THREADS = EC_MAIN + 32; // + checker warp
constexpr int EC_COL4 = 256;             // float4 (column pairs) per vector: ld <= 512

struct alignas(16) EigClusterShared {
    LanczosShared L;
    double slot_theta[2];
    int slot_done[2];
    unsigned long long mbar;
    unsigned long long pad;
};

constexpr size_t EC_FIXED_BYTES = sizeof(EigClusterShared) +
                                  (size_t)EC_COL4 * 16 * (1 /*v*/ + 1 /*pr*/ + 2 /*out*/ + 4 /*scratch*/);

// ---- row dealing ------------------------------------------------------------
// CTA r of C owns rows a = 2C g + r and 2C g + 2C-1-r (g = 0, 1, ...), q-th
// owned row: g = q / 2.  Row a keeps the float4 columns [first4, ncol4),
// first4 = (a+1) >> 1, packed back to back in shared memory.
__host__ __device__ inline int ec_row_of(int q, int r, int C) {
    const int g = q >> 1;
    return 2 * C * g + ((q & 1) ? 2 * C - 1 - r : r);
}
__host__ __device__ inline int ec_off4(int q, int r, int C, int ncol4) {
    const int g = q >> 1;
    int o = g * (2 * ncol4 - C) - C * g * (g - 1);
    if (q & 1) o += ncol4 - C * g - ((r + 1) >> 1);
    return o;
}
// number of owned rows with a <= n - 2
__host__ __device__ inline int ec_nrows(int n, int r, int C) {
    const int R = n - 1;                 // rows 0 .. n-2
    const int G = R / (2 * C), rem = R - 2 * C * G;
    return 2 * G + (r < rem ? 1 : 0) + (2 * C - 1 - r < rem ? 1 : 0);
}

__device__ __forceinline__ unsigned ec_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned ec_nctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void ec_cluster_arrive() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void ec_cluster_wait() {
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void ec_bar_main() {
    asm volatile("bar.sync 1, %0;" ::"n"(EC_MAIN) : "memory");
}
__device__ __forceinline__ float4 ec_ld_peer(const float4* local, unsigned rank) {
    unsigned ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(local)), "r"(rank));
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ra));
    return v;
}

// SB_EIG_DEBUG=1: per-phase clock64 of cluster 0 / rank 0 (printed by the launcher)
__device__ long long ec_dbg[64][8];

template <bool DBG>
__global__ void __launch_bounds__(EC_THREADS, 1)
thth_eig_cluster_kernel(const float2* __restrict__ Mbase, int ld,
                        const int* __restrict__ nred, int eta0,
                        double* __restrict__ eigs, int* __restrict__ status,
                        int* __restrict__ iters, double tol, double etol, int max_iter,
                        int npair_max) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    EigClusterShared& S = *reinterpret_cast<EigClusterShared*>(smem_raw);
    LanczosShared& L = S.L;
    float4* v4 = reinterpret_cast<float4*>(smem_raw + sizeof(EigClusterShared));
    float4* pr4 = v4 + EC_COL4;              // row sums of the owned rows
    float4* out4 = pr4 + EC_COL4;            // [2][EC_COL4] partial A v, read by the peers
    float4* scratch = out4 + 2 * EC_COL4;    // [4][EC_COL4] column-sum tree
    int4* ptab = reinterpret_cast<int4*>(scratch + 4 * EC_COL4);   // per row pair: a1, base1, a2, base2
    float4* slice = reinterpret_cast<float4*>(ptab + npair_max);   // packed rows
    float2* v = reinterpret_cast<float2*>(v4);
    float2* pr = reinterpret_cast<float2*>(pr4);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool checker = warp == EC_NW;
    const int C = (int)ec_nctarank(), r = (int)ec_ctarank();
    const int e = blockIdx.x / C;
    const int n = nred[eta0 + e];
    const float2* M = Mbase + (size_t)e * ld * ld;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    const bool writer = (r == 0 && tid == 0);

    // failure modes of the reference's try/except (uniform over the cluster)
    if (status[eta0 + e] & EC_ST_INDEX_ERROR) {
        if (writer) { eigs[eta0 + e] = qnan; iters[eta0 + e] = 0; }
        return;
    }
    if (n < 3) {
        if (writer) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= EC_ST_TOO_SMALL;
        }
        return;
    }
    const int ncol4 = (n + 1) >> 1;
    const int nq = ec_nrows(n, r, C);
    if (tid == 0) {
        mbar_init(&S.mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        L.done = 0; L.lo = 0.0; L.theta = 0.0; L.res = 0.0; L.m_lo2 = 0; L.lo2 = 0.0;
        L.next_check = 1; L.beta2[0] = 0.0;
        S.slot_done[0] = S.slot_done[1] = 0;
        S.slot_theta[0] = S.slot_theta[1] = 0.0;
    }
    __syncthreads();
    // ---- fetch the owned rows: one bulk copy per row, one mbarrier for all
    if (tid == 0) mbar_expect_tx(&S.mbar, (unsigned)ec_off4(nq, r, C, ncol4) * 16u);
    __syncthreads();
    if (!checker) {
        for (int q = tid; q < nq; q += EC_MAIN) {
            const int a = ec_row_of(q, r, C);
            const int first4 = (a + 1) >> 1;
            bulk_g2s(slice + ec_off4(q, r, C, ncol4), M + (size_t)a * ld + 2 * first4,
                     (unsigned)(ncol4 - first4) * 16u, &S.mbar);
        }
    }
    // row-pair table: rows q = 2p, 2p+1 (a1 < a2, lengths within 2C-1 columns of
    // each other) are processed together; element c4 of row a sits at slice[base + c4]
    const int npair = (nq + 1) >> 1;
    for (int p = tid; p < npair; p += EC_THREADS) {
        const int a1 = ec_row_of(2 * p, r, C);
        int4 tb = make_int4(a1, ec_off4(2 * p, r, C, ncol4) - ((a1 + 1) >> 1), -1, 0);
        if (2 * p + 1 < nq) {
            const int a2 = ec_row_of(2 * p + 1, r, C);
            tb.z = a2;
            tb.w = ec_off4(2 * p + 1, r, C, ncol4) - ((a2 + 1) >> 1);
        }
        ptab[p] = tb;
    }
    // ---- v0 = row n//2 of the Hermitian matrix (ththmod.py:398-399), while
    // the copies are in flight.  Main thread t owns columns 2t, 2t+1.
    const int h = n / 2;
    float4 vcur = make_float4(0.f, 0.f, 0.f, 0.f), vprev = vcur;
    if (!checker) {
        float xs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int c = 2 * tid + k;
            float2 x = make_float2(0.f, 0.f);
            if (c < n && c > h) x = M[(size_t)h * ld + c];
            else if (c < h) { x = M[(size_t)c * ld + h]; x.y = -x.y; }
            xs[2 * k] = x.x; xs[2 * k + 1] = x.y;
        }
        vcur = make_float4(xs[0], xs[1], xs[2], xs[3]);
        pr4[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
        double p0 = (double)vcur.x * vcur.x + (double)vcur.y * vcur.y +
                    (double)vcur.z * vcur.z + (double)vcur.w * vcur.w;
        p0 = warp_sum(p0);
        if (lane == 0) L.red[0][warp] = p0;
    }
    __syncthreads();
    double nrm2 = 0.0;
    for (int k = 0; k < EC_NW; ++k) nrm2 += L.red[0][k];
    if (!(nrm2 > 0.0) || !isfinite(nrm2)) {
        // the bulk copies must land before the CTA's shared memory is released
        while (!mbar_try_wait(&S.mbar, 0)) {}
        if (writer) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= EC_ST_ZERO_START;
        }
        return;
    }
    float4 xv[8];
    if (!checker) {
        const float s = (float)(1.0 / sqrt(nrm2));
        vcur.x *= s; vcur.y *= s; vcur.z *= s; vcur.w *= s;
        v4[tid] = vcur;
        ec_bar_main();
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = v4[lane + 32 * j];
        while (!mbar_try_wait(&S.mbar, 0)) {}
    }

    const bool dbg = DBG && blockIdx.x == 0 && (tid == 0 || tid == EC_MAIN);
    long long c0 = 0, c1 = 0;
    if (DBG) c0 = clock64();
    float beta_prev = 0.f;
    int t = 0, m_final = 0;
    double theta_final = 0.0;
    bool converged = false;
    for (;; ++t) {
        const bool step = t < max_iter;
        if (!checker) {
            if (step) {
                const int par = t & 1;
                float4 yc[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) yc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                const bool tail = ncol4 < EC_COL4;
                int k = 0;
                int p = warp;    // snake over the warps: p = 2NW*(k/2) + (k odd ? 2NW-1-warp : warp)
                auto run_rows = [&](auto JSc) {
                    constexpr int JS = decltype(JSc)::value;
                    for (; p < npair; ) {
                        const int4 tb = ptab[p];
                        const int a1 = tb.x, a2 = tb.z;
                        if (((a1 + 1) >> 6) != JS) break;
                        const int f1 = (a1 + 1) >> 1;
                        const int f2 = a2 >= 0 ? (a2 + 1) >> 1 : 2 * EC_COL4;   // no 2nd row: all masked
                        const float2 xa1 = v[a1];
                        const float2 xa2 = a2 >= 0 ? v[a2] : make_float2(0.f, 0.f);
                        const float4* row1 = slice + tb.y;
                        const float4* row2 = slice + (a2 >= 0 ? tb.w : tb.y);   // no 2nd row: xa2 = 0
                        float r1xa = 0.f, r1xb = 0.f, r1ya = 0.f, r1yb = 0.f;
                        float r2xa = 0.f, r2xb = 0.f, r2ya = 0.f, r2yb = 0.f;
#pragma unroll
                        for (int j = JS; j < 8; ++j) {
                            const int c4 = lane + 32 * j;
                            // unconditional loads (the addresses left of the diagonal /
                            // right of the matrix are inside the CTA's shared memory);
                            // masks only where a boundary can fall: the diagonal of row 1
                            // in group JS, of row 2 (<= 2C-1 columns later) in JS, JS+1
                            float4 q1 = row1[c4], q2 = row2[c4];
                            if (j == JS || tail) {
                                bool ok1 = c4 >= f1;
                                if (tail) ok1 = ok1 && (c4 < ncol4);
                                q1.x = ok1 ? q1.x : 0.f; q1.y = ok1 ? q1.y : 0.f;
                                q1.z = ok1 ? q1.z : 0.f; q1.w = ok1 ? q1.w : 0.f;
                            }
                            if (j <= JS + 1 || tail) {
                                bool ok2 = c4 >= f2;
                                if (tail) ok2 = ok2 && (c4 < ncol4);
                                q2.x = ok2 ? q2.x : 0.f; q2.y = ok2 ? q2.y : 0.f;
                                q2.z = ok2 ? q2.z : 0.f; q2.w = ok2 ? q2.w : 0.f;
                            }
                            const float4 x = xv[j];
                            r1xa = fmaf(q1.x, x.x, r1xa); r1xb = fmaf(-q1.y, x.y, r1xb);
                            r1xa = fmaf(q1.z, x.z, r1xa); r1xb = fmaf(-q1.w, x.w, r1xb);
                            r1ya = fmaf(q1.x, x.y, r1ya); r1yb = fmaf(q1.y, x.x, r1yb);
                            r1ya = fmaf(q1.z, x.w, r1ya); r1yb = fmaf(q1.w, x.z, r1yb);
                            r2xa = fmaf(q2.x, x.x, r2xa); r2xb = fmaf(-q2.y, x.y, r2xb);
                            r2xa = fmaf(q2.z, x.z, r2xa); r2xb = fmaf(-q2.w, x.w, r2xb);
                            r2ya = fmaf(q2.x, x.y, r2ya); r2yb = fmaf(q2.y, x.x, r2yb);
                            r2ya = fmaf(q2.z, x.w, r2ya); r2yb = fmaf(q2.w, x.z, r2yb);
                            // conj(A) * v[a] for both rows
                            float4 y = yc[j];
                            y.x = fmaf(q1.x, xa1.x, y.x); y.x = fmaf(q1.y, xa1.y, y.x);
                            y.y = fmaf(q1.x, xa1.y, y.y); y.y = fmaf(-q1.y, xa1.x, y.y);
                            y.z = fmaf(q1.z, xa1.x, y.z); y.z = fmaf(q1.w, xa1.y, y.z);
                            y.w = fmaf(q1.z, xa1.y, y.w); y.w = fmaf(-q1.w, xa1.x, y.w);
                            y.x = fmaf(q2.x, xa2.x, y.x); y.x = fmaf(q2.y, xa2.y, y.x);
                            y.y = fmaf(q2.x, xa2.y, y.y); y.y = fmaf(-q2.y, xa2.x, y.y);
                            y.z = fmaf(q2.z, xa2.x, y.z); y.z = fmaf(q2.w, xa2.y, y.z);
                            y.w = fmaf(q2.z, xa2.y, y.w); y.w = fmaf(-q2.w, xa2.x, y.w);
                            yc[j] = y;
                        }
                        // four sums (re1, im1, re2, im2) in one 6-shuffle tree:
                        // lanes 0-15 end up with row 1, 16-31 with row 2; inside a
                        // half, lanes with bit 3 clear keep re, set keep im
                        const float r1x = r1xa + r1xb, r1y = r1ya + r1yb;
                        const float r2x = r2xa + r2xb, r2y = r2ya + r2yb;
                        const bool hi = lane & 16;
                        float kx = hi ? r2x : r1x, ky = hi ? r2y : r1y;
                        kx += __shfl_xor_sync(0xffffffffu, hi ? r1x : r2x, 16);
                        ky += __shfl_xor_sync(0xffffffffu, hi ? r1y : r2y, 16);
                        const bool b3 = lane & 8;
                        float keep = b3 ? ky : kx;
                        keep += __shfl_xor_sync(0xffffffffu, b3 ? kx : ky, 8);
                        keep += __shfl_xor_sync(0xffffffffu, keep, 4);
                        keep += __shfl_xor_sync(0xffffffffu, keep, 2);
                        keep += __shfl_xor_sync(0xffffffffu, keep, 1);
                        if (lane == 0) pr[a1].x = keep;
                        if (lane == 8) pr[a1].y = keep;
                        if (a2 >= 0) {
                            if (lane == 16) pr[a2].x = keep;
                            if (lane == 24) pr[a2].y = keep;
                        }
                        ++k;
                        p = 2 * EC_NW * (k >> 1) + ((k & 1) ? 2 * EC_NW - 1 - warp : warp);
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
                if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][0] = c1 - c0; c0 = c1; }
                // ---- column sums: 8 warps -> 4 -> 1
                if (warp >= 4) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) scratch[(warp - 4) * EC_COL4 + lane + 32 * j] = yc[j];
                }
                ec_bar_main();
                if (warp < 4) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        float4* p = scratch + warp * EC_COL4 + lane + 32 * j;
                        const float4 o = *p;
                        yc[j].x += o.x; yc[j].y += o.y; yc[j].z += o.z; yc[j].w += o.w;
                        *p = yc[j];
                    }
                }
                ec_bar_main();
                {
                    float4 s = pr4[tid];
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const float4 o = scratch[kk * EC_COL4 + tid];
                        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
                    }
                    out4[par * EC_COL4 + tid] = s;
                }
                if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][1] = c1 - c0; c0 = c1; }
                // ---- exchange: every CTA sums the C partials in rank order
                ec_cluster_arrive();
                ec_cluster_wait();
                if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][2] = c1 - c0; c0 = c1; }
                float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
                {
                    float4 o[8];
#pragma unroll
                    for (int rr = 0; rr < 8; ++rr)
                        if (rr < C) o[rr] = ec_ld_peer(out4 + par * EC_COL4 + tid, (unsigned)rr);
#pragma unroll
                    for (int rr = 0; rr < 8; ++rr)
                        if (rr < C) { w.x += o[rr].x; w.y += o[rr].y; w.z += o[rr].z; w.w += o[rr].w; }
                }
                if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][3] = c1 - c0 + (long long)(w.x == 12345.f); c0 = c1; }
                // ---- alpha = Re <v, A v>
                double apart = (double)(vcur.x * w.x + vcur.y * w.y) +
                               (double)(vcur.z * w.z + vcur.w * w.w);
                apart = warp_sum(apart);
                if (lane == 0) L.red[0][warp] = apart;
                ec_bar_main();
                double alpha = 0.0;
                for (int kk = 0; kk < EC_NW; ++kk) alpha += L.red[0][kk];
                // ---- w -= alpha v + beta_prev vp ; beta = ||w||
                const float af = (float)alpha;
                w.x -= af * vcur.x + beta_prev * vprev.x;
                w.y -= af * vcur.y + beta_prev * vprev.y;
                w.z -= af * vcur.z + beta_prev * vprev.z;
                w.w -= af * vcur.w + beta_prev * vprev.w;
                double bpart = (double)w.x * w.x + (double)w.y * w.y +
                               (double)w.z * w.z + (double)w.w * w.w;
                bpart = warp_sum(bpart);
                if (lane == 0) L.red[1][warp] = bpart;
                ec_bar_main();
                double b2 = 0.0;
                for (int kk = 0; kk < EC_NW; ++kk) b2 += L.red[1][kk];
                const double beta = sqrt(b2);
                if (tid == 0) { L.alpha[t] = alpha; L.beta[t + 1] = beta; L.beta2[t + 1] = b2; }
                // rotate (used only if the sweep goes on)
                const float ib = (float)(1.0 / beta);
                vprev = vcur;
                vcur = make_float4(w.x * ib, w.y * ib, w.z * ib, w.w * ib);
                beta_prev = (float)beta;
                if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][4] = c1 - c0; c0 = c1; }
            }
        } else {
            if (DBG) c0 = clock64();
            // ---- checker warp: verdict on T_m, m = t, while the others run step t
            if (step) ec_cluster_arrive();
            if (t >= 1) {
                const int m = t;
                int done = 0;
                if (m >= L.next_check || m == max_iter || !(L.beta[m] > 0.0)) {
                    lanczos_check_fast(L, m, tol, etol);
                    __syncwarp();
                    done = L.done;
                }
                __syncwarp();
                if (lane == 0) { S.slot_done[t & 1] = done; S.slot_theta[t & 1] = L.theta; }
            }
            if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][6] = c1 - c0; }
            if (step) ec_cluster_wait();
        }
        __syncthreads();   // sync A: alpha_t / beta_{t+1} and the verdict on m = t are published
        const bool done_t = (t >= 1) && S.slot_done[t & 1];
        const bool bad = step && !isfinite(L.alpha[t]);
        if (t >= 1) theta_final = S.slot_theta[t & 1];
        if (done_t) { converged = true; m_final = t; break; }
        if (bad) { m_final = t + 1; break; }
        if (!step) { m_final = max_iter; break; }
        if (!checker) {
            if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][5] = c1 - c0; c0 = c1; }
            v4[tid] = vcur;
            ec_bar_main();
#pragma unroll
            for (int j = 0; j < 8; ++j) xv[j] = v4[lane + 32 * j];
            if (DBG) { c1 = clock64(); if (dbg && t < 64) ec_dbg[t][7] = c1 - c0; c0 = c1; }
        }
    }
    // nobody leaves while a peer may still read its partial vectors
    ec_cluster_arrive();
    ec_cluster_wait();
    if (writer) {
        eigs[eta0 + e] = fabs(theta_final);  // np.abs(w[0])
        iters[eta0 + e] = m_final;
        if (!converged) status[eta0 + e] |= EC_ST_NOT_CONVERGED;
    }
}

// Smallest cluster size whose CTAs can hold their share of an n x n triangle
// (0: none up to 8, use the streaming solver).
static size_t cluster_smem(int n, int C, int* npair_max) {
    const int ncol4 = (n + 1) >> 1;
    size_t worst = 0;
    int nq_max = 0;
    for (int r = 0; r < C; ++r) {
        const int nq = ec_nrows(n, r, C);
        const size_t b = (size_t)ec_off4(nq, r, C, ncol4) * 16;
        worst = b > worst ? b : worst;
        nq_max = nq > nq_max ? nq : nq_max;
    }
    *npair_max = (nq_max + 1) / 2;
    // + slack: a cropped matrix (ncol4 < 256) is read, masked, up to column 255
    return EC_FIXED_BYTES + (size_t)*npair_max * sizeof(int4) + worst +
           (size_t)(EC_COL4 - ncol4) * 16;
}
static int pick_cluster(int n, size_t smem_max, size_t* smem_out, int* npair_max) {
    for (int C = 1; C <= 8; ++C) {
        const size_t b = cluster_smem(n, C, npair_max);
        if (b <= smem_max) {
            *smem_out = b;
            return C;
        }
    }
    return 0;
}

// Launch the on-chip solver for a batch of nb matrices; returns 1 when it ran,
// 0 when the problem does not qualify (caller falls back), < 0 on error.
int eig_cluster_launch(const float2* d_M, int ld, int n_max, const int* d_nred, int e0,
                       int nb, double* d_eigs, int* d_status, int* d_iters, double tol,
                       double etol, int max_iter, cudaStream_t st) {
    if (ld > 2 * EC_COL4 || n_max < 3) return 0;
    // SB_EIG_CLUSTER: unset / 0 = streaming solver (thth.cu), "auto" or 1 = smallest
    // cluster that holds the triangle, k = at least k CTAs per cluster
    int force = 0;
    if (const char* ev = getenv("SB_EIG_CLUSTER")) force = (ev[0] == 'a') ? 1 : atoi(ev);
    if (force <= 0) return 0;
    const size_t smem_max = 232448;   // 227 KB opt-in limit of sm_90
    size_t smem = 0;
    int npair_max = 0;
    int C = pick_cluster(n_max, smem_max, &smem, &npair_max);
    if (C == 0) return 0;
    if (force > C && force <= 8) {     // tests: exercise the DSMEM exchange on small grids
        C = force;
        smem = cluster_smem(n_max, C, &npair_max);
    }
    const bool debug = getenv("SB_EIG_DEBUG") != nullptr;
    auto kern = debug ? thth_eig_cluster_kernel<true> : thth_eig_cluster_kernel<false>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)nb * C);
    cfg.blockDim = dim3(EC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = C;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    SB_CUDA(cudaLaunchKernelEx(&cfg, kern, d_M, ld, d_nred, e0, d_eigs, d_status, d_iters,
                               tol, etol, max_iter, npair_max));
    if (debug) {
        int nclusters = -1;
        cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg);
        SB_CUDA(cudaStreamSynchronize(st));
        static long long h[64][8];
        SB_CUDA(cudaMemcpyFromSymbol(h, ec_dbg, sizeof(h)));
        fprintf(stderr, "[eig_cluster] n_max=%d C=%d smem=%zu nb=%d max_active_clusters=%d\n",
                n_max, C, smem, nb, nclusters);
        fprintf(stderr, "  trip: matvec tree cluster gather alphabeta syncA | check | rotate\n");
        for (int t = 0; t < 64 && h[t][0]; ++t)
            fprintf(stderr, "  %2d: %6lld %6lld %6lld %6lld %6lld %6lld | %6lld | %6lld\n", t, h[t][0],
                    h[t][1], h[t][2], h[t][3], h[t][4], h[t][5], h[t][6], h[t][7]);
    }
    return 1;
}

}  // namespace sb
