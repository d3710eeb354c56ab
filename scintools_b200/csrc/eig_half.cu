// Mixed-precision streaming Lanczos for the theta-theta eigenvalue
// (ththmod.Eval_calc, scintools/ththmod.py:371-401): the DEFAULT solver of
// sb::eta_sweep for ld <= 512.
//
// Why: the fp32 solver (thth_eig_kernel, thth.cu) re-reads the 1 MB fp32
// triangle on every Lanczos step (19.3 GB per 1024-eta sweep) and spends ~16 FFMA
// plus masks and shuffles per matrix element.  This kernel
//   * iterates on an fp16 copy of the triangle (4 B per complex element: half the
//     bytes) written by thth_build_kernel<2>, scaled per curvature by a power of two
//     so that the largest element stays below 2^15 (the scale cancels: only the
//     Ritz VECTOR of this phase is used).  A bf16 copy was measured first: its 8-bit
//     mantissa leaves a residual ||A y - rho y|| / rho of 0.6e-3 .. 3e-3 and
//     Rayleigh-quotient errors up to 1.1e-5 on the 4096x8192 workload -- fp16's
//     11 bits give 8x / 64x less;
//   * does the mat-vec on the tensor cores (mma.sync m16n8k16, fp16 x fp16 -> fp32,
//     see matvec_t), fetching the blocks with per-lane cp.async copies;
//   * runs the convergence check of step m on a ninth warp DURING mat-vec m+1, so
//     nobody idles behind the Sturm sweeps;
//   * keeps the Lanczos vectors (fp32) in global memory, forms the Ritz vector
//     y and reports the Rayleigh quotient <y, A y> / <y, y> with the FP32
//     triangle in one extra pass (second order in the vector error);
//   * safety net: the same fp32 pass yields the true residual
//     ||A y - rho y|| / |rho|; above rtol_r (1e-3) the solve continues as a plain
//     fp32 Lanczos started from y, the loop of thth_eig_kernel (thth_lanczos).
// Failure modes / status bits as thth_eig_kernel (NaN where the reference's
// try/except stores NaN).
#ifndef SB_HOST_EMU
#include <cuda_fp16.h>
#endif
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "../../include/scint_b200.h"   // SB_ETA_* status bits, tests/host_emu too
#include "drivers.cuh"
#include "lanczos.cuh"
#include "tma.cuh"

namespace sb {

constexpr int EB_THREADS = 256;
constexpr int EB_NW = EB_THREADS / 32;
constexpr int EB_NST = 2;             // fp32 pass: ring stages per warp, 4 KB each
#ifdef SB_EB_SLOTS
constexpr int EB_SLOTS = SB_EB_SLOTS; // tests/host_emu: few slots to exercise the fp32 restart
#else
constexpr int EB_SLOTS = 48;          // Lanczos vectors kept for the Ritz vector
#endif

// acc += a * (b, b): two fp32 FMAs, one per component
__device__ __forceinline__ void ffma2(float2& acc, const float2 a, const float b) {
    acc.x = fmaf(a.x, b, acc.x);
    acc.y = fmaf(a.y, b, acc.y);
}

// packed element of the fp16 triangle (thth.cu: pack_f16x2): re in the low, im in
// the high half
__device__ __forceinline__ float2 unpack_f16x2(const unsigned p) {
    __half2 h;
    *reinterpret_cast<unsigned*>(&h) = p;
    return __half22float2(h);
}

// two floats -> packed fp16 pair (first in the low half), round to nearest even
__device__ __forceinline__ unsigned pack_h2(const float lo, const float hi) {
#ifdef SB_HOST_EMU
    const __half2 h = __floats2half2_rn(lo, hi);
    return (unsigned)h.x | ((unsigned)h.y << 16);
#else
    unsigned r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
#endif
}

// ---- tensor-core mat-vec ---------------------------------------------------
// The fp16 copy is stored in 512-byte BLOCKS of 16 rows x 8 complex columns
// (thth_build_kernel<2>): block (I, G) = rows 16 I .., columns 8 G .., at byte
// ((I * ld / 8 + G) * 512); a block row is [re x 8 | im x 8] (planar, 32 bytes).
// One block is one m16n8k16 A operand (k < 8: re, k >= 8: im of column k - 8)
// and, read through ldmatrix.trans, the A operand of the transposed product.
constexpr int EB_TC_NST = 5;          // 1 KB stages (two adjacent blocks) per warp, + 4 KB column sums
// row blocks owned by each mat-vec warp (5-bit fields, count in bits 25+).  Row block I has
// 32 - I units (pairs of column groups 2 h, 2 h + 1, h >= I): {w, 15 - w, 16 + w, 31 - w} is
// (32 - w) + (17 + w) + (16 - w) + (1 + w) = 66 units for every warp, longest stream first.
#define EB_OWN5(a, b, c, d, e, cnt) \
    ((unsigned)(a) | (unsigned)(b) << 5 | (unsigned)(c) << 10 | (unsigned)(d) << 15 | \
     (unsigned)(e) << 20 | (unsigned)(cnt) << 25)
__device__ __forceinline__ unsigned eb_own_pack(const int warp) {
    if (warp >= EB_NW) return 0u;                  // the check warp owns nothing
    return EB_OWN5(warp, 15 - warp, 16 + warp, 31 - warp, 0, 4);
}

#ifdef SB_HOST_EMU
// warp-collective fragment loads / MMA through the emulator's lane exchange
inline void ldsm_x4(unsigned (&r)[4], smem_addr a) {
    unsigned long long all[32];
    emu::warp_gather((unsigned long long)(uintptr_t)a, all);
    const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; ++i)
        std::memcpy(&r[i], (const unsigned char*)(uintptr_t)all[8 * i + g] + 4 * t, 4);
}
inline void ldsm_x4_t(unsigned (&r)[4], smem_addr a) {
    unsigned long long all[32];
    emu::warp_gather((unsigned long long)(uintptr_t)a, all);
    const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; ++i) {
        unsigned short lo, hi;
        std::memcpy(&lo, (const unsigned char*)(uintptr_t)all[8 * i + 2 * t] + 2 * g, 2);
        std::memcpy(&hi, (const unsigned char*)(uintptr_t)all[8 * i + 2 * t + 1] + 2 * g, 2);
        r[i] = (unsigned)lo | ((unsigned)hi << 16);
    }
}
inline void mma16816(float (&d)[4], const unsigned (&a)[4], const unsigned b0, const unsigned b1) {
    unsigned long long A01[32], A23[32], Bq[32];
    emu::warp_gather((unsigned long long)a[0] | ((unsigned long long)a[1] << 32), A01);
    emu::warp_gather((unsigned long long)a[2] | ((unsigned long long)a[3] << 32), A23);
    emu::warp_gather((unsigned long long)b0 | ((unsigned long long)b1 << 32), Bq);
    const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
    auto half_of = [](unsigned w, int hi) { return emu_h2f((unsigned short)(hi ? w >> 16 : w & 0xffffu)); };
    auto Aat = [&](int row, int k) {            // fragment layout of mma.m16n8k16 (row-major A)
        const int ln = (row & 7) * 4 + ((k & 7) >> 1);
        const unsigned long long w = (k < 8) ? A01[ln] : A23[ln];
        return half_of((unsigned)(row < 8 ? w : w >> 32), k & 1);
    };
    auto Bat = [&](int k, int n) {
        const unsigned long long w = Bq[n * 4 + ((k & 7) >> 1)];
        return half_of((unsigned)(k < 8 ? w : w >> 32), k & 1);
    };
    for (int q = 0; q < 4; ++q) {
        const int row = g + 8 * (q >> 1), col = 2 * t + (q & 1);
        float acc = d[q];
        for (int k = 0; k < 16; ++k) acc += Aat(row, k) * Bat(k, col);
        d[q] = acc;
    }
}
#else
__device__ __forceinline__ void ldsm_x4(unsigned (&r)[4], const smem_addr a) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(unsigned (&r)[4], const smem_addr a) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
// d += A (16x16 fp16, row major) * B (16x8 fp16, column major), fp32 accumulate
__device__ __forceinline__ void mma16816(float (&d)[4], const unsigned (&a)[4], const unsigned b0,
                                         const unsigned b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
        "{%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
#endif

// shared-memory bytes of one CTA (host + device agree through this)
// bytes of a warp's slice of the ring: EB_TC_NST 1 KB stages + the 4 KB column-sum buffer
// (the fp32 pass re-uses the first 8 KB as two 4 KB row stages)
__host__ __device__ constexpr size_t eig_half_slice() {
    return (size_t)EB_TC_NST * 1024 + 4096;
}
__host__ __device__ inline size_t eig_half_smem(int ld) {
    return sizeof(LanczosShared) + 4 * (size_t)ld * sizeof(float2) +
           (size_t)EB_NW * eig_half_slice() + (size_t)EB_NW * EB_NST * 8 + 16 +
           4 * (size_t)(ld / 2) * 8;
}

// One more warp than the mat-vec needs (warp EB_NW): it only joins the barriers and runs
// the deferred convergence checks, so the eight mat-vec warps carry equal shares in every
// step (with the check on warp 0 that warp idled through half of every step without a
// check and was the straggler of the steps with one, holding the others at the barrier
// that ends the mat-vec).
__global__ void __launch_bounds__(EB_THREADS + 32, 2)
thth_eig_half_kernel(const float2* __restrict__ Mbase, const unsigned* __restrict__ Mbbase,
                     int ld, const int* __restrict__ nred, int eta0,
                     double* __restrict__ eigs, int* __restrict__ status,
                     int* __restrict__ iters, double tol, double etol, double etol_h, double rtol_r,
                     int max_iter, float2* __restrict__ gbasis) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    LanczosShared& S = *reinterpret_cast<LanczosShared*>(smem_raw);
    float2* v = reinterpret_cast<float2*>(smem_raw + sizeof(LanczosShared));
    float2* vp = v + ld;
    float2* w = vp + ld;          // row sums, then the new Lanczos vector
    float2* u = w + ld;           // column sums
    unsigned char* ring = reinterpret_cast<unsigned char*>(u + ld);     // [NW][WSL]
    float2* part = reinterpret_cast<float2*>(ring);                      // [NW][512] scratch (aliases the ring)
    constexpr int WSL = (int)eig_half_slice();                           // bytes per warp
    static_assert(WSL >= EB_NST * 4096, "the fp32 pass needs two 4 KB stages per warp");
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(ring + (size_t)EB_NW * WSL);
    // fp16 operand forms of the vector, [4 variants][ld / 2] x {b0, b1}
    uint2* P = reinterpret_cast<uint2*>(reinterpret_cast<unsigned char*>(mbar) +
                                        (size_t)EB_NW * EB_NST * 8 + 16);
    const int tid = threadIdx.x, lane = tid & 31;
    // warp index through a shuffle: tells the compiler it is warp-uniform, so the
    // bulk-copy addresses below live in uniform registers (no per-lane election loops)
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    constexpr int CHKW = EB_NW;                              // the warp that runs the deferred checks
    const bool worker = warp < EB_NW;
    const int tidw = worker ? tid : (1 << 24);               // strided loops: worker threads only
    const int e = blockIdx.x;
    const int n = nred[eta0 + e];
    const float2* M = Mbase + (size_t)e * ld * ld;
    const unsigned* Mb = Mbbase + (size_t)e * ld * ld;
    float2* basis = gbasis + (size_t)e * EB_SLOTS * ld;
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);

    if (status[eta0 + e] & SB_ETA_INDEX_ERROR) {
        if (tid == 0) { eigs[eta0 + e] = qnan; iters[eta0 + e] = 0; }
        return;
    }
    if (n < 3) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= SB_ETA_TOO_SMALL;
        }
        return;
    }
    // The ring starts out as zeros: positions a row's copy does not cover keep
    // older (finite) data, which only ever meets vector elements that are zero.
    for (int i = tidw; i < EB_NW * WSL / 16; i += EB_THREADS)
        reinterpret_cast<float4*>(ring)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid == 0) {
        for (int i = 0; i < EB_NW * EB_NST; ++i) mbar_init(mbar + i, 1);
        fence_mbarrier_init();
    }
    fence_proxy_async();
    __syncthreads();
    const int ncol4 = (n + 1) >> 1;            // fp32 rows: float4 groups = two complex columns
    unsigned char* mystage = ring + (size_t)warp * WSL;
    unsigned long long* mybar = mbar + EB_NST * warp;
    unsigned phbits = 0;                       // bit s: phase parity of this warp's barrier s

    // ------------------------------------------------------------------
    // fp16 mat-vec on the TENSOR CORES.  The triangle is a set of
    // 16-row x 8-column blocks (I, G), G >= 2 I; for every block
    //   rows:    D1[r][n] += sum_k A[r][k] B_G[k][n]     A = the block, k = (re | im) x column
    //   columns: D2[m][n]  = sum_r A[r][m] B_I[r][n]     A^T through ldmatrix.trans
    // with the vector in the n-columns of B as fp16 hi + 2^-11 lo pairs (n = 0 / 1: real /
    // imaginary part of the product from the hi halves, n = 2 / 3 from the lo halves;
    // 22 mantissa bits, the fp32 accumulators do the rest): 2 ldmatrix + 2 mma per 128
    // matrix elements instead of 64 FFMA + 16 converts.
    // A warp walks its row blocks one after the other and the blocks of a row block left to
    // right, two adjacent blocks (1 KB, contiguous in memory) per step -- one linear stream
    // per row block, so the producer cursor is an address increment.  (The first version
    // walked column-group major to keep the column sums in registers: its cursor search
    // dominated the instruction count and made it slower than the FMA mat-vec.)  The row
    // sums D1 of the current row block stay in registers; the column sums of every step are added to the warp's private
    // 4 KB column buffer (one lane per slot, LDS.128 / STS.128: no hazards).  Units arrive
    // through a ring of EB_TC_NST 1 KB stages per warp (two 16-byte cp.async chunks per lane,
    // XOR-swizzled so that both ldmatrix forms are conflict free).
    // ------------------------------------------------------------------
    auto matvec_t = [&](int check_m, double et) {
        const int ldh = ld >> 1;
        for (int c = tidw; c < ld; c += EB_THREADS) w[c] = make_float2(0.f, 0.f);
        // operand forms of the vector, [4 variants][ld / 2] x {b0, b1}; the entries of column
        // groups 2 h and 2 h + 1 are interleaved so that one LDS.128 fetches both: entry
        // (G, t) at (4 (G >> 1) + t) * 2 + (G & 1)
        for (int i = tidw; i < ldh; i += EB_THREADS) {
            const float4 x = *reinterpret_cast<const float4*>(v + 2 * i);   // two vector elements
            const unsigned xr = pack_h2(x.x, x.z), xi = pack_h2(x.y, x.w);
            const float2 hr = unpack_f16x2(xr), hi = unpack_f16x2(xi);
            const unsigned lr = pack_h2((x.x - hr.x) * 2048.f, (x.z - hr.y) * 2048.f);
            const unsigned li = pack_h2((x.y - hi.x) * 2048.f, (x.w - hi.y) * 2048.f);
            const int q = (((i >> 3) << 2) + (i & 3)) * 2 + ((i >> 2) & 1);
            P[q] = make_uint2(xr, xi ^ 0x80008000u);             // n = 0: re = Mr xr - Mi xi
            P[ldh + q] = make_uint2(xi, xr);                     // n = 1: im = Mr xi + Mi xr
            P[2 * ldh + q] = make_uint2(lr, li ^ 0x80008000u);   // n = 2 / 3: the same from the lo halves
            P[3 * ldh + q] = make_uint2(li, lr);
        }
        unsigned char* wring = ring + (size_t)warp * WSL;
        // column sums of this warp: float4 slot (h, g) = {re, im of column 16 h + g, re, im of
        // column 16 h + 8 + g} at index 8 h + g
        float4* mypart = reinterpret_cast<float4*>(wring + EB_TC_NST * 1024);
        if (worker) {
#pragma unroll
            for (int i = 0; i < 8; ++i) mypart[lane + 32 * i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
        const int g = lane >> 2, t = lane & 3;
        const int NI = (n + 14) >> 4;          // row blocks with stored elements (rows 0 .. n-2)
        const int NH = (n + 15) >> 4;          // pairs of column groups (a group past n reads the
                                               // zeros thth_build_kernel writes up to the tile edge)
        const int NGL = ld >> 3;               // groups per row block in memory
        const unsigned own = eb_own_pack(warp);
        const int cnt = (int)(own >> 25);
        const smem_addr sbase = smem_addr_of(wring);
        // lane's 16-byte chunk of a block: a linear copy (thth_build_kernel stores the two halves
        // of a block row swapped in rows 4-7 / 12-15, which is the XOR swizzle that makes both
        // ldmatrix forms below conflict free)
        smem_addr cdst = sbase + lane * 16;
        const unsigned char* gsrc = reinterpret_cast<const unsigned char*>(Mb) + lane * 16;
        const int mi = lane >> 3;
        const int arow = (lane & 7) + 8 * (mi & 1), trow = (lane & 7) + 8 * (mi >> 1);
        smem_addr aoff = sbase + arow * 32 + ((((mi >> 1) & 1) ^ ((arow >> 2) & 1)) << 4);
        smem_addr toff = sbase + trow * 32 + (((mi & 1) ^ ((trow >> 2) & 1)) << 4);
#ifndef SB_HOST_EMU
        // keep the per-lane bases in registers (the compiler re-derived them from the lane
        // index inside the loop: ~20 of the 80 instructions per step)
        asm volatile("" : "+r"(cdst), "+r"(aoff), "+r"(toff), "+l"(gsrc));
#endif
        constexpr unsigned RING_BYTES = EB_TC_NST * 1024;
        // producer cursor: row block pj of this warp, prem units (1 KB = blocks (I, 2 h),
        // (I, 2 h + 1)) left in it, next unit at byte pa of the fp16 copy, next stage at pst
        int pj = -1, prem = 0;
        unsigned pa = 0u, pst = 0u;
        unsigned cst = 0u;                   // consumer: byte offset of the stage read next
        bool pend = false;
        auto fetch_next = [&]() {
            if (prem == 0 && !pend) {
                for (;;) {
                    if (++pj >= cnt) { pend = true; break; }
                    const int I = (int)((own >> (5 * pj)) & 31u);
                    if (I < NI) {                 // (then I < NH: the diagonal unit exists)
                        prem = NH - I;
                        pa = (unsigned)(I * NGL + 2 * I) << 9;
                        break;
                    }
                }
            }
            if (!pend) {
                cp_async16_s(cdst + pst, gsrc + pa);
                cp_async16_s(cdst + pst + 512u, gsrc + pa + 512u);
                pa += 1024u;
                --prem;
            }
            pst += 1024u;
            if (pst == RING_BYTES) pst = 0u;
            cp_async_commit();                   // (an empty group keeps the wait count uniform)
        };
        for (int k = 0; k < EB_TC_NST - 1; ++k) fetch_next();
        if (check_m > 0 && warp == CHKW) lanczos_check(S, check_m, tol, et);
        const float lo_scale = 1.f / 2048.f;
        const bool bact = g < 4;                         // n >= 4: unused columns of B (zeros)
        // operand forms of this lane's n-column, pairs of groups: uint4 (h, t) at 4 h + t
        const uint4* Pg = reinterpret_cast<const uint4*>(P + (g & 3) * ldh) + t;
        for (int j = 0; j < cnt; ++j) {
            const int I = (int)((own >> (5 * j)) & 31u);
            if (I >= NI) continue;                       // warp-uniform
            const uint4* pb = Pg + 4 * I;                // groups 2 I, 2 I + 1
            unsigned tb0 = 0u, tb1 = 0u;                 // the vector at the rows of this block
            if (bact) { const uint4 e4 = *pb; tb0 = e4.x; tb1 = e4.z; }
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            float4* pc = mypart + 8 * I + g;
            for (int h = I; h < NH; ++h) {
                // operands that do not come through the ring first: their shared-memory latency
                // overlaps the wait (the asm statements below are barriers to the compiler)
                uint4 bq = make_uint4(0u, 0u, 0u, 0u);
                if (bact) bq = *pb;
                float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t == 0) q = *pc;
                cp_async_wait<EB_TC_NST - 2>();          // this lane's chunks of the unit
                __syncwarp();                            // ... and everybody else's
                unsigned a0[4], t0[4], a1[4], t1[4];
                ldsm_x4(a0, aoff + cst);
                ldsm_x4_t(t0, toff + cst);
                ldsm_x4(a1, aoff + cst + 512u);
                ldsm_x4_t(t1, toff + cst + 512u);
                fetch_next();        // into the stage the previous unit was read from (before the syncwarp)
                float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
                mma16816(acc, a0, bq.x, bq.y);
                mma16816(c0, t0, tb0, tb1);
                mma16816(acc, a1, bq.z, bq.w);
                mma16816(c1, t1, tb0, tb1);
                cst += 1024u;
                if (cst == RING_BYTES) cst = 0u;
                // column sums of the two blocks: conj(A) v = (Mr xr + Mi xi) + i (Mr xi - Mi xr)
                const float yr0 = c0[0] + c0[3], yi0 = c0[1] - c0[2];
                const float yr1 = c1[0] + c1[3], yi1 = c1[1] - c1[2];
                const float lr0 = __shfl_xor_sync(0xffffffffu, yr0, 1), li0 = __shfl_xor_sync(0xffffffffu, yi0, 1);
                const float lr1 = __shfl_xor_sync(0xffffffffu, yr1, 1), li1 = __shfl_xor_sync(0xffffffffu, yi1, 1);
                if (t == 0) {
                    q.x += fmaf(lr0, lo_scale, yr0);
                    q.y += fmaf(li0, lo_scale, yi0);
                    q.z += fmaf(lr1, lo_scale, yr1);
                    q.w += fmaf(li1, lo_scale, yi1);
                    *pc = q;
                }
                pb += 4;
                pc += 8;
            }
            // row sums of this row block
            const float l0 = __shfl_xor_sync(0xffffffffu, acc[0], 1);
            const float l1 = __shfl_xor_sync(0xffffffffu, acc[1], 1);
            const float l2 = __shfl_xor_sync(0xffffffffu, acc[2], 1);
            const float l3 = __shfl_xor_sync(0xffffffffu, acc[3], 1);
            if (t == 0) {
                w[16 * I + g] = make_float2(fmaf(l0, lo_scale, acc[0]), fmaf(l1, lo_scale, acc[1]));
                w[16 * I + g + 8] = make_float2(fmaf(l2, lo_scale, acc[2]), fmaf(l3, lo_scale, acc[3]));
            }
        }
        cp_async_wait<0>();                    // (only empty groups are left)
        __syncthreads();
        for (int c = tidw; c < ld; c += EB_THREADS) {
            float sx = 0.f, sy = 0.f;
            if (c < 16 * NH) {
                const int slot = (((c >> 4) << 3) + (c & 7)) * 2 + ((c >> 3) & 1);   // float2 index
#pragma unroll
                for (int kk = 0; kk < EB_NW; ++kk) {
                    const float2 q = reinterpret_cast<const float2*>(ring + (size_t)kk * WSL + EB_TC_NST * 1024)[slot];
                    sx += q.x;
                    sy += q.y;
                }
            }
            u[c] = make_float2(sx, sy);
        }
        __syncthreads();
    };

    // ------------------------------------------------------------------
    // fp32 mat-vec (final Rayleigh quotient, fp32 continuation): one 4 KB row
    // per stage, generic masks.  Stale fp16 words read as fp32 are only ever
    // multiplied into columns that are discarded; the ring is re-zeroed afterwards
    // because fp32 bit patterns read as fp16 could be inf / NaN.
    // ------------------------------------------------------------------
    auto matvec_f = [&]() {
        for (int c = tidw; c < ld; c += EB_THREADS) w[c] = make_float2(0.f, 0.f);
        __syncthreads();
        float4 yc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) yc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int K = (worker && n - 2 >= warp) ? (n - 2 - warp) / EB_NW + 1 : 0;
        auto issue = [&](int k) {
            const int a2 = warp + EB_NW * k;
            const int st = k % EB_NST;
            const int c_lo = (a2 + 1) & ~1;
            const unsigned bytes = (unsigned)(2 * ncol4 - c_lo) * 8u;
            mbar_expect_tx(mybar + st, bytes);
            bulk_g2s(mystage + st * 4096 + c_lo * 8, M + (size_t)a2 * ld + c_lo, bytes, mybar + st);
        };
        if (lane == 0)
            for (int k = 0; k < EB_NST && k < K; ++k) issue(k);
        for (int k = 0; k < K; ++k) {
            const int a = warp + EB_NW * k;
            const int first4 = (a + 1) >> 1;
            const float2 xa = v[a];
            const int st = k % EB_NST;
            while (!mbar_try_wait(mybar + st, (phbits >> st) & 1u)) {}
            phbits ^= 1u << st;
            const float4* sg = reinterpret_cast<const float4*>(mystage + st * 4096);
            float rx = 0.f, ry = 0.f;
            thth_row_fma([&](int, int c4) {
                return (c4 >= first4 && c4 < ncol4) ? sg[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
            }, v, ld, 0, first4 >> 5, xa, rx, ry, yc);
            __syncwarp();
            if (lane == 0 && k + EB_NST < K) issue(k + EB_NST);
            rx = warp_sum(rx);
            ry = warp_sum(ry);
            if (lane == 0) w[a] = make_float2(rx, ry);
        }
        __syncthreads();        // part aliases the stages of other warps
        thth_fold_columns<EB_NW>(yc, part, u, 0, ld);
        // fp32 rows may leave any bit pattern behind: the fp16 passes need zeros
        for (int i = tidw; i < EB_NW * WSL / 16; i += EB_THREADS)
            reinterpret_cast<float4*>(ring)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        fence_proxy_async();
        __syncthreads();
    };

    int m = 0;
    int mv = 0;                                 // mat-vecs done (reported as iters)
    // ------------------------------------------------------------------
    // fp16 Lanczos from the normalised vector in v (vp = 0), basis kept.  The
    // convergence check of the tridiagonal T_it runs on warp CHKW DURING mat-vec it
    // (one step late), so nobody idles behind its Sturm sweeps; when it reports
    // convergence the step just taken is surplus and m = it.  Returns false if
    // the basis slots ran out.  S.done / S.theta / m describe the outcome.
    // ------------------------------------------------------------------
    auto lanczos_b = [&](double et) -> bool {
        lanczos_reset(S);
        __syncthreads();
        float beta_prev = 0.f;
        m = 0;
        for (int it = 0; it < max_iter; ++it) {
            if (it >= EB_SLOTS) return false;
            for (int c = tidw; c < ld; c += EB_THREADS) basis[(size_t)it * ld + c] = v[c];
            const bool chk = it >= 1 && it >= S.next_check;
            matvec_t(chk ? it : 0, et);
            ++mv;
            double alpha, beta;
            lanczos_step<EB_NW>(S, it, n, v, vp, w, u, beta_prev, alpha, beta);
            if (chk && S.done) { m = it; break; }
            m = it + 1;
            if (it + 1 == max_iter || !(beta > 0.0)) {      // last word: check T_m now
                if (warp == CHKW) lanczos_check(S, m, tol, et);
                __syncthreads();
                break;
            }
            if (!isfinite(alpha)) break;
            lanczos_rotate<EB_NW>(v, vp, w, n, beta);
            beta_prev = (float)beta;
        }
        return true;
    };
    // plain fp32 Lanczos (restart / continuation): thth_eig_kernel's loop on matvec_f
    auto lanczos_f = [&](double et) {
        m = thth_lanczos<EB_NW>(S, matvec_f, v, vp, w, u, n, max_iter, tol, et);
        mv += m;
    };
    auto start_vector = [&]() { return thth_start_vector<EB_NW>(M, ld, n, v, vp, S.red[0]); };

    if (!start_vector()) {
        if (tid == 0) {
            eigs[eta0 + e] = qnan; iters[eta0 + e] = 0;
            status[eta0 + e] |= SB_ETA_ZERO_START;
        }
        return;
    }
    const bool fits = lanczos_b(etol_h);
    bool plain = !fits || !S.done;              // report the fp32 Ritz value instead
    if (!fits) {                                // more steps than basis slots: redo in fp32
        start_vector();
        lanczos_f(etol);
    } else if (S.done) {
        // ---- Ritz vector y = sum_j s_j q_j of T_m at theta, eigenvalue = Rayleigh
        // quotient with the fp32 triangle
        lanczos_ritz(S, m);
        for (int c = tidw; c < ld; c += EB_THREADS) {
            float sx = 0.f, sy = 0.f;
            if (c < n) {
                for (int j = 0; j < m; ++j) {
                    const float2 q = basis[(size_t)j * ld + c];
                    const float sj = (float)S.piv[j];
                    sx = fmaf(sj, q.x, sx);
                    sy = fmaf(sj, q.y, sy);
                }
            }
            v[c] = make_float2(sx, sy);
            vp[c] = make_float2(0.f, 0.f);
        }
        __syncthreads();
        matvec_f();
        double num = 0.0, den = 0.0;
        for (int c = tidw; c < n; c += EB_THREADS) {
            const float2 y = v[c];
            float2 ay = w[c];
            ay.x += u[c].x;
            ay.y += u[c].y;
            w[c] = ay;
            num += (double)y.x * ay.x + (double)y.y * ay.y;
            den += (double)y.x * y.x + (double)y.y * y.y;
        }
        num = warp_sum(num);
        den = warp_sum(den);
        if (lane == 0) { S.red[0][warp] = num; S.red[1][warp] = den; }
        __syncthreads();
        double sn = 0.0, sd = 0.0;
        for (int k = 0; k < EB_NW; ++k) { sn += S.red[0][k]; sd += S.red[1][k]; }
        const double rho = (sd > 0.0) ? sn / sd : 0.0;
        __syncthreads();
        double rpart = 0.0;
        for (int c = tidw; c < n; c += EB_THREADS) {
            const double rx = (double)w[c].x - rho * v[c].x, ry = (double)w[c].y - rho * v[c].y;
            rpart += rx * rx + ry * ry;
        }
        const double r2 = cta_sum<EB_NW>(rpart, S.red[0]);
        const bool accept = (sd > 0.0) && isfinite(rho) &&
                            (r2 <= rtol_r * rtol_r * rho * rho * sd);
        __syncthreads();
        if (accept) {
            if (tid == 0) { eigs[eta0 + e] = fabs(rho); iters[eta0 + e] = mv + 1; }
            return;
        }
        // fp32 continuation from y
        const float s = (sd > 0.0) ? (float)(1.0 / sqrt(sd)) : 0.f;
        for (int c = tidw; c < ld; c += EB_THREADS) { v[c].x *= s; v[c].y *= s; }
        __syncthreads();
        if (!(sd > 0.0)) start_vector();
        lanczos_f(etol);
        ++mv;                                  // the fp32 Rayleigh-quotient pass
        plain = true;
    } else {
        // iteration cap on the fp16 matrix: report what thth_eig_kernel would
    }
    if (plain && tid == 0) {
        eigs[eta0 + e] = fabs(S.theta);
        iters[eta0 + e] = mv;
        if (!S.done) status[eta0 + e] |= SB_ETA_NOT_CONVERGED;
    }
}

#ifndef SB_HOST_EMU
int eig_half_launch(const float2* d_M, const unsigned* d_Mb, int ld, const int* d_nred, int e0,
                    int nb, double* d_eigs, int* d_status, int* d_iters, double tol, double etol,
                    int max_iter, cudaStream_t st) {
    float2* d_basis = (float2*)workspace(WS_PLANE4, (size_t)nb * EB_SLOTS * ld * sizeof(float2));
    if (!d_basis) return SB_ERR_NOMEM;
    double rtol_r = 1e-3;
    if (const char* ev = getenv("SB_EIG_RTOL_R")) rtol_r = atof(ev);
    // stopping rule of the fp16 phase: res^2 <= etol_h * theta * gap.  Its Ritz vector only
    // feeds the fp32 Rayleigh quotient (second order in the vector error), so it can stop
    // earlier than the fp32 solver's 2e-7: 1e-6 saves one step per curvature on average with
    // the same worst-case error against dense eigenvalues (3e-6)
    double etol_h = 1e-6;
    if (const char* ev = getenv("SB_EIG_ETOL_B")) etol_h = atof(ev);
    const size_t smem = eig_half_smem(ld);
    SB_CUDA(cudaFuncSetAttribute(thth_eig_half_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
    thth_eig_half_kernel<<<nb, EB_THREADS + 32, smem, st>>>(d_M, d_Mb, ld, d_nred, e0, d_eigs,
                                                            d_status, d_iters, tol, etol, etol_h,
                                                            rtol_r, max_iter, d_basis);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
#endif  // SB_HOST_EMU

}  // namespace sb
