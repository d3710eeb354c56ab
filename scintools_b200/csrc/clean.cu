// Cleaning passes of Dynspec (include/scint_b200.h): the zero counts behind trim_edges
// (sb_dyn_zero_counts_f64) and the median-deviation zap (sb_zap_f64).  Everything is float64
// or integer, so both are exact.
//
// zero counts  one thread per column and 64 rows per block: the column count is the thread's
//              own sum, the row count a ballot per warp gathered in shared memory; one
//              integer atomic per column and per row of a block
// zap          two medians, each a radix select on order-preserving 64-bit keys (the key of a
//              pixel is that of x, or of |x - med| computed on the fly), then one pass that
//              writes NaN where |x - med| / mdev > sigma.  A select walks five digits
//              (15, 13, 12, 12, 12 bits) from the top.  The first histogram reads the whole
//              array; once the candidates of both middle ranks fit a buffer of n/8 keys they
//              are compacted into it and the remaining digits read only the buffer, so a
//              spread of values costs three full reads per median: one histogram, one more
//              histogram or the compaction, and the compaction or nothing.  Integer counts
//              make the result independent of the order of the atomics.
#include <math.h>

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int ZC_ROWS = 64;        // rows per block of the count kernel
constexpr int ZC_THREADS = 256;    // columns per block
constexpr int ZP_LEVELS = 5;
constexpr int ZP_BINS0 = 1 << 15;  // digit 0
constexpr int ZP_BINS = 1 << 13;   // digits 1..4, one histogram per middle rank
constexpr int ZP_THREADS = 1024;
constexpr int ZP_SCAN = 256;       // threads of the single-block digit scan

__device__ __forceinline__ int zp_shift(int L) { return L == 0 ? 49 : L == 1 ? 36 : 24 - 12 * (L - 2); }
__device__ __forceinline__ unsigned zp_dmask(int L) { return L == 0 ? 0x7fffu : L == 1 ? 0x1fffu : 0xfffu; }

// ---- zero counts ----------------------------------------------------------

__device__ __forceinline__ bool zc_zero(double v) { return v == 0.0 || v != v; }

// rows [row0, row1) of dyn [..][nt]; block (x, y): columns x*256.., rows row0 + y*64..
__global__ void __launch_bounds__(ZC_THREADS)
zero_counts_kernel(const double* __restrict__ dyn, int nt, int row0, int row1,
                   int* __restrict__ row_counts, int* __restrict__ col_counts) {
    SB_SHARED int s_row[ZC_ROWS];
    const int c = blockIdx.x * ZC_THREADS + threadIdx.x;
    const int rb = row0 + blockIdx.y * ZC_ROWS;
    const int re = min(rb + ZC_ROWS, row1);
    for (int i = threadIdx.x; i < ZC_ROWS; i += blockDim.x) s_row[i] = 0;
    __syncthreads();
    int cc = 0;
    for (int r = rb; r < re; ++r) {
        const bool z = c < nt && zc_zero(dyn[(long long)r * nt + c]);
        cc += z ? 1 : 0;
        const unsigned b = __ballot_sync(0xffffffffu, z);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(&s_row[r - rb], __popc(b));
    }
    __syncthreads();
    if (col_counts && c < nt && cc) atomicAdd(&col_counts[c], cc);
    if (row_counts)
        for (int i = threadIdx.x; i < re - rb; i += blockDim.x)
            if (s_row[i]) atomicAdd(&row_counts[rb - row0 + i], s_row[i]);
}

// ---- zap: radix select ------------------------------------------------------

// The select of one median.  Rank j (0: (m-1)/2, 1: m/2 of the m keys that are not NaN) is
// known down to the bits in mask[j]: prefix[j]; rank[j] is its rank among the keys with that
// prefix.  split: the two prefixes differ.  The buffer holds the keys of both prefixes once
// use_buf is set; compact_now asks the compaction after this digit to fill it.
struct ZapState {
    unsigned long long prefix[2], mask[2];
    long long rank[2];
    long long m, nbuf, cap;
    int split, use_buf, compact_now, empty;
};

struct ZapArgs {
    const double* x;
    long long n;
    const double* med;              // null: keys of x; else keys of |x - *med|
    const unsigned long long* buf;
    unsigned long long* wbuf;
    ZapState* s;
    unsigned long long* hist;       // [ZP_BINS0], or [2][ZP_BINS] after digit 0
};

// order-preserving key of v; false for NaN
__device__ __forceinline__ bool zp_key(double x, bool dev, double med, unsigned long long* k) {
    const double v = dev ? fabs(__dsub_rn(x, med)) : x;
    if (v != v) return false;
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    *k = (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
    return true;
}

__device__ __forceinline__ double zp_value(unsigned long long k) {
    const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffULL) : ~k;
    return __longlong_as_double((long long)u);
}

__global__ void zap_init_kernel(ZapArgs a, long long cap) {
    for (int i = threadIdx.x; i < ZP_BINS0; i += blockDim.x) a.hist[i] = 0;
    if (threadIdx.x == 0) {
        ZapState* s = a.s;
        for (int j = 0; j < 2; ++j) s->prefix[j] = s->mask[j] = 0, s->rank[j] = 0;
        s->m = s->nbuf = 0;
        s->cap = cap;
        s->split = s->use_buf = s->compact_now = s->empty = 0;
    }
}

// histogram of digit L over the keys that match a prefix
__global__ void __launch_bounds__(ZP_THREADS) zap_hist_kernel(ZapArgs a, int L) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned* h = reinterpret_cast<unsigned*>(smem_raw);
    const ZapState* s = a.s;
    if (s->empty) return;
    const int nb = L == 0 ? ZP_BINS0 : 2 * ZP_BINS;
    for (int i = threadIdx.x; i < nb; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const bool buf = s->use_buf || s->compact_now;
    const long long cnt = buf ? s->nbuf : a.n;
    const unsigned long long p0 = s->prefix[0], m0 = s->mask[0], p1 = s->prefix[1],
                             m1 = s->mask[1];
    const bool split = s->split != 0;
    const int sh = zp_shift(L);
    const unsigned dm = zp_dmask(L);
    const bool dev = a.med != nullptr;
    const double med = dev ? *a.med : 0.0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += stride) {
        unsigned long long k;
        if (buf) k = a.buf[i];
        else if (!zp_key(a.x[i], dev, med, &k)) continue;
        const unsigned d = (unsigned)(k >> sh) & dm;
        if ((k & m0) == p0) atomicAdd(&h[d], 1u);
        else if (split && (k & m1) == p1) atomicAdd(&h[ZP_BINS + d], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nb; i += blockDim.x)
        if (h[i]) atomicAdd(&a.hist[i], (unsigned long long)h[i]);
}

// one block of ZP_SCAN threads: the digit of each middle rank, then the state for the next
// digit; zeroes the histogram behind it
__global__ void __launch_bounds__(ZP_SCAN) zap_scan_kernel(ZapArgs a, int L) {
    SB_SHARED unsigned long long s_sum[2][ZP_SCAN];
    SB_SHARED unsigned long long s_cnt[2];
    SB_SHARED unsigned s_dig[2];
    SB_SHARED long long s_rank[2];
    ZapState* s = a.s;
    if (s->empty) return;
    const int t = threadIdx.x;
    const int nbin = L == 0 ? ZP_BINS0 : ZP_BINS;
    const int per = nbin / ZP_SCAN;
    const bool split = L > 0 && s->split;
    unsigned long long* h[2] = {a.hist, a.hist + (split ? ZP_BINS : 0)};
    for (int j = 0; j < 2; ++j) {
        unsigned long long v = 0;
        for (int i = 0; i < per; ++i) v += h[j][t * per + i];
        s_sum[j][t] = v;
    }
    __syncthreads();
    if (t < 2) {       // exclusive scans, serial: 256 adds
        unsigned long long run = 0;
        for (int i = 0; i < ZP_SCAN; ++i) {
            const unsigned long long v = s_sum[t][i];
            s_sum[t][i] = run;
            run += v;
        }
        if (t == 0 && L == 0) {
            s->m = (long long)run;
            s->rank[0] = ((long long)run - 1) / 2;
            s->rank[1] = (long long)run / 2;
            if (run == 0) s->empty = 1;
        }
    }
    __syncthreads();
    if (s->empty) return;
    for (int j = 0; j < 2; ++j) {
        const unsigned long long r = (unsigned long long)s->rank[j];
        const unsigned long long lo = s_sum[j][t];
        const unsigned long long hi = t + 1 < ZP_SCAN ? s_sum[j][t + 1] : ~0ULL;
        if (r >= lo && r < hi) {
            unsigned long long run = lo;
            for (int i = 0; i < per; ++i) {
                const unsigned long long v = h[j][t * per + i];
                if (r < run + v) {
                    s_dig[j] = (unsigned)(t * per + i);
                    s_rank[j] = (long long)(r - run);
                    s_cnt[j] = v;
                    break;
                }
                run += v;
            }
        }
    }
    __syncthreads();
    for (int j = 0; j < (split ? 2 : 1); ++j)
        for (int i = 0; i < per; ++i) h[j][t * per + i] = 0;
    if (t == 0) {
        const int sh = zp_shift(L);
        const unsigned long long dm = zp_dmask(L);
        for (int j = 0; j < 2; ++j) {
            s->prefix[j] |= (unsigned long long)s_dig[j] << sh;
            s->mask[j] |= dm << sh;
            s->rank[j] = s_rank[j];
        }
        s->split = s->prefix[0] != s->prefix[1];
        const unsigned long long c = s->split ? s_cnt[0] + s_cnt[1] : s_cnt[0];
        s->use_buf = s->use_buf || s->compact_now;
        s->compact_now = (!s->use_buf && L + 1 < ZP_LEVELS && (long long)c <= s->cap) ? 1 : 0;
    }
}

// copy the keys of both prefixes into the buffer, once
__global__ void zap_compact_kernel(ZapArgs a) {
    const ZapState* s = a.s;
    if (s->empty || !s->compact_now) return;
    const unsigned long long p0 = s->prefix[0], m0 = s->mask[0], p1 = s->prefix[1],
                             m1 = s->mask[1];
    const bool dev = a.med != nullptr;
    const double med = dev ? *a.med : 0.0;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // every lane of a warp runs the same trips: the loop tests the warp's first index
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i - lane < a.n;
         i += stride) {
        unsigned long long k = 0;
        const bool hit = i < a.n && zp_key(a.x[i], dev, med, &k) &&
                         ((k & m0) == p0 || (k & m1) == p1);
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (!b) continue;
        unsigned long long base = 0;
        if (lane == 0)
            base = atomicAdd((unsigned long long*)&a.s->nbuf, (unsigned long long)__popc(b));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (hit) a.wbuf[base + __popc(b & ((1u << lane) - 1u))] = k;
    }
}

// np.median: the middle key, or the mean of the two middle keys; NaN for no key
__global__ void zap_final_kernel(ZapArgs a, double* out) {
    const ZapState* s = a.s;
    if (s->empty) {
        *out = __longlong_as_double(0x7ff8000000000000LL);
        return;
    }
    const double lo = zp_value(s->prefix[0]);
    *out = (s->m & 1) ? lo : __ddiv_rn(__dadd_rn(lo, zp_value(s->prefix[1])), 2.0);
}

__global__ void zap_apply_kernel(double* __restrict__ x, long long n, double sigma,
                                 const double* __restrict__ stats) {
    const double med = stats[0], mdev = stats[1];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        if (__ddiv_rn(fabs(__dsub_rn(x[i], med)), mdev) > sigma)
            x[i] = __longlong_as_double(0x7ff8000000000000LL);
}

// candidate buffer of a select over n keys
inline long long zap_cap(long long n) {
    const long long c = n / 8;
    return c > 4096 ? c : (n < 4096 ? n : 4096);
}

#ifndef SB_HOST_EMU

int dyn_zero_counts(const double* dyn, int nf, int nt, int row0, int row1, int* row_counts,
                    int* col_counts, cudaStream_t st) {
    SB_ARG(dyn != nullptr && nf >= 1 && nt >= 1 && row0 >= 0 && row0 <= row1 && row1 <= nf);
    const long long yb = ((long long)(row1 - row0) + ZC_ROWS - 1) / ZC_ROWS;
    if (yb > 65535) {
        set_error("dyn_zero_counts: %d rows in one call (at most %d)", row1 - row0,
                  65535 * ZC_ROWS);
        return SB_ERR_UNSUPPORTED;
    }
    if (row_counts && row1 > row0)
        SB_CUDA(cudaMemsetAsync(row_counts, 0, (size_t)(row1 - row0) * sizeof(int), st));
    if (col_counts) SB_CUDA(cudaMemsetAsync(col_counts, 0, (size_t)nt * sizeof(int), st));
    if (row1 == row0 || (!row_counts && !col_counts)) return SB_OK;
    zero_counts_kernel<<<dim3((unsigned)((nt + ZC_THREADS - 1) / ZC_THREADS), (unsigned)yb),
                         ZC_THREADS, 0, st>>>(dyn, nt, row0, row1, row_counts, col_counts);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int zap(double* x, long long n, double sigma, double* stats, cudaStream_t st) {
    SB_ARG(x != nullptr && stats != nullptr && n >= 0);
    const long long cap = zap_cap(n);
    const size_t head = 256;
    static_assert(sizeof(ZapState) <= 256, "ZapState fits its slot head");
    unsigned char* idx = (unsigned char*)workspace(WS_INDEX, head + ZP_BINS0 * sizeof(unsigned long long));
    unsigned long long* buf =
        (unsigned long long*)workspace(WS_BATCH, (size_t)(cap > 0 ? cap : 1) * sizeof(unsigned long long));
    if (!idx || !buf) return SB_ERR_NOMEM;
    const int smem = ZP_BINS0 * (int)sizeof(unsigned);
    SB_CUDA(cudaFuncSetAttribute(zap_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int g = num_sms();
    const long long ab = (n + 255) / 256;
    const unsigned ga = (unsigned)(ab < 1 ? 1 : (ab < (long long)g * 16 ? ab : (long long)g * 16));
    ZapArgs a{x, n, nullptr, buf, buf, (ZapState*)idx, (unsigned long long*)(idx + head)};
    for (int pass = 0; pass < 2; ++pass) {
        a.med = pass ? stats : nullptr;
        zap_init_kernel<<<1, ZP_THREADS, 0, st>>>(a, cap);
        SB_LAUNCH_CHECK();
        for (int L = 0; L < ZP_LEVELS; ++L) {
            zap_hist_kernel<<<g, ZP_THREADS, L == 0 ? smem : smem / 2, st>>>(a, L);
            SB_LAUNCH_CHECK();
            zap_scan_kernel<<<1, ZP_SCAN, 0, st>>>(a, L);
            SB_LAUNCH_CHECK();
            if (L + 1 < ZP_LEVELS) {
                zap_compact_kernel<<<ga, 256, 0, st>>>(a);
                SB_LAUNCH_CHECK();
            }
        }
        zap_final_kernel<<<1, 1, 0, st>>>(a, stats + pass);
        SB_LAUNCH_CHECK();
    }
    if (n > 0) {
        zap_apply_kernel<<<ga, 256, 0, st>>>(x, n, sigma, stats);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
