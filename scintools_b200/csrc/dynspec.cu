// Dynspec hot path on the device: secondary spectrum (calc_sspec), ACF
// (calc_acf, method='direct') and the padded conjugate spectrum that feeds the
// theta-theta sweep.  All three are real 2-D FFTs done as
//   rows  : one CTA per live row, real->half-spectrum in shared memory
//   cols  : four-step split, two tile passes (A: stride-R2 rows + twiddle,
//           B: R2 consecutive rows) with the epilogue fused into pass B.
// Zero padding is never materialised: only live rows are transformed and the
// column pass A reads zeros for the padded rows.
//
// Reference: scintools/dynspec.py:3664-3721 (sspec), :3780-3797 (acf),
//            scintools/ththmod.py:777-787 + dynspec.py:1572-1579 (CS).
#include <map>
#include <stdlib.h>

#include "fft_kernels.cuh"

namespace sb {

// ---------------------------------------------------------------- twiddles
template <typename T>
__global__ void twiddle_fill_kernel(cx<T>* out, int N, int dir) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    double s, c;
    sincospi(2.0 * (double)i / (double)N, &s, &c);
    out[i] = mkc<T>((T)c, (T)(dir < 0 ? -s : s));
}

template <typename T> static std::map<long, void*>& tw_cache() {
    static std::map<long, void*> m;
    return m;
}

template <typename T>
const cx<T>* twiddle_table(int N, int dir, cudaStream_t st) {
    long key = (long)N * 2 + (dir > 0 ? 1 : 0);
    auto& m = tw_cache<T>();
    auto it = m.find(key);
    if (it != m.end()) return (const cx<T>*)it->second;
    void* p = nullptr;
    if (cudaMalloc(&p, (size_t)N * sizeof(cx<T>)) != cudaSuccess) {
        set_error("twiddle table N=%d: out of memory", N);
        cudaGetLastError();
        return nullptr;
    }
    twiddle_fill_kernel<T><<<(N + 255) / 256, 256, 0, st>>>((cx<T>*)p, N, dir);
    m[key] = p;
    return (const cx<T>*)p;
}
template const float2* twiddle_table<float>(int, int, cudaStream_t);
template const double2* twiddle_table<double>(int, int, cudaStream_t);

void twiddle_release() {
    for (auto& kv : tw_cache<float>()) cudaFree(kv.second);
    for (auto& kv : tw_cache<double>()) cudaFree(kv.second);
    tw_cache<float>().clear();
    tw_cache<double>().clear();
}

// ------------------------------------------------------------------- stats
// Sum over a 1-D CTA (result in thread 0).  One atomic per CTA instead of one per warp: the
// per-warp fp64 atomics of round 1 all hit one address and serialised in the L2
// (acf_mid_kernel issued 263 k of them at 4096x8192; dyn_stats_kernel likewise).
__device__ __forceinline__ double block_sum(double v, double* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double r = 0.0;
    if (w == 0) {
        r = l < (int)((blockDim.x + 31) >> 5) ? sh[l] : 0.0;
        r = warp_sum(r);
    }
    return r;
}
// out[0] = sum dyn, out[1] = sum wt*wf*dyn, out[2] = #finite, out[3] = sum finite
// Work item = (row, chunk of 256 x 8 columns); a thread keeps two 16-byte loads in
// flight per item and the items of a block are independent, so the pass streams
// (unlike a flat one-float-per-iteration loop with i % nt, i / nt).
template <bool VEC>
__global__ void __launch_bounds__(256)
dyn_stats_kernel(const float* __restrict__ dyn, long nf, long nt,
                 const float* __restrict__ wt, const float* __restrict__ wf,
                 double* __restrict__ out) {
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    const long nchunk = (nt + 2047) / 2048;
    const long items = nf * nchunk;
    for (long it = blockIdx.x; it < items; it += gridDim.x) {
        const long row = it / nchunk;
        const long t0 = (it - row * nchunk) * 2048;
        const float* src = dyn + row * nt;
        const float fw = wt ? wf[row] : 0.f;
        float v[8], wv[8];
        bool ok[8];
        if (VEC) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const long t = t0 + 4 * (threadIdx.x + 256 * h);
                const bool in = t < nt;                 // nt % 4 == 0: whole groups
                float4 q = make_float4(0.f, 0.f, 0.f, 0.f), ww = q;
                if (in) {
                    q = *reinterpret_cast<const float4*>(src + t);
                    if (wt) ww = *reinterpret_cast<const float4*>(wt + t);
                }
                v[4 * h] = q.x; v[4 * h + 1] = q.y; v[4 * h + 2] = q.z; v[4 * h + 3] = q.w;
                wv[4 * h] = ww.x; wv[4 * h + 1] = ww.y; wv[4 * h + 2] = ww.z; wv[4 * h + 3] = ww.w;
#pragma unroll
                for (int i = 0; i < 4; ++i) ok[4 * h + i] = in;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const long t = t0 + threadIdx.x + 256 * i;
                ok[i] = t < nt;
                v[i] = ok[i] ? src[t] : 0.f;
                wv[i] = (ok[i] && wt) ? wt[t] : 0.f;
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (!ok[i]) continue;
            s0 += v[i];
            if (wt) s1 += (double)(wv[i] * fw) * v[i];
            if (isfinite(v[i])) { s2 += 1.0; s3 += v[i]; }
        }
    }
    __shared__ double sh[32];
    s0 = block_sum(s0, sh); s1 = block_sum(s1, sh); s2 = block_sum(s2, sh); s3 = block_sum(s3, sh);
    if (threadIdx.x == 0) {
        atomicAdd(out + 0, s0); atomicAdd(out + 1, s1);
        atomicAdd(out + 2, s2); atomicAdd(out + 3, s3);
    }
}
// stats[4] = mu1 (mean), stats[5] = mu2 (mean after window), stats[6] = mean of finite
__global__ void dyn_stats_final_kernel(double* st, double n, double swt, double swf,
                                       int windowed) {
    double mu1 = st[0] / n;
    st[4] = mu1;
    st[5] = windowed ? (st[1] - mu1 * swt * swf) / n : 0.0;
    st[6] = st[3] / st[2];
    st[7] = 0.0;  // accumulator for the ACF power sum
}

// --------------------------------------------------------- row load functors
struct DynRowLoad {
    const float* dyn;
    int nf, nt;            // live size of the source
    const float* wt;       // time taper [nt] or null
    const float* wf;       // frequency taper [nf] or null
    const double* stats;   // device: [4]=mu1 [5]=mu2 [6]=mean(finite)
    int mode;              // 0: sspec (x = wt wf (d-mu1) - mu2), 1: acf (d - mean finite),
                           // 2: raw minus constant `sub`
    int prewhite;
    float sub;
    int vec = 0;                   // init(): rows can be read with 8-byte loads
    float m1c = 0.f, m2c = 0.f;    // the constants of `mode`, read once per thread by init()
    // (they were re-read from `stats` and narrowed for every element: 6 % of the row pass)
    __device__ __forceinline__ void init() {
        vec = !prewhite && !wt && !(nt & 1) && (reinterpret_cast<uintptr_t>(dyn) & 7) == 0;
        m2c = 0.f;
        if (mode == 0) { m1c = (float)stats[4]; m2c = (float)stats[5]; }
        else if (mode == 1) { m1c = (float)stats[6]; }
        else if (mode == 3) { m1c = (float)stats[4]; }     // minus the device-side mean
        else { m1c = sub; }
    }
    // entries n >= live() of a row are zero padding
    __device__ __forceinline__ int live(int N) const {
        const int l = (nt + 1) >> 1;
        return l < N ? l : N;
    }
    __device__ __forceinline__ float val(int f, int t, float m1, float m2) const {
        float v = dyn[(size_t)f * nt + t] - m1;
        if (wt) v *= wt[t] * wf[f];
        return v - m2;
    }
    __device__ __forceinline__ float get(int f, int t, float m1, float m2) const {
        if (!prewhite) return (t < nt) ? val(f, t, m1, m2) : 0.f;
        if (t >= nt - 1) return 0.f;
        return val(f + 1, t + 1, m1, m2) - val(f + 1, t, m1, m2) -
               val(f, t + 1, m1, m2) + val(f, t, m1, m2);
    }
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        const float m1 = m1c, m2 = m2c;
        const int f = (int)row, t = 2 * n;
        if (vec && t < nt) {                                // one 8-byte load
            const float2 d = *reinterpret_cast<const float2*>(dyn + (size_t)f * nt + t);
            return make_float2(d.x - m1 - m2, d.y - m1 - m2);
        }
        return make_float2(get(f, t, m1, m2), get(f, t + 1, m1, m2));
    }
};
__device__ __forceinline__ void row_load_init(DynRowLoad& l) { l.init(); }
__device__ __forceinline__ int row_load_live(const DynRowLoad& l, int N) { return l.live(N); }

struct HalfStore {   // X[k] -> H[row][k], only the first kmax bins are kept
    float2* H;
    long pitch;
    int kmax;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        if (k < kmax) H[row * pitch + k] = v;
    }
};

// conjugate spectrum epilogue: fftshift both axes, Hermitian expansion to the
// full plane, tau row mask, DC correction for a non-zero pad constant
struct CsStore {
    float2* CS;
    int NF, NT, R1;
    const unsigned char* rowmask;   // [NF] in fftshifted row order, or null
    float dc;
    int half;       // 1: write only the fd >= 0 half, [NF][pitch], column = c
    long pitch;
    const double* dc_stats;   // non-null: dc = stats[4] * NF * NT (device-side mean)
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kf = y + R1 * k;
        if (kf == 0 && c == 0)
            v.x += dc_stats ? (float)(dc_stats[4] * (double)NF * (double)NT) : dc;
        const int rs = (kf + NF / 2) & (NF - 1);
        if (half) {
            const bool mh = rowmask && rowmask[rs];
            CS[(size_t)rs * pitch + c] = mh ? make_float2(0.f, 0.f) : v;
            return;
        }
        const int cs = (c + NT / 2) & (NT - 1);
        const bool m0 = rowmask && rowmask[rs];
        CS[(size_t)rs * NT + cs] = m0 ? make_float2(0.f, 0.f) : v;
        if (c != 0 && c != NT / 2) {
            const int mr = ((NF - kf) + NF / 2) & (NF - 1);
            const int mc = ((NT - c) + NT / 2) & (NT - 1);
            const bool m1 = rowmask && rowmask[mr];
            CS[(size_t)mr * NT + mc] = m1 ? make_float2(0.f, 0.f) : make_float2(v.x, -v.y);
        }
    }
};

// secondary spectrum epilogue: |.|^2, fftshift, keep tau >= 0, post-darken, dB
struct SspecStore {
    float* sec;
    int NF, NT, R1;
    int halve, db;
    const float* pd1;   // [NT] sin^2 over the shifted fd axis, or null
    const float* pd2;   // [NF/2] sin^2 over td
    int noshift;        // 1: natural (un-fftshifted) order, full frame only
    __device__ __forceinline__ void put(int kf, int cs, float p) const {
        int row;
        if (noshift) {
            row = kf;
            cs = (cs + NT / 2) & (NT - 1);     // undo the column shift
        } else if (halve) {
            if (kf >= NF / 2) return;
            row = kf;
        } else {
            row = (kf + NF / 2) & (NF - 1);
        }
        if (pd1) {
            const float pd = (cs == NT / 2 || row == 0) ? 1.f : pd1[cs] * pd2[row];
            p = p / pd;
        }
        if (db) p = 10.f * log10f(p);
        sec[(size_t)row * NT + cs] = p;
    }
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kf = y + R1 * k;
        const float p = v.x * v.x + v.y * v.y;
        put(kf, (c + NT / 2) & (NT - 1), p);
        if (c != 0 && c != NT / 2)
            put((NF - kf) & (NF - 1), ((NT - c) + NT / 2) & (NT - 1), p);
    }
};

// ------------------------------------------------------------- ACF kernels
// forward over r2 -> |.|^2 (+ weighted power sum) -> inverse over k2 ->
// twiddle W_R^(+n2 k1); all inside one shared-memory tile.
template <int L, int W>
__global__ void __launch_bounds__(256)
acf_mid_kernel(const float2* __restrict__ A, float2* __restrict__ G, long pitch,
               int R1, int ncols, int NT, const float2* __restrict__ twf,
               const float2* __restrict__ twi, const float2* __restrict__ wRi,
               double* __restrict__ psum) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* s = reinterpret_cast<float2*>(smem_raw);
    float2* tf = s + L * W;
    float2* ti = tf + L;
    const int tid = threadIdx.x;
    constexpr int NTH = 256;
    const int c0 = blockIdx.x * W, k1 = blockIdx.y;
    const int R = R1 * L;
    for (int i = tid; i < L; i += NTH) { tf[i] = twf[i]; ti[i] = twi[i]; }
    for (int idx = tid; idx < L * W; idx += NTH) {
        const int i = idx / W, c = idx % W;
        s[idx] = (c0 + c < ncols) ? A[(size_t)(k1 * L + i) * pitch + c0 + c]
                                  : make_float2(0.f, 0.f);
    }
    __syncthreads();
    fft_axis<float, L, -1, false>(s, W, ILog2<W>::value, 1, tf, tid, NTH);
    double part = 0.0;
    for (int idx = tid; idx < L * W; idx += NTH) {
        const int c = c0 + (idx % W);
        float2 v = s[idx];
        const float p = v.x * v.x + v.y * v.y;
        s[idx] = make_float2(p, 0.f);
        if (c < ncols) part += (c == 0 || c == NT / 2) ? (double)p : 2.0 * (double)p;
    }
    __shared__ double sh[32];
    part = block_sum(part, sh);          // (its barriers also order the power writes)
    if (tid == 0) atomicAdd(psum + ((blockIdx.x + blockIdx.y) & 31), part);   // 32 slots
    __syncthreads();
    // the DIF output order is exactly the DIT input order
    fft_axis<float, L, +1, true>(s, W, ILog2<W>::value, 1, ti, tid, NTH);
    for (int idx = tid; idx < L * W; idx += NTH) {
        const int n2 = idx / W, c = idx % W;
        if (c0 + c < ncols) {
            const float2 w = wRi[(n2 * k1) & (R - 1)];
            G[(size_t)(k1 * L + n2) * pitch + c0 + c] = cmul(s[idx], w);
        }
    }
}

struct AcfRowLoad {   // output row i <- circular row (i - nf) mod PF
    const float2* Q;
    long pitch;
    int nf, PF;
    __device__ __forceinline__ float2 operator()(long row, int k) const {
        const int n = ((int)row - nf + PF) & (PF - 1);
        return Q[(size_t)n * pitch + k];
    }
};
struct AcfRowStore {
    float* acf;
    int nt, PT;
    const float* scale;    // device scalar written by acf_scale_kernel
    __device__ __forceinline__ void one(long row, int t, float x, float sc) const {
        int j;
        if (t < nt) j = t + nt;
        else if (t >= PT - nt) j = t - (PT - nt);
        else return;
        acf[(size_t)row * (2 * nt) + j] = x * sc;
    }
    __device__ __forceinline__ void operator()(long row, int n, float2 z) const {
        const float sc = *scale;
        one(row, 2 * n, z.x, sc);
        one(row, 2 * n + 1, z.y, sc);
    }
};

// stats[7] = full-plane power sum (32 slots at stats[32..63]); the factor the row pass
// multiplies with, as a float at stats[8]: 1 / sum (normalise) or the raw ifft2 scale
__global__ void acf_scale_kernel(double* stats, int normalise, double raw_scale) {
    double v = stats[32 + threadIdx.x];
    v = warp_sum(v);
    if (threadIdx.x == 0) {
        stats[7] = v;
        *reinterpret_cast<float*>(stats + 8) = (float)(normalise ? 1.0 / v : raw_scale);
    }
}

// ------------------------------------------------------------ host drivers
int stats_pass(const float* dyn, int nf, int nt, const float* wt, const float* wf,
               double swt, double swf, double* stats, cudaStream_t st);
static long half_pitch(long NT) { return ((NT / 2 + 1) + 15) & ~15L; }

// rows: real dyn [nf_live][*] -> H[nf_live][pitch] half spectra of length NT
static int rows_r2c(const DynRowLoad& ld, float2* H, long pitch, int NT,
                    long nrows, cudaStream_t st, int kmax = 1 << 30) {
    HalfStore hs{H, pitch, kmax};
    const int N = NT / 2;
    SB_ROW_DISPATCH(N, return (launch_row_r2c<float, N1, N2>(ld, hs, nrows, st)));
    return SB_OK;
}

// ---------------------------------------------------------------- TMA maps
// cuTensorMapEncodeTiled through the runtime's driver entry point (the library
// does not link libcuda).  Returns false when the driver has no such symbol.
typedef CUresult (*TmaEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TmaEncodeFn tma_encoder() {
    static TmaEncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
                cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (TmaEncodeFn)p;
        cudaGetLastError();
    }
    return fn;
}

// The tensor map of a column pass that fetches its tiles by the TMA, or false
// when the pass must use plain loads (tile_fft_kernel) instead: SB_FFT_NO_TMA
// is set, the driver has no encoder, or the live rows are not whole r2-groups.
// float2 matrix [rows][pitch] seen as float32; tiles of L rows x W complex.
// r2 > 0: rank-3 view (col, y < r2, i) of the row i * r2 + y with `nrows / r2`
// valid i (rows past them read as zeros); r2 == 0: plain rank-2 (col, row).
static bool make_tile_map(CUtensorMap* m, const float2* base, long pitch, int ncols, long nrows,
                          int r2, int L, int W) {
    static const bool no_tma = getenv("SB_FFT_NO_TMA") != nullptr;
    if (no_tma || (r2 > 0 && (nrows % r2 != 0 || nrows < r2))) return false;
    TmaEncodeFn enc = tma_encoder();
    if (!enc) return false;
    cuuint64_t gdim[3], gstr[2];
    cuuint32_t box[3], estr[3] = {1, 1, 1};
    cuuint32_t rank;
    gdim[0] = 2ull * (cuuint64_t)ncols;
    box[0] = 2u * (cuuint32_t)W;
    if (r2 > 0) {
        rank = 3;
        gdim[1] = (cuuint64_t)r2;
        gdim[2] = (cuuint64_t)(nrows / r2);
        gstr[0] = (cuuint64_t)pitch * sizeof(float2);
        gstr[1] = (cuuint64_t)r2 * pitch * sizeof(float2);
        box[1] = 1;
        box[2] = (cuuint32_t)L;
    } else {
        rank = 2;
        gdim[1] = (cuuint64_t)nrows;
        gstr[0] = (cuuint64_t)pitch * sizeof(float2);
        box[1] = (cuuint32_t)L;
    }
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, (void*)base, gdim, gstr, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Column transform of length NF (four-step split R1 x R2, two tile passes) over the
// half spectra H[live][pitch] -> epilogue stb.  Tiles are fetched by the TMA
// (cp.async.bulk.tensor, zero fill for the padded rows) when make_tile_map allows it.
template <class StoreB>
static int cols_forward(const float2* H, float2* A, long pitch, int NF, int live,
                        int ncols, StoreB stb, cudaStream_t st, int profA = -1,
                        int profB = -1) {
    int R1, R2;
    split_len(NF, &R1, &R2);
    const float2* wR = twiddle_table<float>(NF, -1, st);
    if (!wR) return SB_ERR_NOMEM;
    ZeroPadALoad<float2> la{H, pitch, R2, live};
    TwiddleAStore<float2> sa{A, pitch, R2, NF, wR};
    BlockBLoad<float2> lb{A, pitch, R2};
    CUtensorMap mapA, mapB;
    const bool tma = make_tile_map(&mapA, H, pitch, ncols, live, R2, R1, 32) &&
                     make_tile_map(&mapB, A, pitch, ncols, NF, 0, R2, 64);
    int rc = SB_OK;
    if (profA >= 0) prof_begin(profA, st);
    if (tma) {
        SB_TILE_DISPATCH(R1, rc = (launch_tile_fft_tma<LL, 32, -1, 3>(mapA, sa, ncols, R2, st)));
    } else {
        SB_TILE_DISPATCH(R1, rc = (launch_tile_fft<float, LL, 32, -1>(la, sa, ncols, R2, st)));
    }
    if (profA >= 0) prof_end(profA, st);
    if (rc) return rc;
    if (profB >= 0) prof_begin(profB, st);
    if (tma) {
        SB_TILE_DISPATCH(R2, rc = (launch_tile_fft_tma<LL, 64, -1, 2>(mapB, stb, ncols, R1, st)));
    } else {
        SB_TILE_DISPATCH(R2, rc = (launch_tile_fft<float, LL, 64, -1>(lb, stb, ncols, R1, st)));
    }
    if (profB >= 0) prof_end(profB, st);
    return rc;
}

int stats_pass(const float* dyn, int nf, int nt, const float* wt, const float* wf,
               double swt, double swf, double* stats, cudaStream_t st) {
    SB_CUDA(cudaMemsetAsync(stats, 0, 64 * sizeof(double), st));
    const bool vec = nt % 4 == 0 && ((uintptr_t)dyn & 15) == 0 && (!wt || ((uintptr_t)wt & 15) == 0);
    if (vec) dyn_stats_kernel<true><<<num_sms() * 8, 256, 0, st>>>(dyn, nf, nt, wt, wf, stats);
    else dyn_stats_kernel<false><<<num_sms() * 8, 256, 0, st>>>(dyn, nf, nt, wt, wf, stats);
    SB_LAUNCH_CHECK();
    dyn_stats_final_kernel<<<1, 1, 0, st>>>(stats, (double)nf * nt, swt, swf, wt != nullptr);
    SB_LAUNCH_CHECK();
    return SB_OK;
}


// ------------------------------------------------------------------------
// calc_sspec(prewhite=True) in float64.  Post-darkening divides by
// sin^2*sin^2 (~1e-8 at the lowest bins), which amplifies any rounding made
// AFTER the first difference; an fp32 transform loses ~1e-4 there.  The
// prewhite variant therefore differences, transforms and post-darkens in
// double (dynspec.py:3680-3717); only the dB result is narrowed to float.
// ------------------------------------------------------------------------
struct DynRowLoadD {
    const float* dyn;
    int nf, nt;
    const float* wt;
    const float* wf;
    const double* stats;   // [4]=mu1 [5]=mu2
    __device__ __forceinline__ double val(int f, int t) const {
        double v = (double)dyn[(size_t)f * nt + t] - stats[4];
        if (wt) v *= (double)wt[t] * (double)wf[f];
        return v - stats[5];
    }
    __device__ __forceinline__ double get(int f, int t) const {
        if (t >= nt - 1) return 0.0;
        return val(f + 1, t + 1) - val(f + 1, t) - val(f, t + 1) + val(f, t);
    }
    __device__ __forceinline__ double2 operator()(long row, int n) const {
        return make_double2(get((int)row, 2 * n), get((int)row, 2 * n + 1));
    }
};
struct SspecStoreD {     // halved frame only (prewhite requires halve)
    float* sec;
    int NF, NT, R1, db;
    __device__ __forceinline__ void put(int kf, int cs, double p) const {
        if (kf >= NF / 2) return;
        const double pi = 3.14159265358979323846;
        if (!(cs == NT / 2 || kf == 0)) {
            const double s1 = sin(pi / NT * (double)(cs - NT / 2));   // fd = cs - NT/2
            const double s2 = sin(pi / NF * (double)kf);
            p = p / ((s1 * s1) * (s2 * s2));
        }
        sec[(size_t)kf * NT + cs] = db ? (float)(10.0 * log10(p)) : (float)p;
    }
    __device__ __forceinline__ void operator()(int y, int k, int c, double2 v) const {
        const int kf = y + R1 * k;
        const double p = v.x * v.x + v.y * v.y;
        put(kf, (c + NT / 2) & (NT - 1), p);
        if (c != 0 && c != NT / 2)
            put((NF - kf) & (NF - 1), ((NT - c) + NT / 2) & (NT - 1), p);
    }
};

static int sspec_prewhite_f64(const float* dyn, int nf, int nt, const float* wt,
                              const float* wf, const double* stats, int db, float* sec,
                              int NF, int NT, cudaStream_t st) {
    if (NT / 2 > 8192) {
        set_error("calc_sspec(prewhite=True): float64 path supports nt <= 8192");
        return SB_ERR_UNSUPPORTED;
    }
    const long pitch = half_pitch(NT);
    const int live = nf - 1;
    double2* H = (double2*)workspace(3, (size_t)live * pitch * sizeof(double2));
    double2* A = (double2*)workspace(4, (size_t)NF * pitch * sizeof(double2));
    if (!H || !A) return SB_ERR_NOMEM;
    DynRowLoadD ld{dyn, nf, nt, wt, wf, stats};
    PlainRowStore<double2> hs{H, pitch};
    int rc = SB_OK;
    const int N = NT / 2;
    SB_ROW_DISPATCH(N, rc = (launch_row_r2c<double, N1, N2>(ld, hs, live, st)));
    if (rc) return rc;
    int R1, R2;
    split_len(NF, &R1, &R2);
    ZeroPadALoad<double2> la{H, pitch, R2, live};
    SspecStoreD ss{sec, NF, NT, R1, db};
    return cols_generic<double, -1>(la, A, pitch, NF, NT / 2 + 1, ss, st);
}

// Dynspec.calc_sspec (dynspec.py:3664-3721)
int sspec(const float* dyn, int nf, int nt, const float* wt, const float* wf,
          double swt, double swf, int prewhite, int halve, int db,
          const float* pd1, const float* pd2, float* sec, cudaStream_t st,
          int noshift = 0) {
    ProfScope prof(PROF_SSPEC, st);
    const int NF = 2 * next_pow2(nf), NT = 2 * next_pow2(nt);  // 2^(ceil(log2 n)+1)
    if (NT / 2 < 8 || NT / 2 > 16384 || NF > 65536 || NF < 4) {
        set_error("calc_sspec: dynspec %dx%d outside the supported sizes (nf 2..32768, nt 5..16384)",
                  nf, nt);
        return SB_ERR_UNSUPPORTED;
    }
    const long pitch = half_pitch(NT);
    double* stats = (double*)workspace(0, 64 * sizeof(double));
    const int live = prewhite ? nf - 1 : nf;
    float2* H = (float2*)workspace(3, (size_t)live * pitch * sizeof(float2));
    float2* A = (float2*)workspace(4, (size_t)NF * pitch * sizeof(float2));
    if (!stats || !H || !A) return SB_ERR_NOMEM;
    int rc = stats_pass(dyn, nf, nt, wt, wf, swt, swf, stats, st);
    if (rc) return rc;
    if (prewhite) return sspec_prewhite_f64(dyn, nf, nt, wt, wf, stats, db, sec, NF, NT, st);
    DynRowLoad ld{dyn, nf, nt, wt, wf, stats, 0, prewhite, 0.f};
    rc = rows_r2c(ld, H, pitch, NT, live, st);
    if (rc) return rc;
    int R1, R2;
    split_len(NF, &R1, &R2);
    SspecStore ss{sec, NF, NT, R1, halve, db, prewhite ? pd1 : nullptr, pd2, noshift};
    return cols_forward(H, A, pitch, NF, live, NT / 2 + 1, ss, st);
}

// sum |dyn - c| (c = stats[4], the mean, when use_mean; else the constant sub)
__global__ void dyn_l1_kernel(const float* __restrict__ dyn, long total, const double* __restrict__ stats,
                              int use_mean, float sub, double* __restrict__ acc) {
    const float c = use_mean ? (float)stats[4] : sub;
    double s = 0.0;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long)gridDim.x * blockDim.x) {
        const float v = fabsf(dyn[i] - c);
        s += (v == v) ? (double)v : 0.0;
    }
    __shared__ double sh[32];
    s = block_sum(s, sh);
    if (threadIdx.x == 0) atomicAdd(acc, s);
}
__global__ void dyn_l1_final_kernel(const double* acc, const double* stats, int use_mean, float sub,
                                    double npix_padded, float* out) {
    const double c = use_mean ? fabs(stats[4]) : fabs((double)sub);
    double b = (acc[0] + c * npix_padded) * 1.000001;
    if (!(b < 3.0e38)) b = 3.0e38;
    *out = (float)b;
}

// upper bound of max |CS| of conj_spectrum() for the same inputs: the L1 norm of what is
// transformed (dyn - c on the live pixels) + the DC correction |c| NF NT
int conj_spectrum_bound(const float* dyn, int nf, int nt, int npad, float pad_value, float* out,
                        cudaStream_t st) {
    double* stats = (double*)workspace(0, 64 * sizeof(double));
    if (!stats) return SB_ERR_NOMEM;
    const bool dev_mean = pad_value != pad_value;
    if (dev_mean) {
        int rc = stats_pass(dyn, nf, nt, nullptr, nullptr, 0, 0, stats, st);
        if (rc) return rc;
    }
    double* acc = stats + 24;
    SB_CUDA(cudaMemsetAsync(acc, 0, sizeof(double), st));
    dyn_l1_kernel<<<num_sms() * 4, 256, 0, st>>>(dyn, (long)nf * nt, stats, dev_mean ? 1 : 0,
                                                 dev_mean ? 0.f : pad_value, acc);
    SB_LAUNCH_CHECK();
    dyn_l1_final_kernel<<<1, 1, 0, st>>>(acc, stats, dev_mean ? 1 : 0, dev_mean ? 0.f : pad_value,
                                         (double)(npad + 1) * nf * (double)(npad + 1) * nt, out);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// ------------------------------------------------------------------------
// 2-D transforms of sizes that are NOT powers of two (e.g. the reference
// tutorial's 64 x 150 chunk -> 256 x 600 conjugate spectrum, and its inverse in
// phase retrieval): Bluestein / chirp-z on both axes on top of the power-of-two
// engine.
//   X[k] = w[k] * sum_n (x[n] w[n]) conj(w)[k - n],  w[n] = exp(-i pi n^2 / N)
// = w[k] * IFFT_M( FFT_M(x w) * FFT_M(b) )[k],  M = 2^p >= 2N - 1.
// Full plane output (no Hermitian shortcut), generic fftshift (odd N too).
// Chirp tables and the load / store functors of these passes: fft_functors.cuh; the
// 2-D driver chirp_fft2: fft_kernels.cuh
// ------------------------------------------------------------------------
// chirp w[N] and the transformed kernel B = FFT_M(b)
int bluestein_tables(int N, int M, float2* w, float2* B, float2* scratch, cudaStream_t st) {
    chirp_fill_kernel<<<(M + 255) / 256, 256, 0, st>>>(w, B, N, M);
    SB_LAUNCH_CHECK();
    if (M <= 16384) {
        SB_CUDA(cudaMemcpyAsync(scratch, B, (size_t)M * sizeof(float2),
                                cudaMemcpyDeviceToDevice, st));
        VecLoad ld{scratch};
        VecStore vs{B};
        int rc = SB_OK;
        SB_ROW_DISPATCH(M, rc = (launch_row_c2c<float, N1, N2, -1>(ld, vs, 1, st)));
        return rc;
    }
    int R1, R2;
    split_len(M, &R1, &R2);
    SB_CUDA(cudaMemcpyAsync(scratch, B, (size_t)M * sizeof(float2),
                            cudaMemcpyDeviceToDevice, st));
    ColVecLoad la{scratch, R2};
    ColVecStore sb_{B, R1};
    return cols_generic<float, -1>(la, scratch + M, 1, M, 1, sb_, st);
}

// conjugate spectrum of a zero(/constant)-padded chunk
// (ththmod.py:777-787, dynspec.py:1572-1579)
int conj_spectrum(const float* dyn, int nf, int nt, int npad, float pad_value,
                  const unsigned char* rowmask, int half, long cs_pitch, int ncols_keep,
                  float2* CS, cudaStream_t st) {
    const long NFl = (long)(npad + 1) * nf, NTl = (long)(npad + 1) * nt;
    if (!is_pow2(NFl) || !is_pow2(NTl) || NTl / 2 < 8 || NFl < 4) {
        // arbitrary lengths: chirp-z on both axes, full plane only
        if (half) {
            set_error("conjugate spectrum: half-plane output needs power-of-two "
                      "padded sizes (got %ldx%ld)", NFl, NTl);
            return SB_ERR_ARG;
        }
        double* bstats = nullptr;
        if (pad_value != pad_value) {
            bstats = (double*)workspace(0, 64 * sizeof(double));
            if (!bstats) return SB_ERR_NOMEM;
            int rc0 = stats_pass(dyn, nf, nt, nullptr, nullptr, 0, 0, bstats, st);
            if (rc0) return rc0;
            pad_value = 0.f;
        }
        const int NF = (int)NFl, NT = (int)NTl;
        return chirp_fft2(ChirpRowLoad{dyn, nt, nullptr, bstats, pad_value}, NF, NT, nf, NT,
                          [&](int R1, const float2* wF, int MF) {
                              return ChirpCsStore{CS, NF, NT, R1, wF, 1.0f / (float)MF, rowmask,
                                                  pad_value * (float)NF * (float)NT, bstats};
                          }, "conjugate spectrum (chirp-z): padded size", st);
    }
    if (NTl / 2 > 16384 || NFl > 65536) {
        set_error("conjugate spectrum: padded size %ldx%ld too large "
                  "(rows <= 65536, cols <= 32768)", NFl, NTl);
        return SB_ERR_UNSUPPORTED;
    }
    const int NF = (int)NFl, NT = (int)NTl;
    const long pitch = half_pitch(NT);
    float2* H = (float2*)workspace(3, (size_t)nf * pitch * sizeof(float2));
    float2* A = (float2*)workspace(4, (size_t)NF * pitch * sizeof(float2));
    if (!H || !A) return SB_ERR_NOMEM;
    // pad_value = NaN: pad with the mean of the chunk (ththmod.py:781), which
    // is then computed on the device instead of a host pass over the data
    const bool dev_mean = pad_value != pad_value;
    double* stats = nullptr;
    if (dev_mean) {
        stats = (double*)workspace(0, 64 * sizeof(double));
        if (!stats) return SB_ERR_NOMEM;
        int rc0 = stats_pass(dyn, nf, nt, nullptr, nullptr, 0, 0, stats, st);
        if (rc0) return rc0;
        pad_value = 0.f;
    }
    DynRowLoad ld{dyn, nf, nt, nullptr, nullptr, stats, dev_mean ? 3 : 2, 0, pad_value};
    // only the first ncols fd >= 0 columns are wanted (the theta-theta gather
    // never reads beyond max(theta) - min(theta)): the column passes, which
    // dominate, shrink proportionally
    int ncols = NT / 2 + 1;
    if (half && ncols_keep > 0 && ncols_keep < ncols) ncols = ncols_keep;
    prof_begin(PROF_CS_ROWS, st);
    int rc = rows_r2c(ld, H, pitch, NT, nf, st, ncols);
    prof_end(PROF_CS_ROWS, st);
    if (rc) return rc;
    int R1, R2;
    split_len(NF, &R1, &R2);
    CsStore cs{CS, NF, NT, R1, rowmask, pad_value * (float)NF * (float)NT, half, cs_pitch,
               dev_mean ? stats : nullptr};
    return cols_forward(H, A, pitch, NF, nf, ncols, cs, st, PROF_CS_COLA, PROF_CS_COLB);
}

// Dynspec.calc_acf(method='direct') (dynspec.py:3780-3797)
int acf(const float* dyn, int nf, int nt, int subtract_mean, int normalise,
        float* out, cudaStream_t st) {
    ProfScope prof(PROF_ACF, st);
    const int PF = next_pow2(2L * nf), PT = next_pow2(2L * nt);
    if (PT / 2 < 8 || PT / 2 > 16384 || PF > 65536 || PF < 4) {
        set_error("calc_acf: dynspec %dx%d outside the supported sizes (nf 2..32768, nt 5..16384)",
                  nf, nt);
        return SB_ERR_UNSUPPORTED;
    }
    const long pitch = half_pitch(PT);
    double* stats = (double*)workspace(0, 64 * sizeof(double));
    float2* H = (float2*)workspace(3, (size_t)nf * pitch * sizeof(float2));
    float2* A = (float2*)workspace(4, (size_t)PF * pitch * sizeof(float2));
    float2* G = (float2*)workspace(5, (size_t)PF * pitch * sizeof(float2));
    if (!stats || !H || !A || !G) return SB_ERR_NOMEM;
    int rc = stats_pass(dyn, nf, nt, nullptr, nullptr, 0, 0, stats, st);
    if (rc) return rc;
    DynRowLoad ld{dyn, nf, nt, nullptr, nullptr, stats, subtract_mean ? 1 : 2, 0, 0.f};
    rc = rows_r2c(ld, H, pitch, PT, nf, st);
    if (rc) return rc;
    int R1, R2;
    split_len(PF, &R1, &R2);
    const int ncols = PT / 2 + 1;
    // forward pass A
    {
        const float2* wR = twiddle_table<float>(PF, -1, st);
        if (!wR) return SB_ERR_NOMEM;
        ZeroPadALoad<float2> la{H, pitch, R2, nf};
        TwiddleAStore<float2> sa{A, pitch, R2, PF, wR};
        CUtensorMap mapA;
        if (make_tile_map(&mapA, H, pitch, ncols, nf, R2, R1, 32)) {
            SB_TILE_DISPATCH(R1, rc = (launch_tile_fft_tma<LL, 32, -1, 3>(mapA, sa, ncols, R2, st)));
        } else {
            SB_TILE_DISPATCH(R1, rc = (launch_tile_fft<float, LL, 32, -1>(la, sa, ncols, R2, st)));
        }
        if (rc) return rc;
    }
    // fused forward pass B -> power -> inverse over k2
    {
        const float2* wRi = twiddle_table<float>(PF, +1, st);
        const float2* twf = twiddle_table<float>(R2, -1, st);
        const float2* twi = twiddle_table<float>(R2, +1, st);
        if (!wRi || !twf || !twi) return SB_ERR_NOMEM;
        dim3 grid((ncols + 31) / 32, R1);
        SB_TILE_DISPATCH(R2, {
            auto kern = acf_mid_kernel<LL, 32>;
            const size_t smem = (size_t)(LL * 32 + 2 * LL) * sizeof(float2);
            SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<grid, 256, smem, st>>>(A, G, pitch, R1, ncols, PT, twf, twi, wRi, stats + 32);
        });
        SB_LAUNCH_CHECK();
        acf_scale_kernel<<<1, 32, 0, st>>>(stats, normalise, 1.0 / ((double)PF * (double)PT));
        SB_LAUNCH_CHECK();
    }
    // inverse over k1 -> Q (reuse A)
    {
        StrideALoad<float2> li{G, pitch, R2};      // y = n2, i = k1
        NaturalBStore<float2> si{A, pitch, R2};    // n = n2 + R2 n1
        CUtensorMap mapG;
        if (make_tile_map(&mapG, G, pitch, ncols, PF, R2, R1, 32)) {
            SB_TILE_DISPATCH(R1, rc = (launch_tile_fft_tma<LL, 32, +1, 3>(mapG, si, ncols, R2, st)));
        } else {
            SB_TILE_DISPATCH(R1, rc = (launch_tile_fft<float, LL, 32, +1>(li, si, ncols, R2, st)));
        }
        if (rc) return rc;
    }
    // rows: half spectrum -> real, crop to lags [-nf, nf) x [-nt, nt)
    AcfRowLoad rl{A, pitch, nf, PF};
    AcfRowStore rs{out, nt, PT, reinterpret_cast<const float*>(stats + 8)};
    const int N = PT / 2;
    SB_ROW_DISPATCH(N, return (launch_row_c2r<float, N1, N2>(rl, rs, 2L * nf, st)));
    return SB_OK;
}

// real part of FFT2 of a real array with fftshift, scaled by 1/sum (ACF through
// the secondary spectrum, dynspec.py:3798-3807)
struct RealShiftStore {
    float* out;
    int NF, NT, R1;
    const double* stats;   // [0] = sum of the input (the zero-frequency bin)
    int normalise;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kf = y + R1 * k;
        const float val = normalise ? (float)((double)v.x / stats[0]) : v.x;
        out[(size_t)((kf + NF / 2) & (NF - 1)) * NT + ((c + NT / 2) & (NT - 1))] = val;
        if (c != 0 && c != NT / 2)
            out[(size_t)(((NF - kf) + NF / 2) & (NF - 1)) * NT + (((NT - c) + NT / 2) & (NT - 1))] = val;
    }
};

// Dynspec.calc_acf(method='sspec'): FFT2 of the un-halved, un-shifted linear
// secondary spectrum (dynspec.py:3798-3807)
int acf_sspec(const float* dyn, int nf, int nt, const float* wt, const float* wf,
              double swt, double swf, int normalise, float* out, cudaStream_t st) {
    const int NF = 2 * next_pow2(nf), NT = 2 * next_pow2(nt);
    float* P = (float*)workspace(5, (size_t)NF * NT * sizeof(float));
    if (!P) return SB_ERR_NOMEM;
    int rc = sspec(dyn, nf, nt, wt, wf, swt, swf, 0, 0, 0, nullptr, nullptr, P, st, 1);
    if (rc) return rc;
    ProfScope prof(PROF_ACF, st);
    if (NT / 2 < 8 || NT / 2 > 16384) {
        set_error("calc_acf(sspec): size outside supported FFT sizes");
        return SB_ERR_UNSUPPORTED;
    }
    const long pitch = half_pitch(NT);
    double* stats = (double*)workspace(0, 64 * sizeof(double));
    float2* H = (float2*)workspace(3, (size_t)NF * pitch * sizeof(float2));
    float2* A = (float2*)workspace(4, (size_t)NF * pitch * sizeof(float2));
    if (!stats || !H || !A) return SB_ERR_NOMEM;
    rc = stats_pass(P, NF, NT, nullptr, nullptr, 0, 0, stats, st);
    if (rc) return rc;
    DynRowLoad ld{P, NF, NT, nullptr, nullptr, nullptr, 2, 0, 0.f};
    rc = rows_r2c(ld, H, pitch, NT, NF, st);
    if (rc) return rc;
    int R1, R2;
    split_len(NF, &R1, &R2);
    RealShiftStore rs{out, NF, NT, R1, stats, normalise};
    return cols_forward(H, A, pitch, NF, NF, NT / 2 + 1, rs, st);
}

}  // namespace sb
