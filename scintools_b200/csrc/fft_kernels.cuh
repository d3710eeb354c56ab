// Generic FFT kernels built on fft_core.cuh.
//
//  tile_fft_kernel : FFT along the STRIDED axis of a row-major 2-D array, one
//                    [L rows x W columns] tile per CTA (W*sizeof(C) = 256 B
//                    contiguous per row).  Long column transforms are done as
//                    a four-step split R = R1 * R2 with two launches of this
//                    kernel (pass A: stride-R2 rows + twiddle, pass B: blocks
//                    of R2 consecutive rows); load/store functors fuse the
//                    pre/post processing (zero-pad pruning, twiddles, |.|^2,
//                    fftshift, Hermitian expansion, dB ...).
//  row_fft_*_kernel: FFT along the CONTIGUOUS axis, one row per CTA, the
//                    whole row resident in shared memory as an N1 x (N2+1)
//                    matrix (four-step inside shared memory).  Variants:
//                    complex->complex, real->half-spectrum, half-spectrum->real.
#pragma once
#include <cuda.h>      // CUtensorMap (type only; the encoder is fetched through the runtime)

#include "fft_core.cuh"
#include "fft_functors.cuh"
#include "tma.cuh"

namespace sb {

// master twiddle tables: W_N^(dir*i), i < N, in global memory (L2 resident)
template <typename T> const cx<T>* twiddle_table(int N, int dir, cudaStream_t st);

template <int V> struct ILog2 { static constexpr int value = 1 + ILog2<V / 2>::value; };
template <> struct ILog2<1> { static constexpr int value = 0; };

// --------------------------------------------------------------------------
// strided-axis tile kernel.  grid = (column tiles, Y).  Load(y, i, c) returns
// element i of the length-L sequence for column c of problem y; Store(y, k, c,
// v) receives output bin k.  DIF transform, digit-reversed read-out.
// --------------------------------------------------------------------------
template <typename T, int L, int W, int DIR, class Load, class Store>
__global__ void __launch_bounds__(256)
tile_fft_kernel(Load ld, Store st, const cx<T>* __restrict__ twL, int ncols) {
    using C = cx<T>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    C* tw = s + L * W;
    const int tid = threadIdx.x;
    constexpr int NT = 256;
    const int c0 = blockIdx.x * W;
    const int y = blockIdx.y;
    for (int i = tid; i < L; i += NT) tw[i] = twL[i];
    for (int idx = tid; idx < L * W; idx += NT) {
        const int i = idx / W, c = idx % W;
        s[idx] = (c0 + c < ncols) ? ld(y, i, c0 + c) : mkc<T>(0, 0);
    }
    __syncthreads();
    fft_axis<T, L, DIR, false>(s, W, ILog2<W>::value, 1, tw, tid, NT);
    for (int idx = tid; idx < L * W; idx += NT) {
        const int k = idx / W, c = idx % W;
        if (c0 + c < ncols) st(y, k, c0 + c, s[digit_pos<L>(k) * W + c]);
    }
}

template <typename T, int L, int W, int DIR, class Load, class Store>
int launch_tile_fft(Load ld, Store st, int ncols, int ny, cudaStream_t stream) {
    const cx<T>* tw = twiddle_table<T>(L, DIR, stream);
    if (!tw) return SB_ERR_NOMEM;
    auto kern = tile_fft_kernel<T, L, W, DIR, Load, Store>;
    const size_t smem = (size_t)(L * W + L) * sizeof(cx<T>);
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((ncols + W - 1) / W, ny);
    kern<<<grid, 256, smem, stream>>>(ld, st, tw, ncols);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// --------------------------------------------------------------------------
// The same tile transform with the tile fetched by the TMA: ONE
// cp.async.bulk.tensor box load ([L rows][W complex] -> dense shared-memory
// tile, exactly the layout fft_axis works on) issued by one thread and awaited
// on an mbarrier by all; rows / columns outside the tensor arrive as zeros
// (zero padding of the live rows and of the last column tile for free).
//   rank 3 (pass A of the four-step split): tensor (col, y = r2, i = r1), row
//          r1 * R2 + r2, box {2W floats, 1, L}, coordinates {2 c0, y, 0};
//   rank 2 (pass B): tensor (col, row), box {2W, L}, coordinates {2 c0, y * L}.
// float2 data only (the tensor is described as float32 with 2 W floats per row).
// --------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            unsigned long long* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1,
                                            unsigned long long* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

template <int L, int W, int DIR, int RANK, class Store>
__global__ void __launch_bounds__(256)
tile_fft_tma_kernel(const __grid_constant__ CUtensorMap tmap, Store st,
                    const float2* __restrict__ twL, int ncols) {
    extern __shared__ __align__(128) unsigned char smem_tma[];
    float2* s = reinterpret_cast<float2*>(smem_tma);
    float2* tw = s + L * W;
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(tw + L);
    const int tid = threadIdx.x;
    constexpr int NT = 256;
    const int c0 = blockIdx.x * W;
    const int y = blockIdx.y;
    if (tid == 0) {
        mbar_init(bar, 1);
        fence_mbarrier_init();
        mbar_expect_tx(bar, (unsigned)(L * W * sizeof(float2)));
        if (RANK == 3) tma_load_3d(s, &tmap, 2 * c0, y, 0, bar);
        else tma_load_2d(s, &tmap, 2 * c0, y * L, bar);
    }
    for (int i = tid; i < L; i += NT) tw[i] = twL[i];
    __syncthreads();                       // barrier initialised (and tw in place) for everybody
    while (!mbar_try_wait(bar, 0)) {}
    fft_axis<float, L, DIR, false>(s, W, ILog2<W>::value, 1, tw, tid, NT);
    for (int idx = tid; idx < L * W; idx += NT) {
        const int k = idx / W, c = idx % W;
        if (c0 + c < ncols) st(y, k, c0 + c, s[digit_pos<L>(k) * W + c]);
    }
}

template <int L, int W, int DIR, int RANK, class Store>
int launch_tile_fft_tma(const CUtensorMap& map, Store st, int ncols, int ny, cudaStream_t stream) {
    const float2* tw = twiddle_table<float>(L, DIR, stream);
    if (!tw) return SB_ERR_NOMEM;
    auto kern = tile_fft_tma_kernel<L, W, DIR, RANK, Store>;
    const size_t smem = (size_t)(L * W + L) * sizeof(float2) + 16;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((ncols + W - 1) / W, ny);
    kern<<<grid, 256, smem, stream>>>(map, st, tw, ncols);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// --------------------------------------------------------------------------
// contiguous-axis kernels: N = N1 * N2 complex points in shared memory.
// --------------------------------------------------------------------------
template <typename T, int N1, int N2> struct RowSmem {
    static constexpr int N = N1 * N2;
    static constexpr int RS = N2 + 1;  // padded row stride (odd)
    // data + tw1[N1] + tw2[N2] + twl[N2] + a[N1+1] + b[N2]
    static constexpr size_t bytes = (size_t)(N1 * RS + N1 + 3 * N2 + N1 + 1) * sizeof(cx<T>);
};

// tables a row kernel needs, all slices of master tables
template <typename T> struct RowTables {
    const cx<T>* wN;    // W_N^(dir i), i < N
    const cx<T>* w2N;   // W_2N^(-i) (forward sign), i < 2N ; only R2C / C2R
};

template <typename T, int N1, int N2, int DIR>
__device__ __forceinline__ void row_load_tables(cx<T>* tw1, cx<T>* tw2, cx<T>* twl,
                                                const cx<T>* __restrict__ wN,
                                                int tid, int nt) {
    for (int i = tid; i < N1; i += nt) tw1[i] = wN[i * N2];   // W_N1^i
    for (int i = tid; i < N2; i += nt) {
        tw2[i] = wN[i * N1];                                   // W_N2^i
        twl[i] = wN[i];                                        // W_N^i
    }
}

// the transform proper: s holds x[n] at [digit_pos<N1>(n / N2)][n % N2];
// afterwards X[k1 + N1 k2] sits at [k1][digit_pos<N2>(k2)].
template <typename T, int N1, int N2, int DIR>
__device__ __forceinline__ void row_fft_smem(cx<T>* s, const cx<T>* tw1,
                                             const cx<T>* tw2, const cx<T>* twl,
                                             int tid, int nt) {
    using C = cx<T>;
    constexpr int RS = N2 + 1;
    constexpr int N = N1 * N2;
    fft_axis<T, N1, DIR, true>(s, RS, ILog2<N2>::value, 1, tw1, tid, nt);
    // twiddle W_N^(n2 k1) = W_N1^(q / N2) * W_N^(q % N2), q = n2 k1
    for (int idx = tid; idx < N; idx += nt) {
        const int k1 = idx / N2, n2 = idx % N2;
        const int q = k1 * n2;
        if (q) {
            C w = cmul(tw1[q / N2], twl[q % N2]);
            s[k1 * RS + n2] = cmul(s[k1 * RS + n2], w);
        }
    }
    __syncthreads();
    fft_axis<T, N2, DIR, false>(s, 1, ILog2<N1>::value, RS, tw2, tid, nt);
}

template <typename T, int N1, int N2>
__device__ __forceinline__ int row_in_pos(int n) {   // where x[n] is loaded
    return digit_pos<N1>(n / N2) * (N2 + 1) + (n % N2);
}
template <typename T, int N1, int N2>
__device__ __forceinline__ int row_out_pos(int k) {  // where X[k] ends up
    return (k % N1) * (N2 + 1) + digit_pos<N2>(k / N1);
}

// complex -> complex
template <typename T, int N1, int N2, int DIR, class Load, class Store>
__global__ void __launch_bounds__(sizeof(T) == 4 ? 1024 : 512) row_fft_c2c_kernel(Load ld, Store st, RowTables<T> tabs) {
    using C = cx<T>;
    constexpr int N = N1 * N2, RS = N2 + 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    C* tw1 = s + N1 * RS; C* tw2 = tw1 + N1; C* twl = tw2 + N2;
    const int tid = threadIdx.x, nt = blockDim.x;
    const long row = blockIdx.x;
    row_load_tables<T, N1, N2, DIR>(tw1, tw2, twl, tabs.wN, tid, nt);
    for (int n = tid; n < N; n += nt) s[row_in_pos<T, N1, N2>(n)] = ld(row, n);
    __syncthreads();
    row_fft_smem<T, N1, N2, DIR>(s, tw1, tw2, twl, tid, nt);
    for (int k = tid; k < N; k += nt) st(row, k, s[row_out_pos<T, N1, N2>(k)]);
}

// hooks of the row load functors (overloaded next to the functor, found by ADL): read
// per-launch constants once per thread; how many leading entries of a row can be non-zero
template <class L> __device__ __forceinline__ void row_load_init(L&) {}
template <class L> __device__ __forceinline__ int row_load_live(const L&, int N) { return N; }

// real (length 2N, packed two per complex) -> half spectrum X[0..N], forward
// Load(row, n) returns (x[2n], x[2n+1]); Store(row, k, X[k]) for k in [0, N].
template <typename T, int N1, int N2, class Load, class Store>
__global__ void __launch_bounds__(sizeof(T) == 4 ? 1024 : 512) row_fft_r2c_kernel(Load ld, Store st, RowTables<T> tabs) {
    using C = cx<T>;
    constexpr int N = N1 * N2, RS = N2 + 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    C* tw1 = s + N1 * RS; C* tw2 = tw1 + N1; C* twl = tw2 + N2;
    C* ta = twl + N2;      // W_2N^(kh N2), kh <= N1
    C* tb = ta + N1 + 1;   // W_2N^(kl),   kl <  N2
    const int tid = threadIdx.x, nt = blockDim.x;
    const long row = blockIdx.x;
    row_load_tables<T, N1, N2, -1>(tw1, tw2, twl, tabs.wN, tid, nt);
    for (int i = tid; i <= N1; i += nt) ta[i] = tabs.w2N[(i * N2) % (2 * N)];
    for (int i = tid; i < N2; i += nt) tb[i] = tabs.w2N[i];
    Load lld = ld;
    row_load_init(lld);
    const int live = row_load_live(lld, N);          // zero padding beyond: no loads
    for (int n = tid; n < N; n += nt)
        s[row_in_pos<T, N1, N2>(n)] = n < live ? lld(row, n) : mkc<T>(0, 0);
    __syncthreads();
    row_fft_smem<T, N1, N2, -1>(s, tw1, tw2, twl, tid, nt);
    const T half = (T)0.5;
    for (int k = tid; k <= N / 2; k += nt) {
        const int km = (N - k) % N;
        C A = s[row_out_pos<T, N1, N2>(k)];
        C B = cconj(s[row_out_pos<T, N1, N2>(km)]);
        C xe = mkc<T>((A.x + B.x) * half, (A.y + B.y) * half);
        C d = mkc<T>((A.x - B.x) * half, (A.y - B.y) * half);
        C xo = mkc<T>(d.y, -d.x);                      // -i * d
        C w = cmul(ta[k / N2], tb[k % N2]);           // W_2N^k
        C wx = cmul(w, xo);
        st(row, k, cadd(xe, wx));
        st(row, N - k, cconj(csub(xe, wx)));
    }
}

// half spectrum X[0..N] -> real length 2N, UNNORMALISED inverse.
// Load(row, k) returns X[k]; Store(row, n, z) receives (x[2n], x[2n+1]).
template <typename T, int N1, int N2, class Load, class Store>
__global__ void __launch_bounds__(sizeof(T) == 4 ? 1024 : 512) row_fft_c2r_kernel(Load ld, Store st, RowTables<T> tabs) {
    using C = cx<T>;
    constexpr int N = N1 * N2, RS = N2 + 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    C* tw1 = s + N1 * RS; C* tw2 = tw1 + N1; C* twl = tw2 + N2;
    C* ta = twl + N2;
    C* tb = ta + N1 + 1;
    const int tid = threadIdx.x, nt = blockDim.x;
    const long row = blockIdx.x;
    row_load_tables<T, N1, N2, +1>(tw1, tw2, twl, tabs.wN, tid, nt);
    for (int i = tid; i <= N1; i += nt) ta[i] = tabs.w2N[(i * N2) % (2 * N)];
    for (int i = tid; i < N2; i += nt) tb[i] = tabs.w2N[i];
    __syncthreads();
    for (int k = tid; k <= N / 2; k += nt) {
        C Xk = ld(row, k);
        C Xm = cconj(ld(row, N - k));
        C S = cadd(Xk, Xm), D = csub(Xk, Xm);
        C w = cmul(ta[k / N2], tb[k % N2]);           // W_2N^k (forward sign)
        C iD = mkc<T>(-D.y, D.x);                      // i * D
        C Zk = cadd(S, cmul(cconj(w), iD));            // S + i conj(w) D
        C iDc = mkc<T>(D.y, D.x);                      // i * conj(D)
        C Zm = cadd(cconj(S), cmul(w, iDc));           // conj(S) + i w conj(D)
        s[row_in_pos<T, N1, N2>(k)] = Zk;
        if (k != 0 && 2 * k != N) s[row_in_pos<T, N1, N2>(N - k)] = Zm;
    }
    __syncthreads();
    row_fft_smem<T, N1, N2, +1>(s, tw1, tw2, twl, tid, nt);
    for (int n = tid; n < N; n += nt) st(row, n, s[row_out_pos<T, N1, N2>(n)]);
}

inline int row_threads(int N, int elem_bytes = 8) {
    // N / 16 threads: one radix-16 butterfly per thread and pass, and two CTAs share an SM for
    // rows up to 8192 points, overlapping their load / transform / store phases (16384-point
    // rows keep 1024 threads either way)
    int t = N / 16;
    if (t < 32) t = 32;
    const int cap = elem_bytes <= 8 ? 1024 : 512;   // fp32 rows: 32 warps hide latency
    if (t > cap) t = cap;
    return t;
}

template <typename T, int N1, int N2, int DIR, class Load, class Store>
int launch_row_c2c(Load ld, Store st, long nrows, cudaStream_t stream) {
    constexpr int N = N1 * N2;
    RowTables<T> tabs;
    tabs.wN = twiddle_table<T>(N, DIR, stream);
    tabs.w2N = nullptr;
    if (!tabs.wN) return SB_ERR_NOMEM;
    auto kern = row_fft_c2c_kernel<T, N1, N2, DIR, Load, Store>;
    const size_t smem = RowSmem<T, N1, N2>::bytes;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)nrows, row_threads(N, (int)sizeof(cx<T>)), smem, stream>>>(ld, st, tabs);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
template <typename T, int N1, int N2, class Load, class Store>
int launch_row_r2c(Load ld, Store st, long nrows, cudaStream_t stream) {
    constexpr int N = N1 * N2;
    RowTables<T> tabs;
    tabs.wN = twiddle_table<T>(N, -1, stream);
    tabs.w2N = twiddle_table<T>(2 * N, -1, stream);
    if (!tabs.wN || !tabs.w2N) return SB_ERR_NOMEM;
    auto kern = row_fft_r2c_kernel<T, N1, N2, Load, Store>;
    const size_t smem = RowSmem<T, N1, N2>::bytes;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)nrows, row_threads(N, (int)sizeof(cx<T>)), smem, stream>>>(ld, st, tabs);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
template <typename T, int N1, int N2, class Load, class Store>
int launch_row_c2r(Load ld, Store st, long nrows, cudaStream_t stream) {
    constexpr int N = N1 * N2;
    RowTables<T> tabs;
    tabs.wN = twiddle_table<T>(N, +1, stream);
    tabs.w2N = twiddle_table<T>(2 * N, -1, stream);
    if (!tabs.wN || !tabs.w2N) return SB_ERR_NOMEM;
    auto kern = row_fft_c2r_kernel<T, N1, N2, Load, Store>;
    const size_t smem = RowSmem<T, N1, N2>::bytes;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)nrows, row_threads(N, (int)sizeof(cx<T>)), smem, stream>>>(ld, st, tabs);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// size dispatch helpers: call F<N1, N2>() for N = N1*N2 = 2^p, p in [3, 14]
#define SB_ROW_DISPATCH(N, ...)                                         \
    switch (N) {                                                        \
        case 8: { constexpr int N1 = 4, N2 = 2; __VA_ARGS__; } break;          \
        case 16: { constexpr int N1 = 4, N2 = 4; __VA_ARGS__; } break;         \
        case 32: { constexpr int N1 = 8, N2 = 4; __VA_ARGS__; } break;         \
        case 64: { constexpr int N1 = 8, N2 = 8; __VA_ARGS__; } break;         \
        case 128: { constexpr int N1 = 16, N2 = 8; __VA_ARGS__; } break;       \
        case 256: { constexpr int N1 = 16, N2 = 16; __VA_ARGS__; } break;      \
        case 512: { constexpr int N1 = 32, N2 = 16; __VA_ARGS__; } break;      \
        case 1024: { constexpr int N1 = 32, N2 = 32; __VA_ARGS__; } break;     \
        case 2048: { constexpr int N1 = 64, N2 = 32; __VA_ARGS__; } break;     \
        case 4096: { constexpr int N1 = 64, N2 = 64; __VA_ARGS__; } break;     \
        case 8192: { constexpr int N1 = 128, N2 = 64; __VA_ARGS__; } break;    \
        case 16384: { constexpr int N1 = 128, N2 = 128; __VA_ARGS__; } break;  \
        default:                                                        \
            sb::set_error("row FFT length %d unsupported (8..16384)", (int)(N)); \
            return SB_ERR_UNSUPPORTED;                                  \
    }

// column length R = R1 * R2, both in [2, 256]
#define SB_TILE_DISPATCH(L, ...)                                        \
    switch (L) {                                                        \
        case 2: { constexpr int LL = 2; __VA_ARGS__; } break;                  \
        case 4: { constexpr int LL = 4; __VA_ARGS__; } break;                  \
        case 8: { constexpr int LL = 8; __VA_ARGS__; } break;                  \
        case 16: { constexpr int LL = 16; __VA_ARGS__; } break;                \
        case 32: { constexpr int LL = 32; __VA_ARGS__; } break;                \
        case 64: { constexpr int LL = 64; __VA_ARGS__; } break;                \
        case 128: { constexpr int LL = 128; __VA_ARGS__; } break;              \
        case 256: { constexpr int LL = 256; __VA_ARGS__; } break;              \
        default:                                                        \
            sb::set_error("tile FFT length %d unsupported", (int)(L));  \
            return SB_ERR_UNSUPPORTED;                                  \
    }

inline void split_len(int R, int* R1, int* R2) {
    int p = 0;
    while ((1 << p) < R) ++p;
    *R1 = 1 << ((p + 1) / 2);
    *R2 = R / *R1;
}
inline bool is_pow2(long v) { return v > 0 && (v & (v - 1)) == 0; }
inline int next_pow2(long v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// generic strided-axis transform of a [R][pitch] complex array with plain-load
// tile passes, functor on the final store: storeB(y=k1, k=k2, c, v)
template <typename T, int DIR, class LoadA, class StoreB>
static inline int cols_generic(LoadA la, cx<T>* tmp, long pitch, int R, int ncols,
                        StoreB sb, cudaStream_t st) {
    using C = cx<T>;
    constexpr int W = 256 / sizeof(C);
    int R1, R2;
    split_len(R, &R1, &R2);
    const C* wR = twiddle_table<T>(R, DIR, st);
    if (!wR) return SB_ERR_NOMEM;
    TwiddleAStore<C> sa{tmp, pitch, R2, R, wR};
    int rc = SB_OK;
    SB_TILE_DISPATCH(R1, rc = (launch_tile_fft<T, LL, W, DIR>(la, sa, ncols, R2, st)));
    if (rc) return rc;
    BlockBLoad<C> lb{tmp, pitch, R2};
    SB_TILE_DISPATCH(R2, rc = (launch_tile_fft<T, LL, W, DIR>(lb, sb, ncols, R1, st)));
    return rc;
}

// chirp-z (Bluestein) tables of length N, padded length M (8 <= M <= 65536): the chirp
// w[N] and the transformed kernel B = FFT_M(b); scratch holds 2 M points (dynspec.cu)
int bluestein_tables(int N, int M, float2* w, float2* B, float2* scratch, cudaStream_t st);

// Row half of a chirp-z transform: every one of nrows rows read by ld (its chirp w is set
// here) is chirped, transformed at length MT, multiplied by BT, inverse transformed into
// buf [nrows][MT] and back; os(row, k, v) receives bin k < MT of the unnormalised inverse,
// before the output chirp w[k] and the 1 / MT.
template <class RowLoad, class Store>
static inline int chirp_rows(RowLoad ld, Store os, float2* buf, int MT, long nrows,
                             const float2* wT, const float2* BT, cudaStream_t st) {
    ld.w = wT;
    MulVecRowStore ms{buf, MT, BT};
    int rc = SB_OK;
    SB_ROW_DISPATCH(MT, rc = (launch_row_c2c<float, N1, N2, -1>(ld, ms, nrows, st)));
    if (rc) return rc;
    PitchRowLoad<float2> pl{buf, MT};
    SB_ROW_DISPATCH(MT, rc = (launch_row_c2c<float, N1, N2, +1>(pl, os, nrows, st)));
    return rc;
}

// Forward chirp-z transform of an n0 x n1 plane whose first `live` rows are read by
// ld (ChirpRowLoad or ChirpRowLoadC; its chirp w is set here) and whose other rows
// are zero.  The final column pass stores through mk(R1, wF, MF) (wF: chirp of the
// column axis, MF: its padded length); columns >= ncols are never stored.  `what`
// begins the error message of a size outside the limits.
template <class RowLoad, class MakeStore>
static inline int chirp_fft2(RowLoad ld, int n0, int n1, int live, int ncols, MakeStore mk,
                             const char* what, cudaStream_t st) {
    const int MT = next_pow2(2L * n1 - 1), MF = next_pow2(2L * n0 - 1);
    // M >= 8 on both axes: bluestein_tables transforms the kernel with a row FFT (>= 8 points)
    if (MT < 8 || MT > 16384 || MF < 8 || MF > 65536) {
        set_error("%s %d x %d outside 3..32768 x 3..8192 (rows 3..32768, cols 3..8192)", what,
                  n0, n1);
        return SB_ERR_UNSUPPORTED;
    }
    const long pt = ((long)n1 + 15) & ~15L;
    float2* tabs = (float2*)workspace(WS_PLANE3, (size_t)(n1 + 3L * MT + n0 + 3L * MF + 64) * sizeof(float2));
    float2* R1buf = (float2*)workspace(WS_PLANE0, (size_t)live * MT * sizeof(float2));
    float2* Ybuf = (float2*)workspace(WS_PLANE1, (size_t)live * pt * sizeof(float2));
    float2* C0 = (float2*)workspace(WS_PLANE2, (size_t)MF * pt * sizeof(float2));
    float2* C1 = (float2*)workspace(WS_PLANE4, (size_t)MF * pt * sizeof(float2));
    if (!tabs || !R1buf || !Ybuf || !C0 || !C1) return SB_ERR_NOMEM;
    float2* wT = tabs;
    float2* BT = wT + n1;
    float2* wF = BT + MT;
    float2* BF = wF + n0;
    float2* scratch = BF + MF;      // 2*max(MT, MF)
    int rc = bluestein_tables(n1, MT, wT, BT, scratch, st);
    if (rc) return rc;
    rc = bluestein_tables(n0, MF, wF, BF, scratch, st);
    if (rc) return rc;
    // rows: chirp, FFT, multiply, inverse FFT, chirp
    rc = chirp_rows(ld, ChirpOutRowStore{Ybuf, pt, wT, n1, 1.0f / (float)MT}, R1buf, MT, live,
                    wT, BT, st);
    if (rc) return rc;
    // columns
    int R1, R2;
    split_len(MF, &R1, &R2);
    ChirpColALoad la{Ybuf, pt, R2, live, wF};
    MulVecColStore mc{C1, pt, R1, BF};
    rc = cols_generic<float, -1>(la, C0, pt, MF, ncols, mc, st);
    if (rc) return rc;
    StrideALoad<float2> pa{C1, pt, R2};
    return cols_generic<float, +1>(pa, C0, pt, MF, ncols, mk(R1, wF, MF), st);
}

}  // namespace sb
