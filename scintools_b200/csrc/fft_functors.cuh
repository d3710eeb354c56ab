// Load / store functors of the FFT passes, shared by every transform driver
// (dynspec.cu, retrieval.cu, sim.cu, slow_ft.cu), and the chirp-z (Bluestein) tables.
// Row kernels: load(row, n), store(row, k, v).  Tile kernels (four-step column
// pass): load(y, i, c), store(y, k, c, v).  Barrier-free, so tests/host_emu can
// compile this header for the CPU (SB_HOST_EMU) and check the index /
// conjugation / scaling logic around a reference DFT.
#pragma once
#ifndef SB_HOST_EMU
#include "fft_core.cuh"
#endif

namespace sb {

// ------------------------------------------------------------ generic passes
template <typename C> struct PitchRowLoad {
    const C* in;
    long pitch;
    __device__ __forceinline__ C operator()(long row, int n) const { return in[row * pitch + n]; }
};
template <typename C> struct PlainRowStore {
    C* out;
    long pitch;
    __device__ __forceinline__ void operator()(long row, int k, C v) const {
        out[row * pitch + k] = v;
    }
};
template <typename C> struct StrideALoad {   // y = r2, i = r1
    const C* in;
    long pitch;
    int R2;
    __device__ __forceinline__ C operator()(int y, int i, int c) const {
        return in[(size_t)(i * R2 + y) * pitch + c];
    }
};
template <typename C> struct ZeroPadALoad {  // StrideALoad, zero beyond the live rows
    const C* in;
    long pitch;
    int R2, live;
    __device__ __forceinline__ C operator()(int y, int i, int c) const {
        const int row = i * R2 + y;
        return row < live ? in[(size_t)row * pitch + c] : C{0, 0};
    }
};
template <typename C> struct TwiddleAStore { // times W_R^(dir y k), row k*R2 + y
    C* out;
    long pitch;
    int R2, R;
    const C* wR;
    __device__ __forceinline__ void operator()(int y, int k, int c, C v) const {
        out[(size_t)(k * R2 + y) * pitch + c] = cmul(v, wR[(y * k) & (R - 1)]);
    }
};
template <typename C> struct BlockBLoad {    // y = k1, i = r2
    const C* in;
    long pitch;
    int R2;
    __device__ __forceinline__ C operator()(int y, int i, int c) const {
        return in[(size_t)(y * R2 + i) * pitch + c];
    }
};
template <typename C> struct NaturalBStore { // out[y + S k][c] = v: natural order of the output
    C* out;
    long pitch;
    int S;
    __device__ __forceinline__ void operator()(int y, int k, int c, C v) const {
        out[(size_t)(y + S * k) * pitch + c] = v;
    }
};

// ------------------------------------------ secondary spectrum and ACF (dynspec.cu)
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

// ------------------------------------------------------------------ chirp-z
static __global__ void chirp_fill_kernel(float2* w, float2* b, int N, int M) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= M) return;
    // b[m] = conj(w[|m|]) for -N < m < N (wrapped mod M), else 0
    const int m = n < N ? n : (M - n < N ? M - n : -1);
    float2 bv = make_float2(0.f, 0.f);
    if (m >= 0) {
        const long long q = ((long long)m * m) % (2LL * N);
        double s, c;
        sincospi((double)q / (double)N, &s, &c);
        bv = make_float2((float)c, (float)s);            // conj(w) = exp(+i pi m^2/N)
        if (n < N) w[n] = make_float2((float)c, (float)-s);
    }
    b[n] = bv;
}

struct VecLoad {     // single row / column loader
    const float2* v;
    __device__ __forceinline__ float2 operator()(long, int n) const { return v[n]; }
};
struct VecStore {
    float2* v;
    __device__ __forceinline__ void operator()(long, int k, float2 x) const { v[k] = x; }
};
struct ColVecLoad {  // y = r2, i = r1 over a [M][1] array
    const float2* v;
    int R2;
    __device__ __forceinline__ float2 operator()(int y, int i, int) const { return v[i * R2 + y]; }
};
struct ColVecStore {
    float2* v;
    int R1;
    __device__ __forceinline__ void operator()(int y, int k, int, float2 x) const { v[y + R1 * k] = x; }
};

struct ChirpRowLoad {    // a[n] = (x[f][n] - sub) * w[n], zero beyond the live samples
    const float* dyn;
    int nt;
    const float2* w;
    const double* stats;  // non-null: subtract stats[4] (device mean)
    float sub;
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        if (n >= nt) return make_float2(0.f, 0.f);
        const float x = dyn[(size_t)row * nt + n] - (stats ? (float)stats[4] : sub);
        const float2 c = w[n];
        return make_float2(x * c.x, x * c.y);
    }
};
struct MulVecRowStore {  // out[row][k] = v * B[k]
    float2* out;
    long pitch;
    const float2* B;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        out[row * pitch + k] = cmul(v, B[k]);
    }
};
struct ChirpOutRowStore {  // Y[row][k] = v * w[k] / M, k < N
    float2* out;
    long pitch;
    const float2* w;
    int N;
    float scale;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        if (k < N) {
            const float2 r = cmul(v, w[k]);
            out[row * pitch + k] = make_float2(r.x * scale, r.y * scale);
        }
    }
};
struct ChirpColALoad {   // y = r2, i = r1 : Y[row][c] * wF[row], zero beyond live rows
    const float2* Y;
    long pitch;
    int R2, live;
    const float2* w;
    __device__ __forceinline__ float2 operator()(int y, int i, int c) const {
        const int row = i * R2 + y;
        return row < live ? cmul(Y[(size_t)row * pitch + c], w[row]) : make_float2(0.f, 0.f);
    }
};
struct MulVecColStore {  // out[k][c] = v * B[k], k = k1 + R1 k2
    float2* out;
    long pitch;
    int R1;
    const float2* B;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kk = y + R1 * k;
        out[(size_t)kk * pitch + c] = cmul(v, B[kk]);
    }
};
struct ChirpCsStore {    // CS[(k + N/2) % N][(c + NT/2) % NT] = v * wF[k] / M (+dc), masks
    float2* CS;
    int NF, NT, R1;
    const float2* w;
    float scale;
    const unsigned char* rowmask;
    float dc;
    const double* dc_stats;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kf = y + R1 * k;
        if (kf >= NF) return;
        float2 r = cmul(v, w[kf]);
        r.x *= scale;
        r.y *= scale;
        if (kf == 0 && c == 0)
            r.x += dc_stats ? (float)(dc_stats[4] * (double)NF * (double)NT) : dc;
        const int rs = (kf + NF / 2) % NF, cs = (c + NT / 2) % NT;
        if (rowmask && rowmask[rs]) r = make_float2(0.f, 0.f);
        CS[(size_t)rs * NT + cs] = r;
    }
};

struct ChirpRowLoadC {   // a[n] = conj(x[r'][n']) * w[n] with the ifftshift folded in
    const float2* in;
    int n0, n1, centred, keep;     // keep != 0: transform conj(in), i.e. no negation here
    const float2* w;
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        if (n >= n1) return make_float2(0.f, 0.f);
        const int r = centred ? (int)((row + n0 / 2) % n0) : (int)row;
        const int c = centred ? (n + n1 / 2) % n1 : n;
        float2 v = in[(size_t)r * n1 + c];
        if (!keep) v.y = -v.y;
        return cmul(v, w[n]);
    }
};

// ------------------------------------------- inverse 2-D transforms (retrieval.cu)
// The last column pass of the power-of-two and of the chirp-z inverse each reach a base
// store, base(row, c, v) with v element (row, c) of the unnormalised inverse, through one
// adapter that forms the output row, drops what lies outside rows x cols and, on the
// chirp-z path, applies the column chirp.  Base stores: CropStore, ResidualSink.
template <class Base> struct RadixStore {   // base(k, c, v), k = k1 + R1 k2
    int R1, rows, cols;
    Base base;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int row = y + R1 * k;
        if (row >= rows || c >= cols) return;
        base(row, c, v);
    }
};
template <class Base> struct ChirpStore {   // base(k, c, conj(v * wF[k])), k = k1 + R1 k2
    int R1, rows, cols;
    const float2* w;
    Base base;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int kf = y + R1 * k;
        if (kf >= rows || c >= cols) return;
        const float2 r = cmul(v, w[kf]);
        base(kf, c, make_float2(r.x, -r.y));
    }
};
struct CropStore {        // out[row][c] = v * scale, or its real part
    float2* outc;
    float* outr;
    int pitch;
    float scale;
    __device__ __forceinline__ void operator()(int row, int c, float2 v) const {
        const size_t o = (size_t)row * pitch + c;
        if (outr) outr[o] = v.x * scale;
        else outc[o] = make_float2(v.x * scale, v.y * scale);
    }
};

// ------------------------------------------- frequency-scaled chirp-z (slow_ft.cu)
// Each column c (channel) has its own chirp rate s[c] / nt, not a multiple of 1 / nt, so
// the chirps are generated here instead of read from tables.
// exp(i pi s q / n) for an integer |q| < 2^31 (exact in float64): the phase is reduced mod
// 2 in float64 (x - 2 floor(x / 2) is exact) before sincospi; at |x| ~ 4e4 a float32
// phase would be off by ~0.03 rad.  A non-finite s gives NaN.
__device__ __forceinline__ float2 chirp_pi(double s, long long q, int n) {
    const double x = s * (double)q / (double)n;
    double sn, cs;
    sincospi(x - 2.0 * floor(0.5 * x), &sn, &cs);
    return make_float2((float)cs, (float)sn);
}
struct SlowKernelColLoad {   // y = r2, i = r1: b_c[n] = exp(+i pi s[c] n^2 / nt), |n| < nt, mod M
    int R2, M, nt;
    const double* s;
    __device__ __forceinline__ float2 operator()(int y, int i, int c) const {
        const int n = i * R2 + y;
        const int m = n < nt ? n : (M - n < nt ? M - n : -1);
        if (m < 0) return make_float2(0.f, 0.f);
        return chirp_pi(s[c], (long long)m * m, nt);
    }
};
struct SlowChirpColLoad {    // y = r2, i = r1: x[t][c] exp(-i pi s[c] (t^2 - 2 (nt/2) t) / nt)
    const float* x;          // [nt][nf]; rows t >= nt are the zero padding
    int nf, nt, R2;
    const double* s;
    __device__ __forceinline__ float2 operator()(int y, int i, int c) const {
        const int t = i * R2 + y;
        if (t >= nt) return make_float2(0.f, 0.f);
        const float v = x[(size_t)t * nf + c];
        const float2 w = chirp_pi(-s[c], (long long)t * (t - 2 * (nt / 2)), nt);
        return make_float2(v * w.x, v * w.y);
    }
};
struct MulPlaneColStore {    // B[k][c] = v * B[k][c], k = k1 + R1 k2 (in place: one thread per element)
    float2* B;
    long pitch;
    int R1;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const size_t o = (size_t)(y + R1 * k) * pitch + c;
        B[o] = cmul(v, B[o]);
    }
};
struct SlowChirpOutColStore {   // out[m][c] = v exp(-i pi s[c] m^2 / nt) * scale, m < nt
    float2* out;
    int nf, nt, R1;
    const double* s;
    float scale;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        const int m = y + R1 * k;
        if (m >= nt) return;
        const float2 r = cmul(v, chirp_pi(-s[c], (long long)m * m, nt));
        out[(size_t)m * nf + c] = make_float2(r.x * scale, r.y * scale);
    }
};
struct ShiftRowStore {       // out[row][(k + N/2) % N] = v: the fftshift of a row
    float2* out;
    int N;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        out[row * N + (k + N / 2) % N] = v;
    }
};
struct ChirpShiftRowStore {  // out[row][(k + N/2) % N] = v * w[k] * scale, k < N
    float2* out;
    int N;
    const float2* w;
    float scale;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        if (k < N) {
            const float2 r = cmul(v, w[k]);
            out[row * N + (k + N / 2) % N] = make_float2(r.x * scale, r.y * scale);
        }
    }
};

}  // namespace sb
