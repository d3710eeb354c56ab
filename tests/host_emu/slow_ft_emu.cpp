// CPU emulation of the frequency-scaled Doppler transform of csrc/slow_ft.cu: the
// per-channel chirp functors, the in-place kernel multiply, the shifted row stores and
// the row chirp-z tables come from csrc/fft_functors.cuh unchanged; the power-of-two FFT
// passes between them (verified on the GPU) are replaced by a plain DFT, and the pass
// order / buffers / scales mirror the driver.  TEST INFRASTRUCTURE.
#define SB_HOST_EMU 1
#include <cmath>
#include <complex>
#include <cstddef>
#include <vector>

struct emu_uint3 { unsigned x, y, z; };
static emu_uint3 blockIdx, threadIdx, blockDim, gridDim;
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
#define __global__
#define __device__
#define __restrict__
#define __forceinline__ inline
static inline void sincospi(double x, double* s, double* c) {
    *s = std::sin(M_PI * x);
    *c = std::cos(M_PI * x);
}
namespace sb {
template <typename C> static inline C cmul(C a, C b) {
    return C{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}
}
#include "../../scintools_b200/csrc/fft_functors.cuh"

using cd = std::complex<double>;
static void dft(std::vector<float2>& v, int dir) {       // unnormalised, like the engine
    const int M = (int)v.size();
    std::vector<float2> o(M);
    for (int k = 0; k < M; ++k) {
        cd s = 0;
        for (int n = 0; n < M; ++n)
            s += cd(v[n].x, v[n].y) * std::polar(1.0, dir * 2.0 * M_PI * ((long long)k * n % M) / M);
        o[k] = make_float2((float)s.real(), (float)s.imag());
    }
    v = o;
}
static int next_pow2(long v) { int p = 1; while (p < v) p <<= 1; return p; }
static void split_len(int R, int* R1, int* R2) {
    int p = 0;
    while ((1 << p) < R) ++p;
    *R1 = 1 << ((p + 1) / 2);
    *R2 = R / *R1;
}
// one column transform of length M over ncols columns: load la(y = r2, i = r1, c) of row
// i R2 + y, store st(y = k1, k = k2, c) of bin k1 + R1 k2 (cols_generic's functor contract)
template <class L, class S>
static void cols(L la, S st, int M, int ncols, int dir) {
    int R1, R2;
    split_len(M, &R1, &R2);
    for (int c = 0; c < ncols; ++c) {
        std::vector<float2> v(M);
        for (int row = 0; row < M; ++row) v[row] = la(row % R2, row / R2, c);
        dft(v, dir);
        for (int kk = 0; kk < M; ++kk) st(kk % R1, kk / R1, c, v[kk]);
    }
}
template <class L, class S>
static void rows(L ld, S st, int N, int nrows, int dir) {
    for (int r = 0; r < nrows; ++r) {
        std::vector<float2> v(N);
        for (int n = 0; n < N; ++n) v[n] = ld(r, n);   // the whole row before any store
        dft(v, dir);
        for (int k = 0; k < N; ++k) st(r, k, v[k]);
    }
}

extern "C" int emu_slow_ft(const float* x, int nt, int nf, const double* s, float* out_) {
    using namespace sb;
    float2* out = reinterpret_cast<float2*>(out_);
    const int M = next_pow2(2L * nt - 1) < 8 ? 8 : next_pow2(2L * nt - 1);
    const long pt = ((long)nf + 15) & ~15L;
    int R1, R2;
    split_len(M, &R1, &R2);
    std::vector<float2> Bp((size_t)M * pt);
    cols(SlowKernelColLoad{R2, M, nt, s}, NaturalBStore<float2>{Bp.data(), pt, R1}, M, nf, -1);
    cols(SlowChirpColLoad{x, nf, nt, R2, s}, MulPlaneColStore{Bp.data(), pt, R1}, M, nf, -1);
    cols(StrideALoad<float2>{Bp.data(), pt, R2},
         SlowChirpOutColStore{out, nf, nt, R1, s, 1.0f / (float)M}, M, nf, +1);
    if (nf >= 8 && (nf & (nf - 1)) == 0) {
        rows(PitchRowLoad<float2>{out, nf}, ShiftRowStore{out, nf}, nf, nt, -1);
        return 0;
    }
    const int MT = next_pow2(2L * nf - 1) < 8 ? 8 : next_pow2(2L * nf - 1);
    std::vector<float2> wT(nf), BT(MT), buf((size_t)nt * MT);
    blockDim = {256, 1, 1};
    for (unsigned b = 0; b < (unsigned)((MT + 255) / 256); ++b)
        for (unsigned t = 0; t < 256; ++t) {
            blockIdx = {b, 0, 0};
            threadIdx = {t, 0, 0};
            chirp_fill_kernel(wT.data(), BT.data(), nf, MT);
        }
    dft(BT, -1);
    rows(ChirpRowLoadC{out, nt, nf, 0, 1, wT.data()}, MulVecRowStore{buf.data(), MT, BT.data()},
         MT, nt, -1);
    rows(PitchRowLoad<float2>{buf.data(), MT}, ChirpShiftRowStore{out, nf, wT.data(),
                                                                  1.0f / (float)MT}, MT, nt, +1);
    return 0;
}
