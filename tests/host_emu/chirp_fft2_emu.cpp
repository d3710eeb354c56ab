// CPU emulation of the any-size (chirp-z) 2-D FFT driver of csrc/fft_kernels.cuh
// (chirp_fft2) and its two uses, the inverse of retrieval.cu (ifft2_chirp) and the
// conjugate spectrum of conj_spectrum: the chirp tables and every load / store
// functor come from csrc/fft_functors.cuh unchanged; the power-of-two FFT kernels between them
// (verified on the GPU by the conjugate-spectrum tests) are replaced by a plain
// DFT, and the pass order / buffers / scales mirror the driver.  TEST INFRASTRUCTURE.
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
static void tables(int N, int M, std::vector<float2>& w, std::vector<float2>& B) {
    w.assign(N, make_float2(0, 0));
    B.assign(M, make_float2(0, 0));
    blockDim = {256, 1, 1};
    for (unsigned b = 0; b < (unsigned)((M + 255) / 256); ++b)
        for (unsigned t = 0; t < 256; ++t) {
            blockIdx = {b, 0, 0};
            threadIdx = {t, 0, 0};
            sb::chirp_fill_kernel(w.data(), B.data(), N, M);
        }
    dft(B, -1);
}

// chirp_fft2: ld reads the first `live` of n0 rows, mk(R1, wF, MF) makes the final store
template <class RowLoad, class MakeStore>
static void chirp_fft2(RowLoad ld, int n0, int n1, int live, int ncols, MakeStore mk) {
    using namespace sb;
    const int MT = next_pow2(2L * n1 - 1), MF = next_pow2(2L * n0 - 1);
    const long pt = ((long)n1 + 15) & ~15L;
    std::vector<float2> wT, BT, wF, BF;
    tables(n1, MT, wT, BT);
    tables(n0, MF, wF, BF);
    std::vector<float2> R1buf((size_t)live * MT), Ybuf((size_t)live * pt), C1((size_t)MF * pt);
    ld.w = wT.data();
    MulVecRowStore ms{R1buf.data(), MT, BT.data()};
    PitchRowLoad<float2> pl{R1buf.data(), MT};
    ChirpOutRowStore os{Ybuf.data(), pt, wT.data(), n1, 1.0f / (float)MT};
    for (int row = 0; row < live; ++row) {
        std::vector<float2> a(MT);
        for (int n = 0; n < MT; ++n) a[n] = ld(row, n);
        dft(a, -1);
        for (int k = 0; k < MT; ++k) ms(row, k, a[k]);
        for (int n = 0; n < MT; ++n) a[n] = pl(row, n);
        dft(a, +1);
        for (int k = 0; k < MT; ++k) os(row, k, a[k]);
    }
    int R1 = 1;
    while (R1 * R1 < MF) R1 <<= 1;
    const int R2 = MF / R1;
    ChirpColALoad la{Ybuf.data(), pt, R2, live, wF.data()};
    MulVecColStore mc{C1.data(), pt, R1, BF.data()};
    StrideALoad<float2> pa{C1.data(), pt, R2};
    auto st = mk(R1, (const float2*)wF.data(), MF);
    for (int c = 0; c < ncols; ++c) {
        std::vector<float2> x(MF);
        for (int row = 0; row < MF; ++row) x[row] = la(row % R2, row / R2, c);
        dft(x, -1);
        for (int kk = 0; kk < MF; ++kk) mc(kk % R1, kk / R1, c, x[kk]);
    }
    for (int c = 0; c < ncols; ++c) {
        std::vector<float2> x(MF);
        for (int row = 0; row < MF; ++row) x[row] = pa(row % R2, row / R2, c);
        dft(x, +1);
        for (int kk = 0; kk < MF; ++kk) st(kk % R1, kk / R1, c, x[kk]);
    }
}

extern "C" int emu_ifft2_any(const float* in_, int n0, int n1, int centred, int crop0, int crop1,
                             double scale, int real_only, int conj_in, float* out) {
    using namespace sb;
    const float2* in = reinterpret_cast<const float2*>(in_);
    if (crop0 <= 0 || crop0 > n0) crop0 = n0;
    if (crop1 <= 0 || crop1 > n1) crop1 = n1;
    chirp_fft2(ChirpRowLoadC{in, n0, n1, centred, conj_in, nullptr}, n0, n1, n0, crop1,
               [&](int R1, const float2* wF, int MF) {
                   const double den = (double)MF * (double)n0 * (double)n1;
                   const CropStore base{real_only ? nullptr : reinterpret_cast<float2*>(out),
                                        real_only ? out : nullptr, crop1, (float)(scale / den)};
                   return ChirpStore<CropStore>{R1, crop0, crop1, wF, base};
               });
    return 0;
}

// conjugate spectrum of dyn [nf][nt] padded with pad_value to NF x NT (fftshifted,
// full plane, rows with rowmask[shifted row] zeroed)
extern "C" int emu_cs_any(const float* dyn, int nf, int nt, int NF, int NT, float pad_value,
                          const unsigned char* rowmask, float* out) {
    using namespace sb;
    float2* CS = reinterpret_cast<float2*>(out);
    chirp_fft2(ChirpRowLoad{dyn, nt, nullptr, nullptr, pad_value}, NF, NT, nf, NT,
               [&](int R1, const float2* wF, int MF) {
                   return ChirpCsStore{CS, NF, NT, R1, wF, 1.0f / (float)MF, rowmask,
                                       pad_value * (float)NF * (float)NT, nullptr};
               });
    return 0;
}
