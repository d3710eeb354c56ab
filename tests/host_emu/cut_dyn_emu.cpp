// CPU run of the batched tile transforms of Dynspec.cut_dyn (csrc/tiles.cuh, drivers
// sspec_tiles / acf_tiles in csrc/dynspec.cu) under the SIMT emulator (simt.h): the
// statistics kernels run as written (warp shuffles, atomics), and every tile load / store
// functor comes from csrc/tiles.cuh and csrc/fft_functors.cuh unchanged; the power-of-two
// FFT kernels between them (checked on the GPU by the single-spectrum tests) are replaced
// by a plain DFT, with the pass order, buffers and the column-to-tile layout of the drivers.
// Built and called by tests/test_cut_dyn_emu_cpu.py.  TEST INFRASTRUCTURE: it checks the
// tile index maps without a GPU; nothing in scintools_b200 loads it.
#define SB_HOST_EMU 1
#include "simt.h"

#include <complex>

// one fiber runs at a time: a plain read-modify-write is atomic here
static inline double atomicAdd(double* p, double v) { double o = *p; *p = o + v; return o; }

static inline void sincospi(double x, double* s, double* c) {
    *s = std::sin(M_PI * x);
    *c = std::cos(M_PI * x);
}
namespace sb {
template <typename C> static inline C cmul(C a, C b) {
    return C{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}
}  // namespace sb

#include "../../scintools_b200/csrc/common.cuh"
#include "../../scintools_b200/csrc/fft_functors.cuh"
#include "../../scintools_b200/csrc/tiles.cuh"

using cd = std::complex<double>;
static std::vector<cd> dft(const std::vector<cd>& v, int dir) {   // unnormalised
    const int M = (int)v.size();
    std::vector<cd> o(M);
    for (int k = 0; k < M; ++k) {
        cd s = 0;
        for (int n = 0; n < M; ++n)
            s += v[n] * std::polar(1.0, dir * 2.0 * M_PI * ((long long)k * n % M) / M);
        o[k] = s;
    }
    return o;
}
static float2 f2(cd z) { return make_float2((float)z.real(), (float)z.imag()); }
static int next_pow2(long v) { int p = 1; while (p < v) p <<= 1; return p; }
static long half_pitch(long NT) { return ((NT / 2 + 1) + 15) & ~15L; }
static int split_r1(int R) { int p = 0; while ((1 << p) < R) ++p; return 1 << ((p + 1) / 2); }

// tile_stats of dynspec.cu: 2 blocks of 64 threads, so items are spread over 4 warps
static std::vector<float2> stats(const float* dyn, int nt, int fnum, int tnum, int ntc, int tile0,
                                 int ntile, const float* wt, const float* wf, double swt,
                                 double swf, double acf_den) {
    std::vector<double> sums(4 * (size_t)ntile, 0.0);
    std::vector<float2> cst(ntile);
    int rpi = 4096 / tnum;
    rpi = rpi < 1 ? 1 : (rpi > fnum ? fnum : rpi);
    for (unsigned b = 0; b < 2; ++b)
        emu::run_block(emu::Dim3{64, 1, 1}, emu::Dim3{b, 0, 0}, emu::Dim3{2, 1, 1}, [&]() {
            sb::tile_stats_kernel(dyn, nt, fnum, tnum, ntc, tile0, ntile, rpi, wt, wf, sums.data());
        });
    const unsigned g = (unsigned)((ntile + 255) / 256);
    for (unsigned b = 0; b < g; ++b)
        emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{b, 0, 0}, emu::Dim3{g, 1, 1}, [&]() {
            sb::tile_stats_final_kernel(sums.data(), ntile, (double)fnum * tnum, swt, swf,
                                        wt != nullptr, acf_den, cst.data());
        });
    return cst;
}

// rows: real rows of length NT (row item r read by ld) -> half spectra through hs
template <class Load, class Store>
static void rows_r2c(const Load& ld, const Store& hs, long nrows, int NT) {
    const int N = NT / 2, live = ld.live(N);
    for (long r = 0; r < nrows; ++r) {
        std::vector<cd> x(NT, 0.0);
        for (int n = 0; n < live; ++n) {
            const float2 p = ld(r, n);
            x[2 * n] = p.x;
            x[2 * n + 1] = p.y;
        }
        const std::vector<cd> X = dft(x, -1);
        for (int k = 0; k <= N; ++k) hs(r, k, f2(X[k]));
    }
}

// group [tile0, tile0 + ntile) of the nfc x ntc tiles of dyn [*][nt]: sec [ntile][NF/2][NT],
// acf [ntile][2 fnum][2 tnum], as sspec_tiles / acf_tiles write them
extern "C" int emu_cut_dyn(const float* dyn, int nt, int fnum, int tnum, int ntc, int tile0,
                           int ntile, const float* wt, const float* wf, double swt, double swf,
                           float* sec, float* acf) {
    using namespace sb;
    {   // secondary spectra
        const int NF = 2 * next_pow2(fnum), NT = 2 * next_pow2(tnum), R1 = split_r1(NF);
        const long tp = half_pitch(NT), pitch = ntile * tp;
        std::vector<float2> H((size_t)fnum * pitch, make_float2(0.f, 0.f));
        const std::vector<float2> cst = stats(dyn, nt, fnum, tnum, ntc, tile0, ntile, wt, wf,
                                              swt, swf, 0.0);
        rows_r2c(TileRowLoad{dyn, nt, fnum, tnum, ntc, tile0, wt, wf, cst.data()},
                 TileHalfStore{H.data(), pitch, (int)tp, fnum}, (long)ntile * fnum, NT);
        const size_t plane = (size_t)(NF / 2) * NT;
        TileSspecStore ss{SspecStore{sec, NF, NT, R1, 1, 1, nullptr, nullptr, 0}, (int)tp,
                          NT / 2 + 1, plane};
        for (long c = 0; c < pitch; ++c) {
            std::vector<cd> x(NF, 0.0);
            for (int f = 0; f < fnum; ++f) x[f] = cd(H[f * pitch + c].x, H[f * pitch + c].y);
            const std::vector<cd> X = dft(x, -1);
            for (int kf = 0; kf < NF; ++kf) ss(kf % R1, kf / R1, (int)c, f2(X[kf]));
        }
    }
    {   // ACFs
        const int PF = next_pow2(2L * fnum), PT = next_pow2(2L * tnum);
        const long tp = half_pitch(PT), pitch = ntile * tp;
        std::vector<float2> H((size_t)fnum * pitch, make_float2(0.f, 0.f));
        std::vector<float2> Q((size_t)PF * pitch, make_float2(0.f, 0.f));
        const std::vector<float2> cst = stats(dyn, nt, fnum, tnum, ntc, tile0, ntile, nullptr,
                                              nullptr, 0.0, 0.0, (double)PF * PT);
        rows_r2c(TileRowLoad{dyn, nt, fnum, tnum, ntc, tile0, nullptr, nullptr, nullptr},
                 TileHalfStore{H.data(), pitch, (int)tp, fnum}, (long)ntile * fnum, PT);
        for (long c = 0; c < pitch; ++c) {     // acf_cols: forward, |.|^2, inverse
            std::vector<cd> x(PF, 0.0);
            for (int f = 0; f < fnum; ++f) x[f] = cd(H[f * pitch + c].x, H[f * pitch + c].y);
            std::vector<cd> X = dft(x, -1);
            for (auto& z : X) z = std::norm(z);
            const std::vector<cd> q = dft(X, +1);
            for (int n = 0; n < PF; ++n) Q[n * pitch + c] = f2(q[n]);
        }
        const int N = PT / 2;
        TileAcfRowLoad rl{AcfRowLoad{Q.data(), pitch, fnum, PF}, 2 * fnum, (int)tp};
        TileAcfRowStore rs{AcfRowStore{acf, tnum, PT, nullptr}, 2 * fnum,
                           (size_t)(2 * fnum) * (2 * tnum), cst.data()};
        for (long r = 0; r < 2L * ntile * fnum; ++r) {   // half spectrum -> real, unnormalised
            std::vector<cd> Y(PT);
            for (int k = 0; k <= N; ++k) {
                const float2 v = rl(r, k);
                Y[k] = cd(v.x, v.y);
                if (k > 0 && k < N) Y[PT - k] = std::conj(Y[k]);
            }
            const std::vector<cd> y = dft(Y, +1);
            for (int n = 0; n < N; ++n)
                rs(r, n, make_float2((float)y[2 * n].real(), (float)y[2 * n + 1].real()));
        }
    }
    return 0;
}
