// CPU run of the device code of the scintillation-scale fits (csrc/scintfit.cu, sources
// unchanged) under the SIMT emulator: the init, eval, solve and count kernels, launched in
// the order of sb::scint_fit.  The blocks of a launch run one after another in block order.
// TEST INFRASTRUCTURE (tests/test_scint_params_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

struct int2 { int x, y; };
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }

// the public struct of include/scint_b200.h (the header itself needs the CUDA runtime)
#include <cstdint>
typedef struct sb_scint_fit {
    const double* acf;
    const double* aux;
    int64_t pitch;
    double s0, s1, c;
    double p0[5];
    int32_t r0, c0, r1, c1, n0, n1;
    int32_t shf, sht, pf, pt, zf, zt;
    int32_t vary, bounded, weighted, max_nfev;
} sb_scint_fit;

#include "../../scintools_b200/csrc/scintfit.cu"

namespace {
using namespace sb;

void grid(unsigned G, int threads, const std::function<void()>& body) {
    for (unsigned x = 0; x < G; ++x)
        emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, 0, 0},
                       emu::Dim3{G, 1, 1}, body);
}

template <class M>
int run(const sb_scint_fit* fits, int nfit, double* out, int* info) {
    std::vector<int2> table, range(nfit);
    int max_nfev = 0;
    for (int i = 0; i < nfit; ++i) {
        const long long n = M::npoints(fits[i]);
        const int nc = (int)((n + SF_CHUNK - 1) / SF_CHUNK);
        range[i] = make_int2((int)table.size(), nc);
        for (int c = 0; c < nc; ++c) table.push_back(make_int2(i, c * SF_CHUNK));
        max_nfev = fits[i].max_nfev > max_nfev ? fits[i].max_nfev : max_nfev;
    }
    const unsigned nch = (unsigned)table.size();
    std::vector<FitState> st(nfit);
    std::vector<double> part((size_t)nch * SF_NPART);
    int done = 0;
    const unsigned gs = (unsigned)((nfit + 127) / 128);
    grid(gs, 128, [&]() { sf_init_kernel(fits, nfit, st.data()); });
    for (int it = 0; it < max_nfev && done < nfit;) {
        const int stop = it + SF_CHECK < max_nfev ? it + SF_CHECK : max_nfev;
        for (; it < stop; ++it) {
            grid(nch, SF_THREADS, [&]() { sf_eval_kernel<M>(fits, table.data(), st.data(), part.data()); });
            grid(gs, 128, [&]() {
                sf_solve_kernel<M>(fits, range.data(), nfit, part.data(), st.data(), out, info);
            });
        }
        grid(1, 1024, [&]() { sf_count_kernel(st.data(), nfit, &done); });
    }
    return 0;
}
}  // namespace

extern "C" int emu_scint_fit(int kind, const sb_scint_fit* fits, int nfit, double* out, int* info) {
    return kind == 1 ? run<Model1D>(fits, nfit, out, info) : run<Model2D>(fits, nfit, out, info);
}
