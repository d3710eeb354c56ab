// CPU run of the device code of sb::vlbi_retrieval around the eigenpair, under the SIMT
// emulator: thth_prep_kernel (csrc/thth.cu), vlbi_composite_kernel, vlbi_scatter_kernel and
// vlbi_finalise_kernel (csrc/retrieval.cu), sources unchanged, launch shapes as in
// sb::vlbi_retrieval (smaller grids; every kernel strides over its work).  The eigenpair
// (w, V) is an input, so the scatter is checked on exactly the vector the oracle uses.
// The transforms are not emulated.  TEST INFRASTRUCTURE (tests/test_vlbi_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include <float.h>
#include <limits.h>

#include <type_traits>

namespace sb {
alignas(128) unsigned char smem_raw[256 * 1024];
}
#include "../../scintools_b200/csrc/thth.cu"
#include "../../scintools_b200/csrc/retrieval.cu"

// cs: n_dish (n_dish + 1) / 2 pointers to float2 [ntau][nfd]; A: float2 [N][N] with
// N = n_dish * nred (room for n_dish * n_th); V: float2 [n_dish * nred]; recov: float2
// [n_dish][ntau][nfd] (finalised bin means); cnt: int [ntau][nfd]
extern "C" int emu_vlbi_stages(const float* const* cs, int n_dish, long long ntau, long long nfd,
                               double tau0, double dtau, double tau_absmax, double fd0,
                               double dfd, double fd_half, const double* th, int n_th, double eta,
                               const double* th_red, double dtau_bin, double dfd_bin,
                               const float* V, double w, int* nred_out, float* A_out,
                               float* recov, int* cnt) {
    using namespace sb;
    ThthGeom g;
    g.cs = nullptr;
    g.ntau = ntau; g.nfd = nfd;
    g.tau0 = tau0; g.dtau = dtau; g.half_dtau = dtau / 2; g.tau_absmax = tau_absmax;
    g.fd0 = fd0; g.dfd = dfd; g.half_dfd = dfd / 2; g.fd_half = fd_half;
    g.inv_dtau = 1.0 / dtau; g.inv_dfd = 1.0 / dfd;
    g.th = th; g.n = n_th; g.coherent = 1; g.cs_half = 0; g.cs_valid_cols = 0; g.cs_bound = nullptr;
    g.cs_pitch = nfd;
    std::vector<int> idx(n_th, 0);
    int nred = 0;
    emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{0, 0, 0}, emu::Dim3{1, 1, 1},
                   [&]() { thth_prep_kernel(g, &eta, 1, n_th, idx.data(), &nred); });
    *nred_out = nred;
    const int n = nred;
    const long N = (long)n_dish * n;
    const float2* const* csp = reinterpret_cast<const float2* const*>(cs);
    float2* A = reinterpret_cast<float2*>(A_out);
    std::memset(A, 0xff, (size_t)N * N * sizeof(float2));        // NaN junk: every element is written
    for (unsigned b = 0; b < 16; ++b)
        emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{b, 0, 0}, emu::Dim3{16, 1, 1}, [&]() {
            vlbi_composite_kernel(g, &eta, csp, n_dish, idx.data(), n, A);
        });
    const int info[3] = {1, 0, n};
    const size_t bins = (size_t)ntau * nfd;
    std::memset(recov, 0, (size_t)n_dish * bins * sizeof(float2));
    std::memset(cnt, 0, bins * sizeof(int));
    const RevGeom rg{th_red, n, eta, tau0, dtau_bin, fd0, dfd_bin, (int)ntau, (int)nfd};
    float2* acc = reinterpret_cast<float2*>(recov);
    for (int d = 0; d <= n_dish; ++d)
        for (unsigned bx = 0; bx < 8; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)d, 0},
                           emu::Dim3{8, (unsigned)n_dish + 1, 1}, [&]() {
                               vlbi_scatter_kernel(rg, n_dish, info, &w,
                                                   reinterpret_cast<const float2*>(V), acc, cnt);
                           });
    for (int d = 0; d < n_dish; ++d)
        for (unsigned bx = 0; bx < 8; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)d, 0},
                           emu::Dim3{8, (unsigned)n_dish, 1},
                           [&]() { vlbi_finalise_kernel(rg, acc, cnt); });
    return 0;
}
