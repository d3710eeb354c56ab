// CPU run of the device code of sb::chisq_sweep up to the inverse FFT, under the
// SIMT emulator: thth_prep_kernel and thth_build_kernel<0, 4> (csrc/thth.cu),
// herm_eigvec_batch_kernel, rev_scatter_rank1_kernel and rev_finalise_batch_kernel
// (csrc/retrieval.cu), sources unchanged, launch geometry as in sb::chisq_sweep.
// The transforms are not emulated.  TEST INFRASTRUCTURE (tests/test_chisq_cpu.py).
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

// recov: float2 [neta][ntau][nfd] (the finalised bin means), cnt: int [neta][ntau][nfd],
// V: float2 [neta][ld] (ld = n_th rounded up to 32)
extern "C" int emu_chisq_stages(const float* cs, long long ntau, long long nfd, double tau0,
                                double dtau, double tau_absmax, double fd0, double dfd,
                                double fd_half, const double* th, int n_th, const double* etas,
                                int neta, const double* th_red, double dtau_bin, double dfd_bin,
                                double tol, int max_iter, int* nred, int* status, double* w,
                                int* iters, float* V_out, float* recov, int* cnt) {
    using namespace sb;
    ThthGeom g;
    g.cs = reinterpret_cast<const float2*>(cs);
    g.ntau = ntau; g.nfd = nfd;
    g.tau0 = tau0; g.dtau = dtau; g.half_dtau = dtau / 2; g.tau_absmax = tau_absmax;
    g.fd0 = fd0; g.dfd = dfd; g.half_dfd = dfd / 2; g.fd_half = fd_half;
    g.inv_dtau = 1.0 / dtau; g.inv_dfd = 1.0 / dfd;
    g.th = th; g.n = n_th; g.coherent = 1; g.cs_half = 0; g.cs_valid_cols = 0; g.cs_bound = nullptr;
    g.cs_pitch = nfd;
    const int ld = (n_th + 31) / 32 * 32;
    std::vector<int> idx((size_t)neta * ld, 0);
    std::vector<float2> M((size_t)neta * ld * ld);
    std::memset(M.data(), 0xff, M.size() * sizeof(float2));          // NaN junk, like a fresh slab
    for (int e = 0; e < neta; ++e) status[e] = 0;
    for (int e = 0; e < neta; ++e)
        emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)neta, 1, 1},
                       [&]() { thth_prep_kernel(g, etas, neta, ld, idx.data(), nred); });
    const int T = ld / 32, npairs = T * (T + 1) / 2;
    const unsigned gx = (unsigned)((neta + SB_BUILD_EB - 1) / SB_BUILD_EB);
    for (unsigned bx = 0; bx < gx; ++bx)
        for (unsigned by = 0; by < (unsigned)npairs; ++by)
            emu::run_block(emu::Dim3{32, 8, 1}, emu::Dim3{bx, by, 0},
                           emu::Dim3{gx, (unsigned)npairs, 1}, [&]() {
                               thth_build_kernel<0, 4, unsigned>(g, etas, 0, neta, ld, idx.data(),
                                                                 nred, M.data(), nullptr, nullptr,
                                                                 0.f);
                           });
    std::vector<float2> Q((size_t)neta * (max_iter + 1) * ld);
    float2* V = reinterpret_cast<float2*>(V_out);
    for (int e = 0; e < neta; ++e)
        emu::run_block(emu::Dim3{(unsigned)EV_THREADS, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)neta, 1, 1}, [&]() {
                           herm_eigvec_batch_kernel(M.data(), ld, nred, 0, Q.data(), max_iter, tol,
                                                    w, V, status, iters);
                       });
    const size_t bins = (size_t)ntau * nfd;
    std::memset(recov, 0, (size_t)neta * bins * sizeof(float2));
    std::memset(cnt, 0, (size_t)neta * bins * sizeof(int));
    const RevGeom rg{nullptr, 0, 0.0, tau0, dtau_bin, fd0, dfd_bin, (int)ntau, (int)nfd};
    float2* acc = reinterpret_cast<float2*>(recov);
    for (int e = 0; e < neta; ++e)
        for (unsigned bx = 0; bx < 8; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)e, 0},
                           emu::Dim3{8, (unsigned)neta, 1}, [&]() {
                               rev_scatter_rank1_kernel(rg, th_red, n_th, etas, 0, nred, status, w,
                                                        V, ld, acc, cnt);
                           });
    for (int e = 0; e < neta; ++e)
        for (unsigned bx = 0; bx < 8; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)e, 0},
                           emu::Dim3{8, (unsigned)neta, 1},
                           [&]() { rev_finalise_batch_kernel(rg, acc, cnt); });
    return 0;
}
