// CPU run of the curvature-sweep device code of csrc/thth.cu under the SIMT
// emulator: thth_prep_kernel (crop mask + compaction), thth_indexerr_kernel,
// thth_build_kernel (gather into the strict upper triangle) and the fp32
// thth_eig_kernel (SB_EIG_FP32=1), sources unchanged, launch geometry as in
// sb::eta_sweep.  mixed != 0: the default solver csrc/eig_half.cu (fp16 tensor-core
// iteration + fp32 Rayleigh quotient) instead of thth_eig_kernel; mixed == 2 forces
// its fp32 continuation (rtol_r = 0); -DSB_EB_SLOTS=3 exercises its fp32 restart.
// TEST INFRASTRUCTURE (tests/test_host_emulation.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include <float.h>
#include <limits.h>

namespace sb {
alignas(128) unsigned char smem_raw[256 * 1024];
}
#include "../../scintools_b200/csrc/thth.cu"
#include "../../scintools_b200/csrc/eig_half.cu"

extern "C" int emu_eta_sweep(const float* cs, long long ntau, long long nfd, long long cs_pitch,
                             int cs_half, double tau0, double dtau, double tau_absmax, double fd0,
                             double dfd, double fd_half, const double* th, int n_th, int coherent,
                             const double* etas, int neta, double tol, int max_iter, int mixed,
                             double* eigs, int* status, int* nred, int* iters,
                             float* M_out) {
    using namespace sb;
    ThthGeom g;
    g.cs = reinterpret_cast<const float2*>(cs);
    g.ntau = ntau; g.nfd = nfd;
    g.tau0 = tau0; g.dtau = dtau; g.half_dtau = dtau / 2; g.tau_absmax = tau_absmax;
    g.fd0 = fd0; g.dfd = dfd; g.half_dfd = dfd / 2; g.fd_half = fd_half;
    g.inv_dtau = 1.0 / dtau; g.inv_dfd = 1.0 / dfd;
    g.th = th; g.n = n_th; g.coherent = coherent; g.cs_half = cs_half; g.cs_valid_cols = 0; g.cs_bound = nullptr;
    g.cs_pitch = cs_half ? cs_pitch : (cs_pitch > 0 ? cs_pitch : nfd);
    const int ld = (n_th + 31) / 32 * 32;
    if (ld > 512) return -1;
    std::vector<int> idx((size_t)neta * ld, 0);
    std::vector<float2> M((size_t)neta * ld * ld);
    std::memset(M.data(), 0xff, M.size() * sizeof(float2));          // NaN junk, like a fresh slab
    std::vector<unsigned> Mb(mixed ? M.size() : 0, 0xffffffffu);      // written by the build kernel
    for (int e = 0; e < neta; ++e) status[e] = 0;
    for (int e = 0; e < neta; ++e)
        emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)neta, 1, 1},
                       [&]() { thth_prep_kernel(g, etas, neta, ld, idx.data(), nred); });
    for (int e = 0; e < neta; ++e)
        for (unsigned bx = 0; bx < 4; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)e, 0},
                           emu::Dim3{4, (unsigned)neta, 1},
                           [&]() { thth_indexerr_kernel(g, etas, status); });
    // scale inputs of the fp16 copy (host versions of cs_absmax_kernel / the span in eta_sweep)
    unsigned absmax_bits = 0;
    {
        float m = 0.f;
        const long long ncols = cs_half ? nfd / 2 + 1 : nfd;
        for (long long r = 0; r < ntau; ++r)
            for (long long c = 0; c < ncols; ++c) {
                const float2 q = g.cs[r * g.cs_pitch + c];
                m = std::fmax(std::fmax(std::fabs(q.x), std::fabs(q.y)), m);
            }
        absmax_bits = __float_as_uint(m);
    }
    double tmin = th[0], tmax = th[0];
    for (int k = 1; k < n_th; ++k) { tmin = th[k] < tmin ? th[k] : tmin; tmax = th[k] > tmax ? th[k] : tmax; }
    const float span = (float)((tmax - tmin) * 1.0001);
    const int T = ld / 32, npairs = T * (T + 1) / 2;
    const unsigned gx = (unsigned)((neta + SB_BUILD_EB - 1) / SB_BUILD_EB);
    for (unsigned bx = 0; bx < gx; ++bx)
        for (unsigned by = 0; by < (unsigned)npairs; ++by)
            emu::run_block(emu::Dim3{32, 8, 1}, emu::Dim3{bx, by, 0},
                           emu::Dim3{gx, (unsigned)npairs, 1},
                           [&]() {
                               if (mixed)
                                   thth_build_kernel<2, unsigned>(g, etas, 0, neta, ld, idx.data(), nred,
                                                                  M.data(), Mb.data(), &absmax_bits, span);
                               else
                                   thth_build_kernel<0, size_t>(g, etas, 0, neta, ld, idx.data(), nred,
                                                                M.data(), nullptr, nullptr, 0.f);
                           });
    if (M_out) std::memcpy(M_out, M.data(), M.size() * sizeof(float2));   // [neta][ld][ld] triangle
    if (max_iter <= 0 || max_iter > SB_LANCZOS_MAXIT) max_iter = SB_LANCZOS_MAXIT;
    if (mixed) {
        // mixed = 2: residual threshold 0 -> every curvature takes the fp32 continuation
        // from the Ritz vector
        std::vector<float2> gbasis((size_t)neta * EB_SLOTS * ld);
        for (int e = 0; e < neta; ++e) {
            std::memset(smem_raw, 0xa5, sizeof(smem_raw));     // garbage, like real shared memory
            emu::run_block(emu::Dim3{EB_THREADS + 32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                           emu::Dim3{(unsigned)neta, 1, 1}, [&]() {
                               thth_eig_half_kernel(M.data(), Mb.data(), ld, nred, 0, eigs, status,
                                                    iters, tol, 2e-7, 1e-6, mixed == 2 ? 0.0 : 1e-3,
                                                    max_iter, gbasis.data());
                           });
        }
    } else {
        for (int e = 0; e < neta; ++e)
            emu::run_block(emu::Dim3{EIG_THREADS, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                           emu::Dim3{(unsigned)neta, 1, 1}, [&]() {
                               thth_eig_kernel(M.data(), ld, nred, 0, eigs, status, iters, tol,
                                               2e-7, max_iter);
                           });
    }
    return 0;
}

// Eigen solvers on PRE-BUILT triangles M [nb][ld][ld] (strict upper triangle valid,
// diagonal / columns >= n zero): mixed == 0 -> thth_eig_kernel, else
// thth_eig_half_kernel on an fp16 copy packed here in the block layout with the same
// rule as the build kernel (power-of-two scale from the largest element).
extern "C" int emu_eig_triangles(const float* Mf, int ld, const int* nred, int nb, int mixed,
                                 double tol, int max_iter, double* eigs, int* status, int* iters) {
    using namespace sb;
    const float2* M = reinterpret_cast<const float2*>(Mf);
    if (max_iter <= 0 || max_iter > SB_LANCZOS_MAXIT) max_iter = SB_LANCZOS_MAXIT;
    for (int e = 0; e < nb; ++e) status[e] = 0;
    std::vector<unsigned> Mb;
    std::vector<float2> gbasis;
    if (mixed) {
        Mb.assign((size_t)nb * ld * ld, 0u);
        gbasis.resize((size_t)nb * EB_SLOTS * ld);
        for (int e = 0; e < nb; ++e) {
            const int n = nred[e];
            float mx = 0.f;
            for (int a = 0; a < n; ++a)
                for (int c = a + 1; c < n; ++c) {
                    const float2 q = M[((size_t)e * ld + a) * ld + c];
                    mx = std::fmax(std::fmax(std::fabs(q.x), std::fabs(q.y)), mx);
                }
            const float sc = mx > 0.f ? std::exp2(std::floor(std::log2(32768.f / mx))) : 1.f;
            for (int a = 0; a < n; ++a)
                for (int c = a; c < ld; ++c) {
                    float2 q = M[((size_t)e * ld + a) * ld + c];
                    if (c >= n || c == a) q = make_float2(0.f, 0.f);
                    const unsigned h = pack_f16x2(make_float2(q.x * sc, q.y * sc));
                    // block layout (zeros elsewhere: Mb starts as zeros)
                    unsigned short* Mh = reinterpret_cast<unsigned short*>(Mb.data() + (size_t)e * ld * ld);
                    const size_t ob = ((size_t)(a >> 4) * (ld >> 3) + (c >> 3)) * 256 + (a & 15) * 16 + (c & 7);
                    const int sw = (((a & 15) >> 2) & 1) * 8;      // halves swapped in rows 4-7, 12-15
                    Mh[ob + sw] = (unsigned short)(h & 0xffffu);
                    Mh[ob + (8 - sw)] = (unsigned short)(h >> 16);
                }
        }
    }
    for (int e = 0; e < nb; ++e) {
        std::memset(smem_raw, 0xa5, sizeof(smem_raw));
        if (mixed)
            emu::run_block(emu::Dim3{EB_THREADS + 32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                           emu::Dim3{(unsigned)nb, 1, 1}, [&]() {
                               thth_eig_half_kernel(M, Mb.data(), ld, nred, 0, eigs, status, iters, tol,
                                                    2e-7, 1e-6, mixed == 2 ? 0.0 : 1e-3, max_iter,
                                                    gbasis.data());
                           });
        else
            emu::run_block(emu::Dim3{EIG_THREADS, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                           emu::Dim3{(unsigned)nb, 1, 1}, [&]() {
                               thth_eig_kernel(M, ld, nred, 0, eigs, status, iters, tol, 2e-7,
                                               max_iter);
                           });
    }
    return 0;
}
