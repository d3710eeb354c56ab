// CPU run of the device code of sb::asymmetry_batch around the eigenpair, under the SIMT
// emulator: thth_prep_table_kernel (csrc/thth.cu), asym_gather_kernel and
// asym_finish_kernel (csrc/retrieval.cu), sources unchanged, launch shapes as in
// sb::asymmetry_batch (smaller gather grids; the kernel strides over its work).  The
// eigenvectors are inputs, so the asymmetry is checked on exactly the vectors the oracle
// uses.  TEST INFRASTRUCTURE (tests/test_asymmetry_cpu.py).
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

// nchunk chunks sharing ntau x nfd full-plane spectra and n_th centres; per chunk k:
// cs[k] float2 [ntau][nfd], ax[k] = {tau0, dtau, tau_absmax, fd0, dfd, fd_half}, th[k] [n_th],
// etas[k].  Outputs: nred [nchunk], M float2 [nchunk][ld][ld] (strict upper triangles of
// the crops; everything else keeps the caller's fill), ld = n_th rounded up to 32.
extern "C" int emu_asym_gather(const float* const* cs, int nchunk, long long ntau, long long nfd,
                               const double* ax, const double* const* th, int n_th,
                               const double* etas, int* nred, float* M_out) {
    using namespace sb;
    std::vector<ThthGeom> geoms(nchunk);
    for (int k = 0; k < nchunk; ++k) {
        ThthGeom& g = geoms[k];
        const double* a = ax + 6 * k;
        g.cs = reinterpret_cast<const float2*>(cs[k]);
        g.ntau = ntau; g.nfd = nfd;
        g.tau0 = a[0]; g.dtau = a[1]; g.half_dtau = a[1] / 2; g.tau_absmax = a[2];
        g.fd0 = a[3]; g.dfd = a[4]; g.half_dfd = a[4] / 2; g.fd_half = a[5];
        g.inv_dtau = 1.0 / a[1]; g.inv_dfd = 1.0 / a[4];
        g.th = th[k]; g.n = n_th; g.coherent = 1; g.cs_half = 0; g.cs_valid_cols = 0;
        g.cs_bound = nullptr; g.cs_pitch = nfd;
    }
    const int ld = (n_th + 31) / 32 * 32;
    std::vector<int> idx((size_t)nchunk * ld, 0);
    for (int e = 0; e < nchunk; ++e)
        emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)nchunk, 1, 1},
                       [&]() { thth_prep_table_kernel(geoms.data(), etas, ld, idx.data(), nred); });
    float2* M = reinterpret_cast<float2*>(M_out);
    for (int e = 0; e < nchunk; ++e)
        for (unsigned bx = 0; bx < 8; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)e, 0},
                           emu::Dim3{8, (unsigned)nchunk, 1}, [&]() {
                               asym_gather_kernel(geoms.data(), etas, 0, ld, idx.data(), nred, M);
                           });
    return 0;
}

// V float2 [nb][ld]; nred, status [nb]; outputs asym [nb], v_out float2 [nb][ld]
extern "C" int emu_asym_finish(const float* V, int nb, int ld, const int* nred, const int* status,
                               double* asym, float* v_out) {
    using namespace sb;
    for (int e = 0; e < nb; ++e)
        emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)nb, 1, 1}, [&]() {
                           asym_finish_kernel(reinterpret_cast<const float2*>(V), ld, nred, status,
                                              0, asym, reinterpret_cast<float2*>(v_out));
                       });
    return 0;
}
