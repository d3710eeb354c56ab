// CPU run of the device code of the wavefield mosaic (csrc/mosaic.cu, sources unchanged)
// under the SIMT emulator: mosaic_tile_kernel in all five modes and the four reduction
// kernels, launched as sb::mosaic_* launches them (one 128-thread block per tile; the
// reductions as one block that strides over its items).  TEST INFRASTRUCTURE
// (tests/test_mosaic_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include <limits.h>

namespace sb {
alignas(128) unsigned char smem_raw[64 * 1024];
}
#include "../../scintools_b200/csrc/mosaic.cu"

namespace {
using namespace sb;

template <int MODE>
void run_tiles(const MosGeom& g, const float* chunks, const double* phi, const double* amp,
               float* W, const float* dspec, const float* noise, double* part) {
    for (long long t = 0; t < g.ntiles; ++t)
        emu::run_block(emu::Dim3{MOS_THREADS, 1, 1}, emu::Dim3{(unsigned)t, 0, 0},
                       emu::Dim3{(unsigned)g.ntiles, 1, 1}, [&]() {
                           mosaic_tile_kernel<MODE>(g, reinterpret_cast<const float2*>(chunks),
                                                    phi, amp, reinterpret_cast<float2*>(W),
                                                    dspec, noise, part);
                       });
}

void run1(int threads, const std::function<void()>& body) {
    emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{0, 0, 0}, emu::Dim3{1, 1, 1},
                   body);
}
}  // namespace

// mode 0 build: W float2 [nF][nT].  1 rot (W in): out0 = power [1], out1 = der [P].
// 2 overlap: out0 = C float64 complex [P][4].  3 fit (W in): out0 = fit [1], out1 = grad [P][2].
// 4 hess (W in): rows, cols int64 [40 P], out0 = vals [40 P].
extern "C" int emu_mosaic(int mode, const float* chunks, int ncf, int nct, int cwf, int cwt,
                          const double* phi, const double* amp, float* W, const float* dspec,
                          const float* noise, double* out0, double* out1, long long* rows,
                          long long* cols) {
    MosGeom g;
    mos_geom_fill(ncf, nct, cwf, cwt, &g);
    std::vector<double> part((size_t)g.ntiles * 44);
    double* p = part.data();
    switch (mode) {
    case MOS_BUILD:
        run_tiles<MOS_BUILD>(g, chunks, phi, amp, W, nullptr, nullptr, nullptr);
        break;
    case MOS_ROT:
        run_tiles<MOS_ROT>(g, chunks, phi, nullptr, W, nullptr, nullptr, p);
        run1(256, [&]() { mosaic_chunk_kernel<MOS_ROT>(g, p, nullptr, out1); });
        run1(256, [&]() { mosaic_total_kernel<MosNq<MOS_ROT>::value>(g.ntiles, p, out0); });
        break;
    case MOS_OVERLAP:
        run_tiles<MOS_OVERLAP>(g, chunks, nullptr, nullptr, nullptr, nullptr, nullptr, p);
        run1(256, [&]() { mosaic_overlap_kernel(g, p, out0); });
        break;
    case MOS_FIT:
        run_tiles<MOS_FIT>(g, chunks, phi, amp, W, dspec, noise, p);
        run1(256, [&]() { mosaic_chunk_kernel<MOS_FIT>(g, p, amp, out1); });
        run1(256, [&]() { mosaic_total_kernel<MosNq<MOS_FIT>::value>(g.ntiles, p, out0); });
        break;
    case MOS_HESS:
        run_tiles<MOS_HESS>(g, chunks, phi, amp, W, dspec, noise, p);
        run1(256, [&]() { mosaic_hess_kernel(g, p, amp, rows, cols, out0); });
        break;
    default:
        return -1;
    }
    return 0;
}
