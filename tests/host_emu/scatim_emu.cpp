// CPU run of the device code of Dynspec.calc_scattered_image (csrc/scatim.cu, sources
// unchanged) under the SIMT emulator: the linear, delay, Doppler, evaluation and shift
// kernels with the arguments, grids and order of sb::scattered_image.  The blocks of a launch
// run one after another.
// TEST INFRASTRUCTURE (tests/test_scattered_image_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include <vector>

#include "../../include/scint_b200_scatim.h"

#include "../../scintools_b200/csrc/scatim.cu"

namespace {
using namespace sb;

void grid(unsigned gx, unsigned gy, int threads, const std::function<void()>& body) {
    for (unsigned y = 0; y < gy; ++y)
        for (unsigned x = 0; x < gx; ++x)
            emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, y, 0},
                           emu::Dim3{gx, gy, 1}, body);
}
}  // namespace

extern "C" void emu_scattered_image(const sb_scatim* s) {
    const int ni = s->nitem, mx = s->mx, my = s->my, nx = s->nx, ny = s->ny;
    const int nb = si_eval_blocks(nx, ny);
    std::vector<double> w((size_t)mx * my * ni), bmin((size_t)nb * ni);
    grid(3, 1, 64, [&]() {
        si_linear_kernel(s->sspec, (const long long*)s->offset, (long long)s->pitch, ni, mx, my,
                         w.data());
    });
    grid((unsigned)((my + 127) / 128), (unsigned)ni, 128,
         [&]() { si_delay_kernel(w.data(), mx, my, s->fx); });
    grid((unsigned)((mx + 32 * SI_WARPS - 1) / (32 * SI_WARPS)), (unsigned)ni, 32 * SI_WARPS,
         [&]() { si_doppler_kernel(w.data(), mx, my, s->fy); });
    SiEval e{s->tx, s->ty, s->ax, s->ay, w.data(), s->eta, s->image, bmin.data(), mx, my, nx, ny};
    grid((unsigned)nb, (unsigned)ni, SI_THREADS, [&]() { si_eval_kernel(e); });
    if (s->shift)
        grid(2, (unsigned)ni, 256,
             [&]() { si_shift_kernel(s->image, (long long)nx * nx, bmin.data(), nb); });
}
