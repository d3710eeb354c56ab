// CPU run of the device code of the gap fills (csrc/inpaint.cu, sources unchanged) under
// the SIMT emulator: the map, setup, residual, three BiCGSTAB step and clip kernels, launched
// in the order, batches and restarts of sb::inpaint_biharmonic, and the masked median
// kernel.  The blocks of a launch run one after another in block order, so a block that
// read a flag written by an earlier block of its own launch would show here.  The block
// size and grid are arguments, so several blocks and the grid-stride loops can be
// exercised on small images.  TEST INFRASTRUCTURE (tests/test_refill_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include "../../scintools_b200/csrc/inpaint.cu"

namespace {
using namespace sb;

void grid(unsigned G, int threads, const std::function<void()>& body) {
    for (unsigned x = 0; x < G; ++x)
        emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, 0, 0},
                       emu::Dim3{G, 1, 1}, body);
}
}  // namespace

// sb_inpaint_biharmonic_f64 with `threads` per block and G blocks for every solver kernel;
// info: steps, converged, restarts, and the stop launch of the first run (-1 if none)
extern "C" int emu_inpaint(const double* img, int nf, int nt, const int* pix, int n,
                           const double* tables, const unsigned char* rcls, int nrc,
                           const unsigned char* ccls, int ncc, double lo, double hi, double tol,
                           int maxit, int threads, int G, double* out, int* info, double* resid) {
    const size_t npix = (size_t)nf * nt;
    std::vector<double> b(n), invd(n), x(n), r(n), rhat(n), s(n), t(n), p0(n), p1(n), v0(n),
        v1(n), rho(maxit + 1), alpha(maxit + 1), omega(maxit + 1), part(7 * (size_t)G);
    std::vector<int> map(npix, -1);
    double* pb[2] = {p0.data(), p1.data()};
    double* vb[2] = {v0.data(), v1.data()};
    InpState state{INP_RUNNING, 0, 0};
    InpSys S{pix, map.data(), rcls, ccls, tables, invd.data(), nf, nt, n, ncc, nrc * ncc};
    grid(2, 32, [&]() { inp_map_kernel(pix, n, map.data()); });
    grid(G, threads, [&]() { inp_setup_kernel(S, img, b.data(), invd.data(), x.data(), part.data()); });
    double bb = 0.0;
    for (int i = 0; i < G; ++i) bb += part[i];
    double* P = part.data();
    InpIter I{r.data(), rhat.data(), x.data(), s.data(), t.data(), rho.data(), alpha.data(),
              omega.data(), P, P + G, P + 2 * G, P + 3 * G, P + 4 * G, P + 5 * G, &state,
              tol * tol * bb, G};
    int used = 0, restarts = 0, first_stop = -1;
    bool converged = false;
    double rr = 0.0;
    for (;;) {
        grid(G, threads, [&]() {
            inp_residual_kernel(S, b.data(), x.data(), r.data(), rhat.data(), I.part_rr,
                                I.part_rhr, &state);
        });
        int it = 0;
        while (state.stop_at == INP_RUNNING && used + it < maxit) {
            const int stop = (used + it + INP_CHECK < maxit) ? it + INP_CHECK : maxit - used;
            for (; it < stop; ++it) {
                const int c = it & 1;
                grid(G, threads, [&]() {
                    inp_step_a_kernel(S, I, it, pb[c ^ 1], vb[c ^ 1], pb[c], vb[c]);
                });
                grid(G, threads, [&]() { inp_step_b_kernel(S, I, it, vb[c]); });
                grid(G, threads, [&]() { inp_step_c_kernel(S, I, it, pb[c]); });
            }
        }
        if (restarts == 0) first_stop = state.stop_at == INP_RUNNING ? -1 : state.stop_at;
        used += state.stop_at != INP_RUNNING ? state.steps : it;
        grid(G, threads, [&]() {
            inp_residual_kernel(S, b.data(), x.data(), nullptr, nullptr, P + 6 * G, nullptr,
                                nullptr);
        });
        rr = 0.0;
        for (int i = 0; i < G; ++i) rr += P[6 * G + i];
        converged = rr <= I.thr;
        if (converged || used >= maxit || restarts >= INP_RESTARTS || !std::isfinite(rr)) break;
        ++restarts;
    }
    grid(2, 32, [&]() { inp_clip_kernel(x.data(), n, lo, hi, out); });
    info[0] = used;
    info[1] = converged ? 1 : 0;
    info[2] = restarts;
    info[3] = first_stop;
    *resid = bb > 0.0 ? std::sqrt(rr / bb) : std::sqrt(rr);
    return 0;
}

extern "C" int emu_medfilt(const double* img, int nf, int nt, const int* pix, int n, int kh,
                           int kw, double nan_value, double* out) {
    if (kh * kw <= 25)
        grid(3, 32, [&]() { med_masked_kernel<25>(img, nf, nt, pix, n, kh, kw, nan_value, out); });
    else if (kh * kw <= 121)
        grid(3, 32, [&]() { med_masked_kernel<121>(img, nf, nt, pix, n, kh, kw, nan_value, out); });
    else
        grid(3, 32, [&]() { med_masked_kernel<961>(img, nf, nt, pix, n, kh, kw, nan_value, out); });
    return 0;
}
