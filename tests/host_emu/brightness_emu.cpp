// CPU run of the device code of scint_sim.Brightness (csrc/brightness.cu, sources unchanged)
// under the SIMT emulator: the rho, twiddle, matrix-product, query, flip and normalise
// kernels with the arguments and in the order of sb::brightness.  The blocks of a launch run
// one after another.  The FP64 tensor-core instruction is replaced by a warp-wide exchange
// with the same fragment layout (br_mma below).
// TEST INFRASTRUCTURE (tests/test_brightness_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include "../../include/scint_b200_brightness.h"

static inline void sincospi(double x, double* s, double* c) {
    *s = std::sin(M_PI * x);
    *c = std::cos(M_PI * x);
}

struct dim3 { unsigned x, y, z; };

namespace sb {
// mma.sync m8n8k4 .f64: lane l holds A[l / 4][l % 4], B[l % 4][l / 4] and
// D[l / 4][2 (l % 4) + {0, 1}]
inline void br_mma(double2& d, double a, double b) {
    unsigned long long A[32], Bv[32];
    emu::warp_gather(emu::to_bits(a), A);
    emu::warp_gather(emu::to_bits(b), Bv);
    const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
    for (int k = 0; k < 4; ++k) {
        const double ak = emu::from_bits<double>(A[g * 4 + k]);
        d.x = std::fma(ak, emu::from_bits<double>(Bv[(2 * t) * 4 + k]), d.x);
        d.y = std::fma(ak, emu::from_bits<double>(Bv[(2 * t + 1) * 4 + k]), d.y);
    }
}
}  // namespace sb

#include "../../scintools_b200/csrc/brightness.cu"

namespace {
using namespace sb;

void grid(unsigned gx, unsigned gy, unsigned gz, int threads, const std::function<void()>& body) {
    for (unsigned z = 0; z < gz; ++z)
        for (unsigned y = 0; y < gy; ++y)
            for (unsigned x = 0; x < gx; ++x)
                emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, y, z},
                               emu::Dim3{gx, gy, gz}, body);
}

dim3 tiles(int M, int N, int nset) {
    return dim3{(unsigned)((N + BR_BN - 1) / BR_BN), (unsigned)((M + BR_BM - 1) / BR_BM),
                (unsigned)nset};
}
}  // namespace

extern "C" void emu_brightness(const sb_brightness* d) {
    const int n = d->n, ntd = d->ntd, nfd = d->nfd, ns = d->nset, stg = d->stages;
    const long long n2 = (long long)n * n, nq = (long long)ntd * nfd;
    if (stg & SB_BRIGHT_EFIELD) {
        std::vector<double> w(2 * n2), t(2 * n2 * ns);
        grid(3, 1, 1, 64, [&]() { br_rho_kernel(ns, n, d->x, d->par, d->rho); });
        grid(3, 1, 1, 64, [&]() { br_twiddle_kernel(n, n / 2, n / 2, w.data(), w.data() + n2); });
        BrGemm g1{w.data(), w.data() + n2, d->rho, nullptr, t.data(), t.data() + n2 * ns,
                  nullptr, 0, n2, n2, n, n, n};
        const dim3 gr = tiles(n, n, ns);
        grid(gr.x, gr.y, gr.z, BR_THREADS, [&]() { br_gemm_kernel<false, BR_STORE>(g1); });
        BrGemm g2{t.data(), t.data() + n2 * ns, w.data(), w.data() + n2, d->B, nullptr,
                  nullptr, n2, 0, n2, n, n, n};
        grid(gr.x, gr.y, gr.z, BR_THREADS, [&]() { br_gemm_kernel<true, BR_ABS>(g2); });
    }
    if (stg & SB_BRIGHT_SSPEC) {
        std::vector<double> pre(nq * ns);
        BrQuery a{d->x, d->td, d->colx, d->colq, d->par, d->B, d->diag, d->thetax, d->thetay,
                  d->jac, pre.data(), ns, n, ntd, nfd, d->half_df, d->jac_cap, d->jac_out};
        grid(3, 1, 1, 64, [&]() { br_query_kernel(a); });
        grid(3, 1, 1, 64, [&]() { br_flip_kernel(ns, ntd, nfd, pre.data(), d->ss, d->lss); });
    }
    if (stg & SB_BRIGHT_ACF) {
        const long long m1 = (long long)ntd * ntd, m2 = (long long)nfd * nfd;
        const dim3 gr = tiles(ntd, nfd, ns);
        const int ntile = (int)(gr.x * gr.y);
        std::vector<double> w(2 * (m1 + m2)), t(2 * nq * ns), cmax((size_t)ntile * ns);
        double *w1 = w.data(), *w2 = w.data() + 2 * m1;
        const int h1 = ntd / 2, h2 = nfd / 2;
        grid(3, 1, 1, 64, [&]() { br_twiddle_kernel(ntd, ntd - h1, h1, w1, w1 + m1); });
        grid(3, 1, 1, 64, [&]() { br_twiddle_kernel(nfd, h2, nfd - h2, w2, w2 + m2); });
        BrGemm g1{w1, w1 + m1, d->ss, nullptr, t.data(), t.data() + nq * ns, nullptr, 0, nq, nq,
                  ntd, nfd, ntd};
        grid(gr.x, gr.y, gr.z, BR_THREADS, [&]() { br_gemm_kernel<false, BR_STORE>(g1); });
        BrGemm g2{t.data(), t.data() + nq * ns, w2, w2 + m2, d->acf, nullptr, cmax.data(), nq, 0,
                  nq, ntd, nfd, nfd};
        grid(gr.x, gr.y, gr.z, BR_THREADS, [&]() { br_gemm_kernel<true, BR_REAL>(g2); });
        grid(2, (unsigned)ns, 1, 256,
             [&]() { br_normalise_kernel(d->acf, nq, cmax.data(), ntile); });
    }
}
