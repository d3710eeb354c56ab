// CPU run of the device code of the flux-variation correction (csrc/svd.cu, sources
// unchanged) under the SIMT emulator: the gram pass (svd_gram_kernel, G blocks of
// SVD_THREADS, then svd_reduce_kernel), the final pass (svd_apply_kernel), the Lanczos
// vector kernels, the three bandpass kernels and the host QL of the tridiagonal, launched
// as sb::svd_topk / svd_apply / bandpass_* launch them.  TEST INFRASTRUCTURE
// (tests/test_correct_dyn_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

namespace sb {
alignas(128) unsigned char smem_raw[256 * 1024];
}
#include "../../scintools_b200/csrc/svd.cu"

namespace {
using namespace sb;

int cols_of(int nt) {
    int C = 1;
    while (C * SVD_THREADS < nt) C *= 2;
    return C;
}

void grid(unsigned gx, unsigned gy, int threads, const std::function<void()>& body) {
    for (unsigned y = 0; y < gy; ++y)
        for (unsigned x = 0; x < gx; ++x)
            emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, y, 0},
                           emu::Dim3{gx, gy, 1}, body);
}

#define EMU_DISPATCH(C, call)                                   \
    switch (C) {                                                \
    case 1: call(1); break;                                     \
    case 2: call(2); break;                                     \
    case 4: call(4); break;                                     \
    case 8: call(8); break;                                     \
    case 16: call(16); break;                                   \
    default: call(32); break;                                   \
    }
}  // namespace

// w = A^T (A x) through G gram blocks (part: G x nt partials) and the reduction
extern "C" int emu_gram(const float* A, int nf, int nt, int G, const double* x, double* part,
                        double* w) {
#define GRAM(C) grid(G, 1, SVD_THREADS, [&]() { svd_gram_kernel<C>(A, nf, nt, x, part); })
    EMU_DISPATCH(cols_of(nt), GRAM)
#undef GRAM
    grid(2, 1, 64, [&]() { svd_reduce_kernel(part, G, nt, w); });
    return 0;
}

extern "C" int emu_apply(const float* A, int nf, int nt, int k, const double* Y, int G,
                         float* out, float* model) {
#define APPLY(C) grid(G, 1, SVD_THREADS, [&]() { svd_apply_kernel<C>(A, nf, nt, k, Y, out, model); })
    EMU_DISPATCH(cols_of(nt), APPLY)
#undef APPLY
    return 0;
}

// one full re-orthogonalised step's vector work: h = V^T w, w -= V h (twice), *nrm = ||w||,
// alpha[m] = h1[m] + h2[m], v = w / nrm, or -- on breakdown -- the restart vector
extern "C" int emu_orth(const double* V, int nq, int nt, double* w, double* h1, double* h2,
                        double* alpha, double* nrm, double* v, double* amax, int* restart) {
    for (int pass = 0; pass < 2; ++pass) {
        double* h = pass ? h2 : h1;
        grid(nq, 1, SVD_RED_THREADS, [&]() { svd_dots_kernel(V, nq, nt, w, h); });
        grid(2, 1, 64, [&]() { svd_orth_kernel(V, nq, nt, h, w); });
    }
    grid(1, 1, SVD_RED_THREADS, [&]() {
        svd_norm_kernel(w, nt, nrm, nq - 1, h1, h2, alpha, amax, restart);
    });
    grid(2, 1, 64, [&]() { svd_scale_kernel(w, nt, nrm, restart, v); });
    grid(1, 1, 128, [&]() { svd_restart_kernel(restart, V, nq, nt, v); });
    return 0;
}

extern "C" int emu_ql(int n, double* d, double* e, double* Z, int nz) {
    return svd_tridiag_ql(n, d, e, Z, nz);
}

extern "C" int emu_bandpass(const float* A, int nf, int nt, int zero_as_nan, const double* rowdiv,
                            const double* coldiv, int nchunk, double* rowmean, double* colmean,
                            float* out) {
    grid(3, 1, BP_THREADS, [&]() { bandpass_row_kernel(A, nf, nt, zero_as_nan, rowmean); });
    const int rows_per = (nf + nchunk - 1) / nchunk;
    nchunk = (nf + rows_per - 1) / rows_per;
    std::vector<double> ps((size_t)nchunk * nt), pc((size_t)nchunk * nt);
    const unsigned gx = (nt + BP_THREADS - 1) / BP_THREADS;
    grid(gx, nchunk, BP_THREADS, [&]() {
        bandpass_col_kernel(A, nf, nt, zero_as_nan, rowdiv, rows_per, ps.data(), pc.data());
    });
    grid(1, 1, 64, [&]() { bandpass_col_reduce_kernel(ps.data(), pc.data(), nchunk, nt, colmean); });
    grid(3, 1, 128, [&]() {
        bandpass_divide_kernel(A, nf, nt, zero_as_nan, rowdiv, coldiv, out);
    });
    return 0;
}
