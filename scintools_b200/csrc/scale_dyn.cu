// Dynspec.scale_dyn(scale='lambda') (scintools/dynspec.py:3926-3957): resample
// every time column from the frequency grid to equal wavelength steps with a
// not-a-knot cubic spline (scipy interp1d(kind='cubic')).
//
// Algorithm: second-derivative form, Thomas factors shared by all columns,
// 4 weights per output row; host tables built by the Python mirror in fp64.
// GPU parity vs the reference: tests/test_gpu_parity.py::test_scale_dyn_lambda.
//
// The knots are the same for every column, so the tridiagonal system for the
// second derivatives M has column-independent factors (host, fp64):
//   forward   d_i = (r_i - a_i d_{i-1}) * inv_i,   r_i = (y_{i+1}-y_i) g_i - (y_i-y_{i-1}) g_{i-1}
//   backward  M_i = d_i - cp_i M_{i+1}             (i = n-2 .. 1)
//   ends      M_0 = (1+p0) M_1 - p0 M_2,  M_{n-1} = (1+pn) M_{n-2} - pn M_{n-3}
// One thread per time column (coalesced over t), then a gather kernel
//   out[nlam-1-k][t] = W_k0 y[i_k][t] + W_k1 y[i_k+1][t] + W_k2 M[i_k][t] + W_k3 M[i_k+1][t].
// HBM-bound: ~7 passes over nf*nt*4 B.
#include "common.cuh"
#include "drivers.cuh"

namespace sb {

__global__ void spline_moments_kernel(const float* __restrict__ dyn, int nf, int nt, int flip,
                                      const float* __restrict__ a, const float* __restrict__ cp,
                                      const float* __restrict__ inv, const float* __restrict__ g,
                                      float p0, float pn, float* __restrict__ M) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    // knot i (ascending frequency) lives in row (flip ? nf-1-i : i)
    auto Y = [&](int i) { return dyn[(size_t)(flip ? nf - 1 - i : i) * nt + t]; };
    float ym = Y(0), y0 = Y(1), prev = 0.f;
    for (int i = 1; i < nf - 1; ++i) {
        const float yp = Y(i + 1);
        const float r = (yp - y0) * g[i] - (y0 - ym) * g[i - 1];
        prev = (r - a[i] * prev) * inv[i];
        M[(size_t)i * nt + t] = prev;
        ym = y0;
        y0 = yp;
    }
    float nxt = 0.f, m1 = 0.f, m2 = 0.f;      // M_{i+1}, and M_1 / M_2 for the left end
    float mn2 = 0.f, mn3 = 0.f;               // M_{n-2}, M_{n-3}
    for (int i = nf - 2; i >= 1; --i) {
        nxt = M[(size_t)i * nt + t] - cp[i] * nxt;
        M[(size_t)i * nt + t] = nxt;
        if (i == nf - 2) mn2 = nxt;
        if (i == nf - 3) mn3 = nxt;
        if (i == 2) m2 = nxt;
        if (i == 1) m1 = nxt;
    }
    if (nf == 4) { mn3 = m1; m2 = mn2; }      // n-3 == 1 and 2 == n-2
    M[t] = (1.f + p0) * m1 - p0 * m2;
    M[(size_t)(nf - 1) * nt + t] = (1.f + pn) * mn2 - pn * mn3;
}

__global__ void spline_eval_kernel(const float* __restrict__ dyn, const float* __restrict__ M,
                                   int nf, int nt, int flip, const int* __restrict__ idx,
                                   const float4* __restrict__ W, int nlam,
                                   float* __restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    // rows k = blockIdx.y + m gridDim.y: gridDim.y is capped at 65535, nlam is not
    for (int k = blockIdx.y; k < nlam; k += gridDim.y) {
        const int i = idx[k];
        const float4 w = W[k];
        const size_t r0 = (size_t)(flip ? nf - 1 - i : i) * nt + t;
        const size_t r1 = (size_t)(flip ? nf - 2 - i : i + 1) * nt + t;
        const float v = w.x * dyn[r0] + w.y * dyn[r1] + w.z * M[(size_t)i * nt + t] +
                        w.w * M[(size_t)(i + 1) * nt + t];
        out[(size_t)(nlam - 1 - k) * nt + t] = v;     // np.flipud: wavelength ascending
    }
}

#ifndef SB_HOST_EMU
int scale_dyn_lambda(const float* dyn, int nf, int nt, int flip, const float* a,
                     const float* cp, const float* inv, const float* g, float p0, float pn,
                     const int* idx, const float4* W, int nlam, float* out, cudaStream_t st) {
    if (nf < 4) {
        set_error("scale_dyn: a cubic spline needs at least 4 channels (got %d)", nf);
        return SB_ERR_UNSUPPORTED;
    }
    float* M = (float*)workspace(WS_PLANE0, (size_t)nf * nt * sizeof(float));
    if (!M) return SB_ERR_NOMEM;
    spline_moments_kernel<<<(nt + 127) / 128, 128, 0, st>>>(dyn, nf, nt, flip, a, cp, inv, g, p0,
                                                           pn, M);
    SB_LAUNCH_CHECK();
    dim3 grid((nt + 255) / 256, nlam < 65535 ? nlam : 65535);
    spline_eval_kernel<<<grid, 256, 0, st>>>(dyn, M, nf, nt, flip, idx, W, nlam, out);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
#endif  // SB_HOST_EMU

}  // namespace sb
