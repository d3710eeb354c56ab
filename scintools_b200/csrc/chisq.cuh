// Residual of the rank-1 theta-theta model against the dynamic spectrum
// (ththmod.chisq_calc, ththmod.py:330-368), fused into the final store of the
// inverse 2-D FFT so that the model is never written to memory.
#pragma once
#include "common.cuh"

namespace sb {

// fp64 partial sums per curvature; consecutive columns go to different slots so
// that the atomics of one warp never meet on one address
constexpr int CHISQ_SLOTS = 64;

// sum over mask of (model - dspec)^2; mask == nullptr: isfinite(dspec)
struct ResidualSink {
    const float* dspec;            // [nf][nt]
    const unsigned char* mask;     // [nf][nt] or null
    int nf, nt;
    double* part;                  // [CHISQ_SLOTS]
    __device__ __forceinline__ void operator()(int row, int c, float model) const {
        if (row >= nf || c >= nt) return;
        const size_t o = (size_t)row * nt + c;
        const float d = dspec[o];
        if (mask ? !mask[o] : !isfinite(d)) return;
        const double r = (double)model - (double)d;
        atomicAdd(part + (o % CHISQ_SLOTS), r * r);
    }
};

}  // namespace sb
