// scint_utils.slow_FT (scint_utils.py:655-702): the Doppler transform of a wideband
// dynamic spectrum with time scaled by s_f = f / fref in each channel, then the FFT over
// frequency.  x is [nt][nf] (time-major); with c = nt / 2 and a_f = s_f / nt
//   Y[m][f]   = sum_t x[t][f] exp(-2 pi i a_f t (m - c))                   m < nt
//   out[m][j] = sum_f Y[m][f] exp(-2 pi i f (j - nf/2) / nf)              j < nf
// Doppler axis: a fractional Fourier transform per channel, by Bluestein's identity
// t (m - c) = (t^2 + m^2 - (m - t)^2) / 2 - c t
//   Y[m][f] = exp(-i pi a_f m^2) sum_t [x[t][f] exp(-i pi a_f (t^2 - 2 c t))] b_f[m - t],
//   b_f[n] = exp(+i pi a_f n^2),
// a cyclic convolution of length M = max(8, 2^ceil(log2(2 nt - 1))): three column
// transforms of length M over the nf channels (the kernels b_f, the chirped data, the
// inverse), each the four-step pair of tile passes of cols_generic.  The chirps are
// generated in the load / store functors (fft_functors.cuh) from float64 phases.
// Delay axis: a length-nf FFT of every row of Y, in place in `out`, with the fftshift
// folded into the store: the radix row kernel for powers of two from 8, the row chirp-z
// of chirp_fft2 for every other length.
#include "drivers.cuh"
#include "fft_kernels.cuh"

namespace sb {

int slow_ft(const float* x, int nt, int nf, const double* s, float2* out, cudaStream_t st) {
    if (nt < 1 || nt > 32768 || nf < 1 || nf > 8192) {
        set_error("slow_FT: dynspec %d x %d outside 1..32768 x 1..8192 (ntime x nfreq)", nt, nf);
        return SB_ERR_UNSUPPORTED;
    }
    const int M = next_pow2(2L * nt - 1) < 8 ? 8 : next_pow2(2L * nt - 1);
    const long pt = ((long)nf + 15) & ~15L;
    // C0: cols_generic's intermediate; Bp: the kernel transforms B_f, then A_f B_f in place
    float2* C0 = (float2*)workspace(WS_PLANE2, (size_t)M * pt * sizeof(float2));
    float2* Bp = (float2*)workspace(WS_PLANE4, (size_t)M * pt * sizeof(float2));
    if (!C0 || !Bp) return SB_ERR_NOMEM;
    int R1, R2;
    split_len(M, &R1, &R2);
    int rc;
    {
        ProfScope prof(PROF_SFT_DOPPLER, st);
        rc = cols_generic<float, -1>(SlowKernelColLoad{R2, M, nt, s}, C0, pt, M, nf,
                                     NaturalBStore<float2>{Bp, pt, R1}, st);
        if (rc) return rc;
        rc = cols_generic<float, -1>(SlowChirpColLoad{x, nf, nt, R2, s}, C0, pt, M, nf,
                                     MulPlaneColStore{Bp, pt, R1}, st);
        if (rc) return rc;
        rc = cols_generic<float, +1>(StrideALoad<float2>{Bp, pt, R2}, C0, pt, M, nf,
                                     SlowChirpOutColStore{out, nf, nt, R1, s, 1.0f / (float)M},
                                     st);
        if (rc) return rc;
    }
    ProfScope prof(PROF_SFT_DELAY, st);
    if (nf >= 8 && is_pow2(nf)) {
        // in place: a row's CTA loads the whole row before it stores any of it
        SB_ROW_DISPATCH(nf, rc = (launch_row_c2c<float, N1, N2, -1>(
                                PitchRowLoad<float2>{out, nf}, ShiftRowStore{out, nf}, nt, st)));
        return rc;
    }
    const int MT = next_pow2(2L * nf - 1) < 8 ? 8 : next_pow2(2L * nf - 1);
    float2* tabs = (float2*)workspace(WS_PLANE3, (size_t)(nf + 3L * MT) * sizeof(float2));
    float2* buf = (float2*)workspace(WS_PLANE0, (size_t)nt * MT * sizeof(float2));
    if (!tabs || !buf) return SB_ERR_NOMEM;
    float2* wT = tabs;
    float2* BT = wT + nf;
    rc = bluestein_tables(nf, MT, wT, BT, BT + MT, st);
    if (rc) return rc;
    return chirp_rows(ChirpRowLoadC{out, nt, nf, 0, 1, nullptr},
                      ChirpShiftRowStore{out, nf, wT, 1.0f / (float)MT}, buf, MT, nt, wT, BT, st);
}

}  // namespace sb
