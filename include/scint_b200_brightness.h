/* libscint_b200 -- scint_sim.Brightness (reference scintools/scint_sim.py:768-958).
 *
 * Declared apart from include/scint_b200.h so that header keeps the entry points of ABI
 * version 8 exactly; the conventions of scint_b200.h hold here too (status codes,
 * sb_last_error, device pointers, caller stream, calls ordered across streams).
 */
#ifndef SCINT_B200_BRIGHTNESS_H
#define SCINT_B200_BRIGHTNESS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* stages of sb_brightness_f64, any combination; they run in this order */
#define SB_BRIGHT_EFIELD 1   /* calc_brightness: rho, B */
#define SB_BRIGHT_SSPEC 2    /* calc_SS: thetax, thetay, jac, ss, lss (reads B) */
#define SB_BRIGHT_ACF 4      /* calc_acf: acf (reads ss) */

/* per-set scalars in par[set][SB_BRIGHT_NPAR], each built on the host by the reference's own
 * expression: a, b, c (the quadratic form), alph2 = alpha/2, thetagy, thetarx**2, thetary**2 */
#define SB_BRIGHT_NPAR 7

/* Limits: lattice side n 2..1024, ntd and nfd 1..4096, nset 1..65535. */
#define SB_BRIGHT_MAX_N 1024
#define SB_BRIGHT_MAX_Q 4096

/* A batch of nset parameter sets on one lattice x (n points, strictly increasing) and one
 * (td, fd) query grid.  All float64, C-contiguous, device pointers.
 *   x [n]; diag: the Delaunay diagonal of each lattice cell, (n-1)^2 bits in numpy packbits
 *     order (bit k of cell k = i (n-1) + j set: the cell's triangles share the corner pair
 *     (x[j], x[i]), (x[j+1], x[i+1]); clear: the other pair); td [ntd];
 *   colx [nset][nfd]: thetax of each Doppler column, fd - thetagx + thetarx;
 *   colq [nset][nfd]: (thetax + thetagx)**2 as the reference's scalar power rounds it;
 *   half_df = 0.5*df, jac_cap = 2/df, jac_out = 10**(-6).
 * EFIELD writes rho [nset][n][n] (acf_efield) and B [nset][n][n] = |ifftshift(fft2(
 * fftshift(rho)))|.  SSPEC reads B and writes thetax, thetay, jac, ss, lss [nset][ntd][nfd]:
 * ss interpolates B linearly on the triangulation (NaN outside the lattice), is multiplied
 * by the Jacobian and flip-added as numpy does; lss = 10 log10(ss).  ACF reads ss and writes
 * acf [nset][ntd][nfd] = real(fftshift(fft2(fftshift(ss)))) / its maximum.  Pointers of
 * stages not run may be NULL.  Workspace: the twiddle matrices (16 (n^2 or ntd^2 + nfd^2)
 * bytes) and, per set, 16 max(n^2, ntd nfd) + 8 ntd nfd bytes.  No atomics: each set's
 * result is bit-identical in any batch and on repeat. */
typedef struct sb_brightness {
    int32_t nset, n, ntd, nfd, stages;
    const double* x;
    const uint8_t* diag;
    const double* td;
    const double* par;
    const double* colx;
    const double* colq;
    double half_df, jac_cap, jac_out;
    double* rho;
    double* B;
    double* thetax;
    double* thetay;
    double* jac;
    double* ss;
    double* lss;
    double* acf;
} sb_brightness;

int sb_brightness_f64(const sb_brightness* d, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SCINT_B200_BRIGHTNESS_H */
