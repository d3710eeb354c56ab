/* libscint_b200 -- Dynspec.calc_scattered_image (reference scintools/dynspec.py:3412-3582).
 *
 * Declared apart from include/scint_b200.h so that header keeps the entry points of ABI
 * version 8 exactly; the conventions of scint_b200.h hold here too (status codes,
 * sb_last_error, device pointers, caller stream, calls ordered across streams).
 */
#ifndef SCINT_B200_SCATIM_H
#define SCINT_B200_SCATIM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Limits: crop boxes of 4..65536 delays by 4..32768 Doppler columns (every halved or full
 * secondary spectrum of a dynamic spectrum up to 32768 x 16384), images of nx = 1..8193
 * (sampling 0..4096), 1..65535 items per call. */
#define SB_SCATIM_MIN_M 4
#define SB_SCATIM_MAX_MX 65536
#define SB_SCATIM_MAX_MY 32768
#define SB_SCATIM_MAX_NX 8193

/* Band factors of one axis's collocation matrix A[i][j] = B_j(x_i) (cubic B-splines on the
 * knots [x0]*4 + x[2:-2] + [x_last]*4), A = L U without pivoting; L is unit lower with two
 * subdiagonals, U upper with two superdiagonals.  Stored [5][m]:
 *   l2[i] = L[i][i-2], l1[i] = L[i][i-1], dinv[i] = 1 / U[i][i], u1[i] = U[i][i+1],
 *   u2[i] = U[i][i+2], zero where the index leaves the matrix. */
#define SB_SCATIM_NFAC 5

/* A stack of nitem items that share one crop box shape (mx delays by my Doppler columns),
 * the axes' tables and the image grid.  All float64, device pointers.
 *   sspec: the dB spectra; item k's crop box starts at sspec + offset[k], rows pitch
 *     elements apart (offset [nitem], int64, device);
 *   eta [nitem]: each item's curvature;
 *   tx [mx + 4], fx [5][mx]: knots and band factors of the delay axis; ty [my + 4],
 *     fy [5][my]: those of the Doppler axis;
 *   ax [nx]: fdop_x; ay [ny]: fdop_y; nx = 2 ny - 1;
 *   shift: 1 applies image -= min(image); image += 1e-10 (NaN if any pixel is NaN).
 * Writes image [nitem][nx][nx]: the interpolating bicubic spline of 10**(sspec/10) over the
 * crop box, evaluated as FITPACK's fpbisp does (each query clamped to the knot range) at
 * (delay, Doppler) = ((ax[c]**2 + ay[i]**2) * eta, ax[c]), times ay[i], at rows ny-1 +- i.
 * Workspace: 8 nitem mx my bytes (the coefficients) and 8 bytes per evaluation block.
 * No atomics: each item's image is bit-identical in any stack and on repeat. */
typedef struct sb_scatim {
    int32_t nitem, mx, my, nx, ny, shift;
    int64_t pitch;
    const double* sspec;
    const int64_t* offset;
    const double* eta;
    const double* tx;
    const double* fx;
    const double* ty;
    const double* fy;
    const double* ax;
    const double* ay;
    double* image;
} sb_scatim;

int sb_scattered_image_f64(const sb_scatim* s, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SCINT_B200_SCATIM_H */
