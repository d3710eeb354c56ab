/* libscint_b200 -- C ABI of the CUDA-native scintools arc-measurement hot path.
 *
 * The reference (danielreardon/scintools) is pure Python and has no FFI; each
 * entry point below names the reference callable whose arithmetic it replaces
 * (file:line relative to the reference checkout).  INTEGRATION.md shows the
 * ctypes binding a scintools maintainer would add.
 *
 * Conventions
 *  - every function returns 0 on success, <0 on failure (sb_last_error()
 *    holds the message); nothing throws, nothing is printed;
 *  - pointers are DEVICE pointers unless the parameter name ends in _host;
 *    buffers are caller owned; `stream` is a cudaStream_t passed as void*;
 *  - 2-D arrays are C-contiguous (row-major); complex = interleaved
 *    (re, im) float pairs; dyn is [freq][time] like Dynspec.dyn;
 *  - one CUDA context per process, calls into one device from one host
 *    thread at a time (the library keeps a grow-only scratch workspace and
 *    twiddle tables per process; sb_release() frees them).  Not fork-safe
 *    (CUDA is not).
 *  - calls may use different streams.  The library orders each call after the
 *    previous one: a call on another stream than the previous call's waits on
 *    the device for that call's work, so the shared workspace never sees two
 *    calls at once.  sb_convert_* touch only caller buffers and are not ordered.
 *  - sm_90a (H100) only; there is no CPU fallback.
 */
#ifndef SCINT_B200_H
#define SCINT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_ERR_CUDA (-1)
#define SB_ERR_ARG (-2)
#define SB_ERR_NOMEM (-3)
#define SB_ERR_UNSUPPORTED (-4)

/* per-eta status bits written by sb_eta_sweep */
#define SB_ETA_OK 0
#define SB_ETA_INDEX_ERROR 1   /* numpy would raise IndexError -> NaN (ththmod.py:795-799) */
#define SB_ETA_ZERO_START 2    /* start row all zero -> NaN v0 -> ARPACK error -> NaN */
#define SB_ETA_TOO_SMALL 4     /* cropped matrix smaller than 3x3 -> eigsh raises -> NaN */
#define SB_ETA_NOT_CONVERGED 8 /* Lanczos hit max_iter; best Ritz value returned */

int sb_abi_version(void);
const char* sb_last_error(void);
/* select device, create the context, query SM count. */
int sb_init(int device);
/* free the scratch workspace. */
int sb_release(void);

/* Per-kernel timing with CUDA events recorded on the launching stream.
 * Slots: 0 cs_rows 1 cs_colA 2 cs_colB 3 thth_prep 4 thth_build 5 thth_eig
 * 6 sspec 7 acf 8 sim_screen 9 sim_freq 10 mosaic_tile 11 mosaic_reduce
 * 12 svd_gram (one A^T A pass of sb_svd_topk) 13 svd_apply 14 slow_ft_doppler (the three
 * column transforms of sb_slow_ft_f32) 15 slow_ft_delay (its row transform).
 * sb_profile_collect synchronises the
 * device, writes accumulated milliseconds and launch counts (host arrays of
 * at least 16 entries) and resets the accumulators. */
/* number of kernels this library has launched so far in this process */
int64_t sb_launch_count(void);
int sb_profile_enable(int32_t on);
int sb_profile_collect(double* ms_host, int32_t* count_host, int32_t n);

/* ---- theta-theta ------------------------------------------------------- */

/* Geometry of a conjugate spectrum + theta grid.  Scalars are the
 * reference's own numpy expressions evaluated by the host layer
 * (scintools/ththmod.py:83-97,153-156):
 *   tau0 = tau[0]; dtau = np.diff(tau).mean(); tau_absmax = abs(tau.max())
 *   fd0  = fd[0];  dfd  = np.diff(fd).mean();  fd_half = abs(fd.max())/2
 *   th_cents = recentred bin centres of `edges` (device, float64, n of them)
 */
typedef struct sb_thth_geom {
    const void* cs;        /* float2 conjugate spectrum, rows fftshifted (see cs_half) */
    int64_t ntau, nfd;     /* logical size: len(tau), len(fd) */
    double tau0, dtau, tau_absmax;
    double fd0, dfd, fd_half;
    const double* th_cents;      /* device */
    const double* th_cents_host; /* same values on the host */
    int32_t n_th;
    int32_t coherent;      /* 1: complex CS; 0: |CS| (ththmod.py:801) */
    int64_t cs_pitch;      /* elements per stored row (nfd for a plain full array) */
    int32_t cs_half;       /* 0: full fftshifted [ntau][nfd].  1: Hermitian half as
                              written by sb_cs_f32(half_plane=1): [ntau][cs_pitch],
                              columns k = 0..nfd/2 are the NON-shifted fd >= 0 bins;
                              the rest follows from CS[-tau,-fd] = conj(CS[tau,fd])
                              (valid for the CS of a real dynamic spectrum) */
    int32_t cs_valid_cols; /* cs_half only: how many of the nfd/2+1 stored columns hold data
                              (sb_cs_f32 with ncols_keep > 0 computes only those the theta
                              grid can reach); 0 = all.  Nothing beyond is ever read. */
    const float* cs_bound; /* device scalar: an upper bound of max |re|, |im| over the CS
                              (sb_cs_bound_f32), or NULL -> the sweep scans the CS itself.
                              Only used to scale the fp16 iteration copy of the matrices. */
} sb_thth_geom;

/* Replaces the eta loop of ththmod.single_search (ththmod.py:789-811) /
 * Dynspec.thetatheta_single (dynspec.py:1587-1600), i.e. neta calls of
 * ththmod.Eval_calc (ththmod.py:371-401 -> thth_redmap :119-173 -> thth_map
 * :56-116 -> scipy eigsh(k=1, which="LA")).
 * etas: device float64[neta].  Outputs (device): eigs float64[neta] (NaN where
 * the reference would have produced NaN), status int32[neta] (SB_ETA_*),
 * nred int32[neta] (size of the cropped matrix), iters int32[neta].
 * tol: relative residual tolerance of the Lanczos solve (<=0 -> 2e-5);
 * max_iter: <=0 -> 256. */
int sb_eta_sweep(const sb_thth_geom* geom, const double* etas, int32_t neta,
                 double tol, int32_t max_iter, double* eigs, int32_t* status,
                 int32_t* nred, int32_t* iters, void* stream);

/* Replaces ththmod.thth_map (ththmod.py:56-116) for one eta.  Any output may
 * be NULL.  thth: float2 [n][n]; tau_inv / fd_inv: int32 [n][n]
 * (ththmod.py:94-97, bit exact); pnts: uint8 [n][n] (ththmod.py:100);
 * th_pnts: uint8 [n] crop mask of thth_redmap (ththmod.py:153-156);
 * err: int32[1], SB_ETA_INDEX_ERROR if numpy would have raised. */
int sb_thth_map(const sb_thth_geom* geom, double eta, int32_t hermitian,
                void* thth, int32_t* tau_inv, int32_t* fd_inv, uint8_t* pnts,
                uint8_t* th_pnts, int32_t* err, void* stream);

/* "Thin" (arclet) theta-theta: replaces the eta loop of
 * ththmod.single_search_thin (scintools/ththmod.py:589-627), i.e. neta calls of
 * ththmod.singularvalue_calc (:496-512 -> two_curve_map :1557-1636 ->
 * numpy.linalg.svd, S[0]).  geom describes the CS and the theta1 (column) grid
 * with THIS path's conventions: th_cents = (edges1[1:]+edges1[:-1])/2 (not
 * recentred), tau0 = tau[1], fd0 = fd[1] (ththmod.py:1602-1604), tau_absmax =
 * tau.max(), fd_half unused.  th2_cents: device float64 [n_th2], centres of
 * the arclet grid (rows).  eta1 / eta2: device float64 [neta] (main-arc and
 * arclet curvature per trial).  center_cut: columns with |theta1| < center_cut
 * are zeroed.  power=1 gathers |CS|^2 (incoherent thin search, :609).
 * Outputs: svals float64 [neta] (NaN where numpy would raise), status (SB_ETA_*
 * bits), n1_red / n2_red (cropped sizes), iters.  Pairs run in batches whose
 * matrices fit the 3 GiB budget of sb_eta_sweep (SB_SWEEP_SLAB_MB overrides it). */
int sb_thin_sweep(const sb_thth_geom* geom, const double* th2_cents, int32_t n_th2,
                  double center_cut, int32_t power, const double* eta1, const double* eta2,
                  int32_t neta, double tol, int32_t max_iter, double* svals,
                  int32_t* status, int32_t* n1_red, int32_t* n2_red, int32_t* iters,
                  void* stream);

/* Uncropped two-curvature map thth [n_th2][n_th] (float2) of
 * ththmod.two_curve_map (:1585-1617) for one (eta1, eta2); err as sb_thth_map. */
int sb_thin_map(const sb_thth_geom* geom, const double* th2_cents, int32_t n_th2,
                int32_t power, double eta1, double eta2, void* thth, int32_t* err,
                void* stream);

/* ---- phase retrieval (SURVEY 8f rank 1) ----------------------------------- */

/* ththmod.rev_map (scintools/ththmod.py:176-258): scatter the n x n theta-theta
 * matrix thth (float2, row-major, device) back into the conjugate spectrum
 * recov [ntau][nfd] (float2, = the reference's recov.T).  Bins are those of
 * np.histogram2d with edges (k - 0.5) * d + x0, bit-exact (x0 = tau[0] / fd[0],
 * d = tau[1]-tau[0] / fd[1]-fd[0], both > 0); weights 1/sqrt|2 eta dtheta|; bin
 * means; empty bins and the (0, 0) bin (zero Jacobian -> NaN -> nan_to_num) are 0.
 * hermitian != 0 also adds the conjugate at (-fd, -tau) (:229-256).
 * th_cents: float64 [n] on the device, already centred as in :208-209. */
int sb_rev_map(const void* thth, int32_t n, const double* th_cents, double eta, double tau0,
               double dtau, int32_t ntau, double fd0, double dfd, int32_t nfd,
               int32_t hermitian, void* recov, void* stream);

/* Largest-algebraic eigenpair of a full Hermitian float2 matrix a [n][ld] on
 * the device: eigsh(thth_red, 1, which='LA') in ththmod.modeler (:300-307).
 * w: float64 [1], v: float2 [n] (unit norm, arbitrary global phase like ARPACK),
 * info: int32 [2] = {lanczos steps, status (SB_ETA_* bits)}.  tol: residual
 * bound relative to w (<= 0: 1e-7); max_iter <= 0: 96. */
int sb_herm_eigvec(const void* a, int32_t n, int32_t ld, double tol, int32_t max_iter,
                   double* w, void* v, int32_t* info, void* stream);

/* Replaces the curvature loop of the chi-square search (scintools/examples/
 * THTHSample.ipynb, "Chisquared Search"), i.e. neta calls of ththmod.chisq_calc
 * (:330-368 -> modeler :261-327 hermitian branch -> thth_redmap, eigsh(k=1,
 * which='LA'), rev_map of |w| V V^H, ifft2(ifftshift(recov)).real), without the
 * division by N:
 *   ssq[e] = sum over mask of (model_e[:nf, :nt] - dspec)^2   (float64).
 * geom: as sb_eta_sweep (full or half-plane CS, coherent), etas: device float64
 * [neta].  th_red: device float64 [neta][n_th], row e holding the nred[e]
 * rev_map centres of curvature e (theta_centres of its edges_red,
 * ththmod.py:204-205), evaluated by the host with the reference's expressions.
 * dtau_bin = tau[1] - tau[0], dfd_bin = fd[1] - fd[0]: the histogram bin widths
 * of rev_map (:210-215; tau[0] and fd[0] come from geom).  dspec: float32
 * [nf][nt] with nf <= ntau, nt <= nfd; mask: uint8 [nf][nt] (non-zero = use)
 * or NULL for isfinite(dspec).  tol (<= 0: 1e-7) and max_iter (<= 0: 96) as
 * sb_herm_eigvec.  The eigenpair Lanczos starts from row n//2; if that row is
 * zero it starts from a fixed non-zero vector (eigsh starts from a random one).
 * Outputs (device, [neta] each): ssq float64 (NaN where chisq_calc raises:
 * status bits SB_ETA_INDEX_ERROR, SB_ETA_ZERO_START = the matrix is zero --
 * ARPACK's "starting vector is zero" --, SB_ETA_TOO_SMALL); w float64 (top
 * eigenvalue, NaN for INDEX_ERROR / TOO_SMALL, 0 for a zero matrix); status
 * (SB_ETA_* bits; SB_ETA_NOT_CONVERGED keeps its ssq); nred (cropped size);
 * iters (Lanczos steps).  Curvatures run in batches whose buffers (matrix,
 * Lanczos basis and a few CS-sized arrays per curvature) fit the 3 GiB budget
 * of sb_eta_sweep (SB_SWEEP_SLAB_MB overrides it).  Errors: SB_ERR_ARG if dspec
 * is larger than the CS; SB_ERR_UNSUPPORTED for more than 4096 theta centres
 * or CS sizes outside those of sb_ifft2_c2c_f32. */
int sb_chisq_sweep(const sb_thth_geom* geom, const double* etas, int32_t neta,
                   const double* th_red, double dtau_bin, double dfd_bin, const float* dspec,
                   int32_t nf, int32_t nt, const uint8_t* mask, double tol, int32_t max_iter,
                   double* ssq, double* w, int32_t* status, int32_t* nred, int32_t* iters,
                   void* stream);

/* out[:crop0, :crop1] = scale * ifft2(ifftshift(in)) (centred != 0) or
 * scale * ifft2(in), in: float2 [n0][n1] (ththmod.py:321, :1462-1465).  Powers of two
 * up to 65536 x 16384 (n0 x n1, both >= 8) take the radix path; any other size up to
 * 32768 x 8192 runs a chirp-z transform.  real_only != 0 writes float (the real
 * part), else float2.  crop <= 0: full. */
int sb_ifft2_c2c_f32(const void* in, int32_t n0, int32_t n1, int32_t centred, int32_t crop0,
                     int32_t crop1, double scale, int32_t real_only, void* out, void* stream);

/* The loop of Dynspec.gerchberg_saxton (scintools/dynspec.py:1883-1896), niter
 * times, in place on wavefield (float2 [n0][n1]; sizes as sb_ifft2_c2c_f32: powers of
 * two up to 65536 x 16384, iterated in fp64 when n1 <= 8192; other sizes up to
 * 32768 x 8192 through the fp32 chirp-z transform):
 *   CWF = fft2(w); CWF[rowmask != 0, :] = 0; w = ifft2(CWF);
 *   w = amp * exp(i angle(w)) where amp is not NaN.
 * rowmask: uint8 [n0] over the UNSHIFTED delay rows (1 where tau < 0);
 * amp: float [n0][n1] = sqrt(dyn) where dyn is finite and > 0, NaN elsewhere. */
int sb_gerchberg_saxton_f32(void* wavefield, const float* amp, const uint8_t* rowmask,
                            int32_t n0, int32_t n1, int32_t niter, void* stream);

/* ---- Dynspec 2-D FFT paths ---------------------------------------------- */

/* Dynspec.scale_dyn(scale='lambda')
 * (scintools/dynspec.py:3926-3957): not-a-knot cubic spline of every time
 * column of dyn [nf][nt] at nlam query frequencies, written flipped
 * (out [nlam][nt], wavelength ascending).  The column-independent tables are
 * built by the host (scintools_b200/dynspec.py::_spline_tables, fp64 -> fp32):
 * a, cp, inv, g: float [nf] Thomas factors of the second-derivative system,
 * p0, pn: not-a-knot end ratios, idx: int32 [nlam] interval of each query,
 * w4: float [nlam][4] weights of (y_i, y_i+1, M_i, M_i+1).  flip_rows != 0 when
 * the frequency axis of dyn is descending. */
int sb_scale_dyn_lambda_f32(const float* dyn, int32_t nf, int32_t nt, int32_t flip_rows,
                            const float* a, const float* cp, const float* inv, const float* g,
                            float p0, float pn, const int32_t* idx, const float* w4,
                            int32_t nlam, float* out, void* stream);

/* Dynspec.norm_sspec, the resampling loop (scintools/dynspec.py:2076-2107) and
 * self.powerspectrum (:2120): row ii of the secondary spectrum sspec [nr][nc] (dB,
 * already cropped / masked by the caller like :2040-2046) is resampled with
 * numpy.interp at the nq normalised Doppler values fdopnew[] on the axis
 * fdop / sqrt(tdel[ii] / eta) restricted to |fdop| <= maxnormfac * sqrt(tdel[ii]/eta).
 * out: float [nr][nq], NaN where the reference's mask is set (|fdopnew| beyond the
 * row's reach, or a NaN sample); power: double [nr] = masked mean of 10^(out/10).
 * fdop [nc], tdel [nr], fdopnew [nq]: device float64 (the reference's own axes). */
int sb_norm_sspec_f32(const float* sspec, int32_t nr, int32_t nc, const double* fdop,
                      const double* tdel, double eta, double maxnormfac,
                      const double* fdopnew, int32_t nq, float* out, double* power,
                      void* stream);

/* Delay-scrunched profile of Dynspec.norm_sspec (scintools/dynspec.py:2159-2166):
 * avg[j] = sum_ii w[ii] norm[ii][j] / sum_ii w[ii] over the unmasked (non-NaN)
 * entries of column j (np.ma.average(normSspec, axis=0, weights=w)); NaN where a
 * column is fully masked.  This is fit_arc's power-vs-curvature profile (:1156-1180). */
int sb_norm_sspec_avg_f32(const float* norm, int32_t nr, int32_t nq, const double* weights,
                          double* avg, void* stream);

/* Replaces the arithmetic of Dynspec.calc_sspec (scintools/dynspec.py:3664-3721):
 *   x = win_t[t]*win_f[f]*(dyn - mean(dyn)); x -= mean(x); [prewhite: 2x2
 *   first difference]; |FFT2 zero-padded to nrfft x ncfft|^2; fftshift;
 *   [halve: keep tau >= 0]; [postdark]; [10 log10].
 * nrfft = 2^(ceil(log2 nf)+1), ncfft likewise (dynspec.py:3677-3678).
 * dyn: float32 [nf][nt].  win_t [nt] / win_f [nf]: tapers from
 * scint_utils.get_window (scint_utils.py:810-832) or both NULL (window=None);
 * sum_win_*: their sums.  pd_fd [ncfft], pd_td [nrfft/2]: the sin^2 post-darken
 * vectors of dynspec.py:3706-3711 (only read when prewhite).  sec: float32
 * [nrfft/2 or nrfft][ncfft]; db=0 returns linear power. */
int sb_sspec_f32(const float* dyn, int32_t nf, int32_t nt, const float* win_t,
                 const float* win_f, double sum_win_t, double sum_win_f,
                 int32_t prewhite, int32_t halve, int32_t db, const float* pd_fd,
                 const float* pd_td, float* sec, void* stream);

/* Replaces Dynspec.calc_acf(method='direct') (scintools/dynspec.py:3780-3797):
 * real(fftshift(ifft2(|fft2(dyn - mean(valid), [2nf, 2nt])|^2))) [/ max].
 * acf: float32 [2nf][2nt].  subtract_mean=0 reproduces the input_dyn branch
 * (dynspec.py:3786-3789).  nf 2..32768, nt 5..16384, not only powers of two: the
 * transform runs on the next power of two and the lags [-nf,nf) x [-nt,nt) are
 * extracted (identical by the correlation theorem).  The normalisation divides by
 * the zero-lag value, which is the maximum of an autocovariance. */
int sb_acf_f32(const float* dyn, int32_t nf, int32_t nt, int32_t subtract_mean,
               int32_t normalise, float* acf, void* stream);

/* Replaces Dynspec.calc_acf(method='sspec') (scintools/dynspec.py:3798-3807):
 * real(fftshift(fft2(linear un-halved secondary spectrum))) [/ max], with the
 * window arguments of sb_sspec_f32.  acf: float32 [nrfft][ncfft]. */
int sb_acf_sspec_f32(const float* dyn, int32_t nf, int32_t nt, const float* win_t,
                     const float* win_f, double sum_win_t, double sum_win_f,
                     int32_t normalise, float* acf, void* stream);

/* Replaces the tile loop of Dynspec.cut_dyn (scintools/dynspec.py:3158-3271): the
 * secondary spectrum of every tile, each exactly as sb_sspec_f32 with halve=1, db=1,
 * prewhite=0 would make it from that tile alone.  The parent dyn: float32 [nf][nt] (row
 * pitch nt); tile (ii, jj), ii < nfc, jj < ntc, is dyn[ii*fnum + f][jj*tnum + t]
 * (f < fnum, t < tnum), so nfc*fnum <= nf and ntc*tnum <= nt.  win_t [tnum] / win_f
 * [fnum]: the tile's tapers (scint_utils.get_window of the tile size) or both NULL;
 * sum_win_*: their sums.  sec: float32 [nfc][ntc][nrfft/2][ncfft] with nrfft, ncfft of
 * sb_sspec_f32 for an fnum x tnum spectrum.  Each tile's means are its own: a NaN makes its
 * own tile NaN and no other.  fnum 2..32768, tnum 5..16384 (SB_ERR_UNSUPPORTED otherwise);
 * any number of tiles, run in groups whose workspace fits a fixed 1 GiB (one tile at least). */
int sb_sspec_tiles_f32(const float* dyn, int32_t nf, int32_t nt, int32_t fnum, int32_t tnum,
                       int32_t nfc, int32_t ntc, const float* win_t, const float* win_f,
                       double sum_win_t, double sum_win_f, float* sec, void* stream);

/* The ACFs of the tiles of sb_sspec_tiles_f32 (same dyn, nf, nt, fnum, tnum, nfc, ntc),
 * each as sb_acf_f32(subtract_mean=0, normalise=1) makes it from that tile alone, i.e.
 * Dynspec.calc_acf(input_dyn=tile): acf float32 [nfc][ntc][2 fnum][2 tnum], every tile
 * divided by its own zero-lag value.  Limits and grouping as sb_sspec_tiles_f32. */
int sb_acf_tiles_f32(const float* dyn, int32_t nf, int32_t nt, int32_t fnum, int32_t tnum,
                     int32_t nfc, int32_t ntc, float* acf, void* stream);

/* Replaces the CS stage of ththmod.single_search (scintools/ththmod.py:777-787)
 * and Dynspec.thetatheta_single (scintools/dynspec.py:1572-1579):
 *   CS = fftshift(fft2(pad(dspec, npad copies, constant pad_value)));
 *   CS[tau_rowmask] = 0
 * pad_value = NaN pads with the mean of dspec computed on the device
 * (constant_values=dspec2.mean(), ththmod.py:781) without a host pass.
 * dspec float32 [nf][nt]; cs: float2 [(npad+1)nf][(npad+1)nt]; tau_rowmask:
 * uint8 [(npad+1)nf] (1 = zero that fftshifted row) or NULL.  half_plane=1
 * writes only the fd >= 0 half, [(npad+1)nf][cs_pitch] with cs_pitch >=
 * (npad+1)nt/2 + 1 (see sb_thth_geom.cs_half): half the HBM traffic, and all
 * the theta-theta sweep needs.  half_plane=0: full array, cs_pitch ignored.
 * ncols_keep > 0 (half-plane only): compute just the first ncols_keep fd >= 0
 * columns; the others are left untouched.  The sweep gathers at
 * fd = theta_j - theta_i <= max(theta) - min(theta), so a caller that knows
 * its theta grid can skip the columns beyond that (the column passes dominate
 * the transform).  0 = all nfd/2 + 1 columns.
 * Power-of-two padded sizes take the direct radix-16 path (rows <= 65536, cols
 * <= 32768); any other size runs a chirp-z (Bluestein) transform on both axes
 * (rows 3..32768, cols 3..8192, half_plane must be 0). */
int sb_cs_f32(const float* dspec, int32_t nf, int32_t nt, int32_t npad,
              float pad_value, const uint8_t* tau_rowmask, int32_t half_plane,
              int64_t cs_pitch, int32_t ncols_keep, void* cs, void* stream);

/* Upper bound of max |CS| for the conjugate spectrum sb_cs_f32 makes from the same
 * (dspec, nf, nt, npad, pad_value): sum |dspec - c| + |c| (npad+1)^2 nf nt with c the
 * padding constant (the mean when pad_value is NaN) -- the L1 norm bounds every Fourier
 * coefficient.  One pass over dspec.  bound_out: device float.  Feeds
 * sb_thth_geom.cs_bound (the eigen solver's fp16 scale); a loose bound is fine. */
int sb_cs_bound_f32(const float* dspec, int32_t nf, int32_t nt, int32_t npad, float pad_value,
                    float* bound_out, void* stream);

/* Conjugate spectrum of a COMPLEX chunk vis (float2 [nf][nt], e.g. a VLBI
 * visibility, ththmod.py:1313-1325): pad to (npad+1) nf x (npad+1) nt with
 * pad_re + i pad_im (pad_re NaN: the mean of vis, computed on the device),
 * fft2, fftshift both axes, zero the rows where tau_rowmask (uint8 [ntau],
 * fftshifted order, or NULL) is set.  cs: float2 [ntau][nfd], always the full
 * plane.  Padded sizes that are powers of two in 8..65536 x 8..16384 take the
 * radix path (a complex row is one transform of nfd points, so the column limit
 * is half that of sb_cs_f32); any other size in 3..32768 x 3..8192 runs a
 * chirp-z transform.  Other sizes: SB_ERR_UNSUPPORTED. */
int sb_cs_c2c_f32(const void* vis, int32_t nf, int32_t nt, int32_t npad, float pad_re,
                  float pad_im, const uint8_t* tau_rowmask, void* cs, void* stream);

/* One chunk of ththmod.VLBI_chunk_retrieval (:1223-1387), steps after the
 * conjugate spectra, with no host synchronisation.  cs_list_host: host array of
 * n_dish (n_dish+1)/2 device pointers to full-plane float2 [ntau][nfd] spectra in
 * the reference's order [I1, V12, .., V1N, I2, V23, .., IN]; geom supplies the
 * axes and the theta grid (cs_half must be 0; cs, cs_pitch, cs_valid_cols,
 * cs_bound and coherent are not read: every spectrum is dense and complex).
 *   - every spectrum is cropped and gathered with thth_redmap's rules (autos
 *     hermetian=True, visibilities hermetian=False) straight into the composite
 *     [n_dish n][n_dish n] matrix, n = the cropped size: block (d1, d1+d2) =
 *     conj(T).T, block (d1+d2, d1) = T (:1342-1362);
 *   - top eigenpair (w, V) as sb_herm_eigvec, starting from the sum of row n//2
 *     of every station's block row (one row alone would keep Lanczos inside one
 *     station's block when the visibilities are zero), or from a fixed vector if
 *     that sum is zero;
 *   - per station d: rev_map(hermetian=False) of the n x n matrix whose row n//2
 *     is conj(V[d n:(d+1) n]) sqrt(w), ifft2(ifftshift(.))[:nf, :nt] nf nt / 4.
 * th_red: device float64 [n], the rev_map centres (theta_centres of edges_red);
 * dtau_bin, dfd_bin: as sb_chisq_sweep.  tol / max_iter as sb_herm_eigvec.
 * Outputs (device): model_e float2 [n_dish][nf][nt]; w float64 [1] (NaN for
 * SB_ETA_INDEX_ERROR / SB_ETA_TOO_SMALL, 0 for an all-zero composite with
 * SB_ETA_ZERO_START); v float2 [n_dish n]; info int32 [3] = {Lanczos steps,
 * SB_ETA_* status, n}.  A failed eigenpair leaves model_e zero.
 * Errors: SB_ERR_ARG for n_dish < 1, nf > ntau, nt > nfd or a null spectrum;
 * SB_ERR_UNSUPPORTED for n_dish n > 8192 or CS sizes outside those of
 * sb_ifft2_c2c_f32.  Sizes are checked before any workspace is allocated. */
int sb_vlbi_retrieval(const sb_thth_geom* geom, const void* const* cs_list_host, int32_t n_dish,
                      double eta, const double* th_red, double dtau_bin, double dfd_bin,
                      int32_t nf, int32_t nt, double tol, int32_t max_iter, void* model_e,
                      double* w, void* v, int32_t* info, void* stream);

/* ththmod.calc_asymmetry (:2385-2463) for nchunk chunks after their conjugate
 * spectra (made by sb_cs_f32 with the chunk's mean as pad value; no tau mask),
 * i.e. the chunk loop of Dynspec.calc_asymmetry (dynspec.py:1892-1918), in one
 * launch sequence with no host synchronisation.  geoms_host: host array of
 * nchunk geometries, one per chunk, each with its own cs, delay / Doppler axes
 * and theta grid (th_cents and th_cents_host); all of them share ntau, nfd,
 * n_th and the spectrum layout (cs_half, cs_pitch, cs_valid_cols, coherent),
 * else SB_ERR_ARG.  etas: device float64 [nchunk].  Per chunk:
 *   - crop and gather of thth_redmap (hermetian=True), as sb_eta_sweep;
 *   - top eigenpair (w, V) as sb_herm_eigvec, one thread block per chunk,
 *     starting from row n//2 or, if that row is zero, from a fixed vector;
 *   - with m = nred and h = (m - 1) // 2, in float64:
 *     asym = (sum |V[:h]|^2 - sum |V[h+1:]|^2) / (sum |V[:h]|^2 + sum |V[h+1:]|^2).
 * Outputs (device, [nchunk] each): asym float64 (NaN where the reference's
 * try/except gives NaN: status bits SB_ETA_INDEX_ERROR, SB_ETA_ZERO_START (a
 * zero matrix), SB_ETA_TOO_SMALL (fewer than 3 centres), SB_ETA_NOT_CONVERGED;
 * 0 / 0 is NaN); w float64 (NaN for INDEX_ERROR / TOO_SMALL, 0 for a zero
 * matrix); status (SB_ETA_* bits); nred (cropped size); iters (Lanczos steps);
 * v float2 [nchunk][ld], ld = n_th rounded up to a multiple of 32, or NULL:
 * each chunk's unit eigenvector (arbitrary global phase) zero-padded to ld,
 * zeros where none was computed.  tol (<= 0: 1e-7) and max_iter (<= 0: 96) as
 * sb_herm_eigvec.  Chunks run in batches whose matrix, Lanczos basis and vector
 * fit the 3 GiB budget of sb_eta_sweep (SB_SWEEP_SLAB_MB overrides it).
 * Limits, checked before any workspace is allocated: n_th <= 4096
 * (SB_ERR_UNSUPPORTED); spectra of the sizes sb_cs_f32 makes: powers of two in
 * 4..65536 x 16..32768 (full or half plane), other sizes in 3..32768 x 3..8192
 * (full plane only). */
int sb_asymmetry_batch(const sb_thth_geom* geoms_host, int32_t nchunk, const double* etas,
                       double tol, int32_t max_iter, double* asym, double* w, int32_t* status,
                       int32_t* nred, int32_t* iters, void* v, void* stream);

/* ---- wavefield mosaic ---------------------------------------------------- */

/* ththmod.rotMos / rotFit / rotDer / rotInit and fullMos / fullMosFit /
 * fullMosGrad / fullMosHess (:1708-2310) for ncf x nct half-overlapping chunks
 * of cwf x cwt: chunks float2 [ncf*nct][cwf][cwt], chunk k = cf*nct + ct covers
 * mosaic rows cf*(cwf/2) .. +cwf and columns ct*(cwt/2) .. +cwt, weighted by the
 * separable sin^2 ramps of mask_func.  The mosaic is nF x nT =
 * ((ncf-1)*(cwf/2)+cwf) x ((nct-1)*(cwt/2)+cwt).  phi: device float64 [P]
 * phases per chunk (phi[0] is the first chunk's, 0 in the reference); amp:
 * device float64 [P] amplitudes or NULL (ones, sb_mosaic_build only).  e^{i phi}
 * is formed in float64 per chunk; pixels are float32 arithmetic, every sum is
 * accumulated in float64 in a fixed order (results are deterministic).
 * Limits, checked before any workspace is allocated: an axis with more than one
 * chunk needs an even width (SB_ERR_ARG); half-tile extents (cwf/2, or cwf for a
 * single chunk; the same in time) <= 2048, mosaic sides < 2^31 and fewer than
 * 2^28 chunks (SB_ERR_UNSUPPORTED). */

/* wavefield float2 [nF][nT] = sum_k amp_k e^{i phi_k} mask_k chunk_k */
int sb_mosaic_build(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                    const double* phi, const double* amp, void* wavefield, void* stream);
/* from the wavefield sb_mosaic_build made with the same phi and amp = NULL:
 * power float64 [1] = sum |W|^2 (rotFit = -power), der float64 [P] with
 * der[k] = 2 sum Im(conj(W) e^{i phi_k} mask_k chunk_k) (rotDer[k-1] = der[k]).
 * NaN propagates. */
int sb_mosaic_rot(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                  const double* phi, const void* wavefield, double* power, double* der,
                  void* stream);
/* overlap float64 complex [P][4]: overlap[k][e] = sum over the overlap of
 * mask_j chunk_j conj(mask_k chunk_k) with the earlier neighbour j of chunk
 * (cf, ct) at e = 0 (cf-1, ct-1), 1 (cf-1, ct), 2 (cf-1, ct+1), 3 (cf, ct-1);
 * 0 where there is none.  rotInit is then rot_k = angle(sum_e e^{i rot_j} overlap[k][e]). */
int sb_mosaic_overlap(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                      double* overlap, void* stream);
/* from the wavefield sb_mosaic_build made with the same phi and amp, dspec and
 * noise float32 [nF][nT]: fit float64 [1] = sum ((|W|^2 - dspec) / noise)^2 and
 * grad float64 [P][2] = (d fit / d amp_k, d fit / d phi_k), NaN terms skipped
 * (numpy nansum; a complex gradient term is skipped if either part is NaN). */
int sb_mosaic_fit(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                  const double* phi, const double* amp, const void* wavefield, const float* dspec,
                  const float* noise, double* fit, double* grad, void* stream);
/* Hessian of that fit as COO triplets, 8 per (chunk, forward neighbour) slot,
 * rows / cols int64 and vals float64 of 40 P entries each.  Parameter index
 * of phi_k is k-1 (k >= 1), of amp_k is k+P-1 (fullMosHess's p layout); every
 * (row, col) appears at most once; unused slots have row = col = -1.  Sums
 * over each pair's overlap; NaN propagates (numpy sum). */
int sb_mosaic_hess(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                   const double* phi, const double* amp, const void* wavefield, const float* dspec,
                   const float* noise, int64_t* rows, int64_t* cols, double* vals, void* stream);

/* ---- flux-variation correction ------------------------------------------ */

/* Dynspec.correct_dyn (dynspec.py:3325-3410) and svd_model (scint_utils.py:705-729,
 * ththmod.py:18-35).  A: device float32 [nf][nt], NaN read as 0.  Shapes: 1 <= nf <=
 * 32768, 1 <= nt <= 16384, else SB_ERR_UNSUPPORTED; 1 <= k <= 32, else SB_ERR_ARG.
 * Every sum is float64 in a fixed order: repeated calls are bit-identical. */

/* Top-k right singular vectors of A: Lanczos on A^T A in float64 with full
 * re-orthogonalisation, one read of A per step, then one more read per mode for the true
 * residual (stopping rule in csrc/svd.cu).  Synchronous.  V: device float64 [k][nt]
 * (orthonormal; rows past the numerical rank are zero).  s_host [k]: singular values,
 * descending; res_host [k]: ||A^T A v_j - s_j^2 v_j||_2; gap_host [1]: the lower bound
 * theta_k - theta_{k+1} - r_{k+1} on the eigenvalue gap of A^T A the rule used (0 when the
 * iteration ended with at most k Ritz values); info_host int32 [4]: Lanczos steps,
 * converged (0/1), tie at the truncation boundary (0/1), exact breakdown (0/1). */
int sb_svd_topk(const float* A, int32_t nf, int32_t nt, int32_t k, double* V, double* s_host,
                double* res_host, double* gap_host, int32_t* info_host, void* stream);
/* Final pass, one read of A: model_ij = sum_j (a_i . v_j) v_j and out_ij = a_ij / |model_ij|
 * (float64, rounded once; 0/0 -> NaN, a/0 -> inf).  out or model may be NULL (not both). */
int sb_svd_apply(const float* A, int32_t nf, int32_t nt, int32_t k, const double* V, float* out,
                 float* model, void* stream);
/* svd=False passes.  A value is NaN if zero_as_nan and it is 0 (the host decides, from
 * whether the array is Dynspec.dyn itself); means skip NaN (numpy nanmean, NaN when no
 * value is left).  rows: mean float64 [nf] over each row.  cols: mean float64 [nt] over
 * each column of value / rowdiv[i] (rowdiv float64 [nf] or NULL).  divide: out float32
 * [nf][nt] = (value / rowdiv[i]) / coldiv[j] in float64 (either NULL: skipped). */
int sb_bandpass_rows(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan, double* mean,
                     void* stream);
int sb_bandpass_cols(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan,
                     const double* rowdiv, double* mean, void* stream);
int sb_bandpass_divide(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan,
                       const double* rowdiv, const double* coldiv, float* out, void* stream);

/* ---- frequency-scaled Doppler transform ----------------------------------- */

/* scint_utils.slow_FT (scint_utils.py:655-702, with its fftshift keyword read as axes=0).
 * x: device float32 [ntime][nfreq] (time-major); fscale: device float64 [nfreq], f / fref;
 * out: device float2 [ntime][nfreq].  With c = ntime / 2,
 *   out[m][j] = sum_f sum_t x[t][f] exp(-2 pi i fscale[f] t (m - c) / ntime)
 *                                   exp(-2 pi i f (j - nfreq/2) / nfreq).
 * Shapes 1..32768 x 1..8192, else SB_ERR_UNSUPPORTED.  A non-finite x or fscale makes
 * every output non-finite.  Asynchronous on `stream`; no atomics, so repeated calls are
 * bit-identical.  Device memory: two grow-only workspace planes of M x nfreq complex64
 * (M = 2^ceil(log2(2 ntime - 1)), at least 8), 8 GiB at 32768 x 8192; a nfreq that is not
 * a power of two >= 8 adds ntime x MT complex64 (MT = 2^ceil(log2(2 nfreq - 1))), at most
 * 4 GiB.  The workspace stays allocated until sb_release. */
int sb_slow_ft_f32(const float* x, int32_t ntime, int32_t nfreq, const double* fscale, void* out,
                   void* stream);

/* ---- gap filling ---------------------------------------------------------- */

/* Dynspec.refill (dynspec.py:3273-3323), method='biharmonic': the inpainting of
 * skimage.restoration.inpaint_biharmonic (split_into_regions=False), solved on the device.
 * img: device float64 [nf][nt], read only at known pixels; pix: device int32 [n], the
 * masked pixels (flat row-major indices, ascending, 1 <= n <= nf nt).  Row k of the system
 * is S = laplace(laplace(e_p)) (scipy.ndimage, mode 'reflect') on the 5x5 box around pix[k]
 * clipped to the image; masked neighbours are unknowns, known ones go to the right-hand
 * side.  The caller supplies the stencils: rcls uint8 [nf] and ccls uint8 [nt] give each
 * row's / column's class (< nrc, < ncc, both <= 5), tables float64 [nrc][ncc][5][5] the
 * stencil of each class pair centred on the pixel, zero outside the clipped box.
 * Matrix-free BiCGSTAB with Jacobi scaling in float64 stops when ||b - A x|| <= tol ||b||
 * (true residual) or after maxit steps; out: device float64 [n] = clip(x, lo, hi).
 * info_host int32 [3]: steps, converged (0/1), restarts; resid_host [1]: the final
 * ||b - A x|| / ||b||.  Synchronous (the host reads the state every 32 steps).  Shapes
 * 1..32768 x 1..16384, else SB_ERR_UNSUPPORTED.  Fixed-order sums: repeated calls are
 * bit-identical.  Workspace: 11 n + 3 maxit doubles and an nf x nt int32 map. */
int sb_inpaint_biharmonic_f64(const double* img, int32_t nf, int32_t nt, const int32_t* pix,
                              int32_t n, const double* tables, const uint8_t* rcls, int32_t nrc,
                              const uint8_t* ccls, int32_t ncc, double lo, double hi, double tol,
                              int32_t maxit, double* out, int32_t* info_host, double* resid_host,
                              void* stream);
/* Dynspec.refill(method='median'): out[k] = scipy.signal.medfilt(img', (kh, kw))[pix[k]],
 * img' = img with NaN read as nan_value, zero padding outside the image; kh, kw odd, at
 * most 31 (else SB_ERR_ARG / SB_ERR_UNSUPPORTED).  Exact (a median is one of the inputs).
 * img float64 [nf][nt], pix int32 [n], out float64 [n], all on the device.  Shapes as
 * sb_inpaint_biharmonic_f64. */
int sb_medfilt_masked_f64(const double* img, int32_t nf, int32_t nt, const int32_t* pix, int32_t n,
                          int32_t kh, int32_t kw, double nan_value, double* out, void* stream);

/* ---- Dynspec.get_scint_params ------------------------------------------- */

/* One least-squares fit of the ACF (host struct; the pointers are device memory).
 * Parameter slots 0..4: tau, dnu, amp, alpha, phasegrad; p0 holds every slot's starting
 * (or fixed) value, bit s of `vary` frees slot s, bit s of `bounded` fits it with min 0,
 * max inf in lmfit's internal variable.  acf: float64 ACF with row pitch `pitch`.
 *   1-D (sb_scint_fit_1d): time cut acf[r0][c0 .. c0 + n0), lags s0 * i (s0 = dt);
 *       frequency cut acf[r1 .. r1 + n1)[c1], lags s1 * i (s1 = df); aux [n0 + n1] the
 *       weights of both cuts (the weight of lag 0 of each is taken as 0).
 *   2-D (sb_scint_fit_2d): the box acf[r0 .. r0 + n0)[c0 .. c0 + n1) (frequency lag by
 *       time lag); s0 = tobs, s1 = bw, c = nsub nchan; aux [2 n1 + 2 n0]: tdata [n1],
 *       fdata [n0], T / max(tticks) [n1], F / max(fticks) [n0]; shf, sht, pf, pt, zf, zt
 *       place the weights (see csrc/scintfit.cu); weighted 0 or 1.
 * max_nfev caps the evaluations. */
typedef struct sb_scint_fit {
    const double* acf;
    const double* aux;
    int64_t pitch;
    double s0, s1, c;
    double p0[5];
    int32_t r0, c0, r1, c1, n0, n1;
    int32_t shf, sht, pf, pt, zf, zt;
    int32_t vary, bounded, weighted, max_nfev;
} sb_scint_fit;

/* Dynspec.get_scint_params (dynspec.py:2470-3156), the lmfit least-squares fits of
 * method='acf1d' (scint_acf_model, scint_models.py:62-120; replaces the fitter() call at
 * dynspec.py:2698-2702) and method='acf2d_approx' (scint_acf_model_2d_approx,
 * scint_models.py:123-161; replaces dynspec.py:2836-2841), batched over nfit fits with an
 * analytic float64 Jacobian.  fits: host [nfit].  out: device float64 [nfit][11]: the five
 * slots' values, their standard errors (NaN where not estimated: fixed, singular J^T J, or
 * not converged) and chi-square; info: device int32 [nfit][2]: evaluations and status (1
 * converged, 2 stopped with no decrease left at float64 precision, -1 hit max_nfev, -2 a
 * non-finite residual).  Synchronous (the host reads the state every 32 iterations).  A
 * fit's result is bit-identical alone or in any batch. */
int sb_scint_fit_1d(const sb_scint_fit* fits, int32_t nfit, double* out, int32_t* info,
                    void* stream);
int sb_scint_fit_2d(const sb_scint_fit* fits, int32_t nfit, double* out, int32_t* info,
                    void* stream);

/* ---- scint_sim.ACF ------------------------------------------------------- */

/* The analytic intensity ACF of scint_sim.ACF.calc_acf (scint_sim.py:494-678), in float64.
 * Device arrays, built on the host with the reference's numpy expressions: snp [n1] (main
 * grid), snp2 [n2] (core grid, used for dnun[1]), dnun [ndnun], snx and sny [nsn] (the time
 * lags' positions).  Scalars: sigxn, sigyn (the phase-gradient offsets), sqrtar = sqrt(ar),
 * alph2 = alpha / 2, step1 and step2 (the two grids' steps), wn_amp = wn / amp, amp.
 * quadrant != 0 for phasegrad == 0: nsn lags from 0 and the quadrant mirrored both ways,
 * wn_amp added at lag 0; else nsn lags across the full range, the half plane
 * point-reflected, wn_amp added where snx == 0 exactly.
 * Outputs (device): acf float64 [2 ndnun - 1][quadrant ? 2 nsn - 1 : nsn] = amp |gamma|^2;
 * efield float64 [n1][n1], the e-field ACF on the main grid (acf_efield).
 * Sizes: n1, n2 1..16384, ndnun 2..4096, nsn 1..8191, else SB_ERR_UNSUPPORTED.  Workspace:
 * the core-grid table (8 n2^2 bytes), 512-byte partial sums and a 16-byte entry per block
 * of the contraction; at the limits about 2.2 GB for the table and 0.6 GB for the rest.
 * Nothing is atomic: a repeated call is bit-identical. */
typedef struct sb_acf_model {
    const double* snp;
    const double* snp2;
    const double* dnun;
    const double* snx;
    const double* sny;
    int32_t n1, n2, ndnun, nsn, quadrant;
    double sigxn, sigyn, sqrtar, alph2, step1, step2, wn_amp, amp;
} sb_acf_model;

int sb_acf_model_f64(const sb_acf_model* m, double* acf, double* efield, void* stream);

/* ---- scint_sim.Simulation ------------------------------------------------ */

typedef struct sb_sim_params {
    int32_t nx, ny;
    double dx, dy, alpha, ar, psi, inner;
    double consp;   /* Simulation.set_constants (scint_sim.py:137-167), host */
} sb_sim_params;

/* Spectral amplitude w[nx][ny] (float64): the swdsp fill of
 * Simulation.get_screen (scint_sim.py:176-198, swdsp :276-292) including the
 * reference's ky=0 mirror quirk (:185). */
int sb_sim_weights(const sb_sim_params* p, double* w, void* stream);

/* xyp = real(fft2(w * (n1 + i n2))) in float64 (scint_sim.py:201-204).
 * noise_re / noise_im: float64 [nx][ny] (the reference's two randn fields, for
 * seed parity) or both NULL -> counter-based device Gaussian noise from `seed`
 * (statistically equivalent, not the MT19937 stream). */
int sb_sim_screen(int32_t nx, int32_t ny, const double* w, const double* noise_re,
                  const double* noise_im, uint64_t seed, double* xyp, void* stream);

/* Simulation.get_intensity + frfilt3 (scint_sim.py:209-236, 294-311).
 * scales_host: float64[nf] HOST array of the per-frequency `scale`
 * (:218-224).  spe_t: complex64 [nf][nx] = spe transposed (spe[:, f] is
 * column ny//2 of ifft2(filter * fft2(exp(i xyp scale)))); xyi: float32
 * [nx][ny] intensity of the LAST frequency (:232) or NULL. */
int sb_sim_intensity(int32_t nx, int32_t ny, int32_t nf, const double* xyp,
                     const double* scales_host, double ffconx, double ffcony,
                     void* spe_t, float* xyi, void* stream);

/* element-wise float64 -> float32 (n elements); complex128 -> complex64 is the
 * same call with 2n.  Lets the host layer upload the reference's float64
 * arrays unchanged. */
int sb_convert_f64_f32(const double* src, float* dst, int64_t n, void* stream);
int sb_convert_f32_f64(const float* src, double* dst, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCINT_B200_H */
