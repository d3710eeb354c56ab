// Host drivers of libscint_b200: the one declaration of each driver api.cu calls, and of
// the parameter structs it hands them.  Every file that defines one includes this header.
#pragma once
#include "thth.cuh"
#include "../../include/scint_b200_brightness.h"
#include "../../include/scint_b200_scatim.h"
#include "../../include/scint_b200_clean.h"

namespace sb {

// thin.cu: the two-curvature (thin screen) theta-theta geometry
struct ThinGeom {
    ThthGeom g;          // cs, ntau, nfd, dtau, dfd ...; tau0 := tau[1], fd0 := fd[1];
                         // g.th / g.n = theta1 centres (columns)
    const double* th2;   // theta2 centres (rows)
    int n2;
    double tau_max;      // tau.max() (not abs)
    double center_cut;
    int power;           // 0: CS as is, 1: |CS|^2 (incoherent thin, ththmod.py:609)
};

// sim.cu: the phase-screen parameters of sim_weights
struct SimParams {
    int nx, ny;
    double dx, dy, alpha, ar, psi, inner, consp;
};

#ifndef SB_HOST_EMU
// thth.cu
int eta_sweep(const ThthGeom& g, const double* th_host, const double* d_etas,
              int neta, double tol, int max_iter, double* d_eigs,
              int* d_status, int* d_nred, int* d_iters, cudaStream_t st);
int thth_map(const ThthGeom& g, double eta, int hermitian, float2* d_out,
             int* d_tau_inv, int* d_fd_inv, unsigned char* d_pnts,
             unsigned char* d_th_pnts, int* d_err, cudaStream_t st);

// eig_half.cu: fp16 iteration + fp32 Rayleigh quotient (default for ld <= 512);
// d_Mb: the scaled fp16 copy of d_M written by thth_build_kernel<2>
int eig_half_launch(const float2* d_M, const unsigned* d_Mb, int ld, const int* d_nred, int e0,
                    int nb, double* d_eigs, int* d_status, int* d_iters, double tol, double etol,
                    int max_iter, cudaStream_t st);

// thin.cu
int thin_sweep(const ThinGeom& t, const double* d_eta1, const double* d_eta2, int neta,
               double tol, int max_iter, double* d_sv, int* d_status, int* d_n1, int* d_n2,
               int* d_iters, cudaStream_t st);
int thin_map(const ThinGeom& t, double e1, double e2, float2* d_out, int* d_err,
             cudaStream_t st);

// dynspec.cu
int sspec(const float* dyn, int nf, int nt, const float* wt, const float* wf,
          double swt, double swf, int prewhite, int halve, int db,
          const float* pd1, const float* pd2, float* sec, cudaStream_t st,
          int noshift = 0);
int conj_spectrum(const float* dyn, int nf, int nt, int npad, float pad_value,
                  const unsigned char* rowmask, int half, long pitch, int ncols_keep,
                  float2* CS, cudaStream_t st);
int conj_spectrum_bound(const float* dyn, int nf, int nt, int npad, float pad_value, float* out,
                        cudaStream_t st);
int acf(const float* dyn, int nf, int nt, int subtract_mean, int normalise,
        float* out, cudaStream_t st);
int acf_sspec(const float* dyn, int nf, int nt, const float* wt, const float* wf,
              double swt, double swf, int normalise, float* out, cudaStream_t st);
int sspec_tiles(const float* dyn, int nf, int nt, int fnum, int tnum, int nfc, int ntc,
                const float* wt, const float* wf, double swt, double swf, float* sec,
                cudaStream_t st);
int acf_tiles(const float* dyn, int nf, int nt, int fnum, int tnum, int nfc, int ntc,
              float* acf, cudaStream_t st);
void twiddle_release();

// sim.cu
int sim_weights(const SimParams& p, double* w, cudaStream_t st);
int sim_screen(int nx, int ny, const double* w, const double* n1, const double* n2,
               unsigned long long seed, double* xyp, cudaStream_t st);
int sim_intensity(int nx, int ny, int nf, const double* xyp, const double* scales_host,
                  double ffconx, double ffcony, float2* spe_t, float* xyi,
                  cudaStream_t st);

// retrieval.cu
int rev_map(const float2* thth, int n, const double* th_dev, double eta, double tau0,
            double dtau, int ntau, double fd0, double dfd, int nfd, int hermitian,
            float2* recov, cudaStream_t st);
int herm_eigvec(const float2* A, int n, int ld, double tol, int max_iter, double* w_dev,
                float2* V_dev, int* info_dev, cudaStream_t st);
int ifft2_c2c(const float2* in, int n0, int n1, int centred, int crop0, int crop1,
              double scale, int real_only, void* out, cudaStream_t st);
int chisq_sweep(const ThthGeom& g, const double* th_host, const double* d_etas, int neta,
                const double* d_th_red, double dtau_bin, double dfd_bin, const float* dspec,
                const unsigned char* mask, int nf, int nt, double tol, int max_iter,
                double* d_ssq, double* d_w, int* d_status, int* d_nred, int* d_iters,
                cudaStream_t st);
int conj_spectrum_c2c(const float2* in, int nf, int nt, int npad, float pad_re, float pad_im,
                      const unsigned char* rowmask, float2* CS, cudaStream_t st);
int vlbi_retrieval(const ThthGeom& g, const double* th_host, const float2* const* cs_host,
                   int n_dish, double eta, const double* d_th_red, double dtau_bin,
                   double dfd_bin, int nf, int nt, double tol, int max_iter, float2* d_model,
                   double* d_w, float2* d_v, int* d_info, cudaStream_t st);
int asymmetry_batch(const ThthGeom* geoms, const double* const* th_host, int nchunk,
                    const double* d_etas, double tol, int max_iter, double* d_asym, double* d_w,
                    int* d_status, int* d_nred, int* d_iters, float2* d_v, cudaStream_t st);
int gerchberg_saxton(float2* W, const float* amp, const unsigned char* rowmask, int n0, int n1,
                     int niter, cudaStream_t st);

// mosaic.cu
int mosaic_build(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
                 const double* amp, float2* W, cudaStream_t st);
int mosaic_rot(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
               const float2* W, double* power, double* der, cudaStream_t st);
int mosaic_overlap(const float2* chunks, int ncf, int nct, int cwf, int cwt, double* C,
                   cudaStream_t st);
int mosaic_fit(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
               const double* amp, const float2* W, const float* dspec, const float* noise,
               double* fit, double* grad, cudaStream_t st);
int mosaic_hess(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
                const double* amp, const float2* W, const float* dspec, const float* noise,
                long long* rows, long long* cols, double* vals, cudaStream_t st);

// svd.cu
int svd_topk(const float* A, int nf, int nt, int k, double* Y, double* s_host, double* res_host,
             double* gap_host, int* info_host, cudaStream_t st);
int svd_apply(const float* A, int nf, int nt, int k, const double* Y, float* out, float* model,
              cudaStream_t st);
int bandpass_rows(const float* A, int nf, int nt, int zero_as_nan, double* mean, cudaStream_t st);
int bandpass_cols(const float* A, int nf, int nt, int zero_as_nan, const double* rowdiv,
                  double* mean, cudaStream_t st);
int bandpass_divide(const float* A, int nf, int nt, int zero_as_nan, const double* rowdiv,
                    const double* coldiv, float* out, cudaStream_t st);

// slow_ft.cu
int slow_ft(const float* x, int nt, int nf, const double* s, float2* out, cudaStream_t st);

// inpaint.cu
int inpaint_biharmonic(const double* img, int nf, int nt, const int* pix, int n,
                       const double* tables, const unsigned char* rcls, int nrc,
                       const unsigned char* ccls, int ncc, double lo, double hi, double tol,
                       int maxit, double* out, int* info_host, double* resid_host,
                       cudaStream_t st);
int medfilt_masked(const double* img, int nf, int nt, const int* pix, int n, int kh, int kw,
                   double nan_value, double* out, cudaStream_t st);

// clean.cu
int dyn_zero_counts(const double* dyn, int nf, int nt, int row0, int row1, int* row_counts,
                    int* col_counts, cudaStream_t st);
int zap(double* x, long long n, double sigma, double* stats, cudaStream_t st);

// scintfit.cu
int scint_fit_1d(const sb_scint_fit* fits, int nfit, double* out, int* info, cudaStream_t st);
int scint_fit_2d(const sb_scint_fit* fits, int nfit, double* out, int* info, cudaStream_t st);

// acf_model.cu
int acf_model(const sb_acf_model* m, double* acf, double* efield, cudaStream_t st);

// brightness.cu
int brightness(const sb_brightness* d, cudaStream_t st);

// scatim.cu
int scattered_image(const sb_scatim* s, cudaStream_t st);

// normsspec.cu
int norm_sspec_rows(const float* sspec, int nr, int nc, const double* fdop, const double* tdel,
                    double eta, double maxnormfac, const double* fdopnew, int nq, float* out,
                    double* power, cudaStream_t st);
int norm_sspec_avg(const float* norm, int nr, int nq, const double* weights, double* avg,
                   cudaStream_t st);

// scale_dyn.cu
int scale_dyn_lambda(const float* dyn, int nf, int nt, int flip, const float* a,
                     const float* cp, const float* inv, const float* g, float p0, float pn,
                     const int* idx, const float4* W, int nlam, float* out, cudaStream_t st);
#endif  // SB_HOST_EMU

}  // namespace sb
