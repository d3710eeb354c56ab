// extern "C" surface of libscint_b200 (see include/scint_b200.h).
#include <stdarg.h>
#include <string.h>

#include <vector>

#include "../../include/scint_b200.h"
#include "../../include/scint_b200_brightness.h"
#include "../../include/scint_b200_scatim.h"
#include "../../include/scint_b200_clean.h"
#include "common.cuh"
#include "drivers.cuh"

namespace sb {

static thread_local char g_err[512] = "";
static void* g_ws[WS_COUNT] = {nullptr};
static size_t g_ws_bytes[WS_COUNT] = {0};
static int g_sms = 132;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }
int num_sms() { return g_sms; }

static long long g_launches = 0;
void count_launch() { ++g_launches; }

// ---- profiling ---------------------------------------------------------
struct ProfPair { int id; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ProfPair> g_prof_pending;
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t g_prof_open[PROF_COUNT];

static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) {
        cudaEvent_t e = g_prof_pool.back();
        g_prof_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
void prof_begin(int id, cudaStream_t st) {
    if (!g_prof_on) return;
    g_prof_open[id] = prof_event();
    cudaEventRecord(g_prof_open[id], st);
}
void prof_end(int id, cudaStream_t st) {
    if (!g_prof_on) return;
    cudaEvent_t b = prof_event();
    cudaEventRecord(b, st);
    g_prof_pending.push_back({id, g_prof_open[id], b});
}

// ---- cross-stream ordering ----------------------------------------------
// The workspace slots and the twiddle tables belong to the process, not to a stream: a call
// on stream B may read a table whose fill is still queued on stream A, or reuse a slot A's
// kernels still use.  Every entry point that touches library memory therefore starts behind
// the previous call when the stream changes, and records the fence when it returns.  The
// event is recorded at exit, not at the next entry, so waiting on it stays valid after the
// caller destroys the earlier stream.  A call on the previous call's stream pays the record.
static cudaEvent_t g_fence = nullptr;
static cudaStream_t g_fence_stream = nullptr;
static bool g_fence_recorded = false;

static cudaError_t fence_init() {
    if (g_fence) return cudaSuccess;
    return cudaEventCreateWithFlags(&g_fence, cudaEventDisableTiming);
}

struct StreamFence {
    cudaStream_t st;
    explicit StreamFence(void* stream) : st((cudaStream_t)stream) {
        if (fence_init() != cudaSuccess) {
            cudaGetLastError();
            return;
        }
        if (g_fence_recorded && st != g_fence_stream) cudaStreamWaitEvent(st, g_fence, 0);
    }
    ~StreamFence() {
        if (!g_fence) return;
        cudaEventRecord(g_fence, st);
        g_fence_stream = st;
        g_fence_recorded = true;
    }
};

void* workspace(WsSlot slot, size_t bytes) {
    if (slot < 0 || slot >= WS_COUNT) return nullptr;
    if (bytes <= g_ws_bytes[slot] && g_ws[slot]) return g_ws[slot];
    if (g_ws[slot]) {
        cudaDeviceSynchronize();
        cudaFree(g_ws[slot]);
        g_ws[slot] = nullptr;
        g_ws_bytes[slot] = 0;
    }
    size_t want = (bytes + (size_t(1) << 20) - 1) & ~((size_t(1) << 20) - 1);
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        set_error("workspace slot %d: cudaMalloc(%zu) -> %s", slot, want,
                  cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    g_ws[slot] = p;
    g_ws_bytes[slot] = want;
    return p;
}

void workspace_release() {
    cudaDeviceSynchronize();
    for (int i = 0; i < WS_COUNT; ++i) {
        if (g_ws[i]) cudaFree(g_ws[i]);
        g_ws[i] = nullptr;
        g_ws_bytes[i] = 0;
    }
}

template <typename A, typename B>
__global__ void convert_kernel(const A* __restrict__ a, B* __restrict__ b, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        b[i] = (B)a[i];
}

static int to_geom(const sb_thth_geom* in, ThthGeom* g) {
    SB_ARG(in != nullptr);
    SB_ARG(in->ntau > 0 && in->nfd > 0);
    SB_ARG(in->th_cents != nullptr && in->th_cents_host != nullptr);
    SB_ARG(in->n_th > 0);
    g->cs = (const float2*)in->cs;
    g->ntau = in->ntau;
    g->nfd = in->nfd;
    g->tau0 = in->tau0;
    g->dtau = in->dtau;
    g->half_dtau = in->dtau / 2;  // dtau / 2 (ththmod.py:95)
    g->tau_absmax = in->tau_absmax;
    g->fd0 = in->fd0;
    g->dfd = in->dfd;
    g->half_dfd = in->dfd / 2;
    g->inv_dtau = 1.0 / in->dtau;
    g->inv_dfd = 1.0 / in->dfd;
    g->fd_half = in->fd_half;
    g->th = in->th_cents;
    g->n = in->n_th;
    g->coherent = in->coherent;
    g->cs_half = in->cs_half;
    g->cs_valid_cols = in->cs_half ? in->cs_valid_cols : 0;
    g->cs_bound = in->cs_bound;
    g->cs_pitch = in->cs_half ? in->cs_pitch : (in->cs_pitch > 0 ? in->cs_pitch : in->nfd);
    SB_ARG(!in->cs_half || (in->cs_pitch >= in->nfd / 2 + 1 && in->nfd % 2 == 0));
    return SB_OK;
}

}  // namespace sb

extern "C" {

int sb_abi_version(void) { return 8; }
const char* sb_last_error(void) { return sb::last_error(); }

int sb_init(int device) {
    SB_CUDA(cudaSetDevice(device));
    SB_CUDA(cudaFree(0));
    cudaDeviceProp prop;
    SB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        sb::set_error("device %d is sm_%d%d; libscint_b200 is sm_90a only",
                      device, prop.major, prop.minor);
        return SB_ERR_UNSUPPORTED;
    }
    sb::g_sms = prop.multiProcessorCount;
    SB_CUDA(sb::fence_init());
    return SB_OK;
}

int64_t sb_launch_count(void) { return sb::g_launches; }

int sb_profile_enable(int32_t on) {
    sb::g_prof_on = on != 0;
    return SB_OK;
}

int sb_profile_collect(double* ms_host, int32_t* count_host, int32_t n) {
    SB_ARG(ms_host && count_host && n >= sb::PROF_COUNT);
    for (int i = 0; i < n; ++i) { ms_host[i] = 0.0; count_host[i] = 0; }
    SB_CUDA(cudaDeviceSynchronize());
    for (auto& p : sb::g_prof_pending) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, p.a, p.b);
        ms_host[p.id] += ms;
        count_host[p.id] += 1;
        sb::g_prof_pool.push_back(p.a);
        sb::g_prof_pool.push_back(p.b);
    }
    sb::g_prof_pending.clear();
    return SB_OK;
}

int sb_release(void) {
    sb::workspace_release();
    sb::twiddle_release();
    return SB_OK;
}

int sb_eta_sweep(const sb_thth_geom* geom, const double* etas, int32_t neta,
                 double tol, int32_t max_iter, double* eigs, int32_t* status,
                 int32_t* nred, int32_t* iters, void* stream) {
    sb::StreamFence fence(stream);
    sb::ThthGeom g;
    int rc = sb::to_geom(geom, &g);
    if (rc) return rc;
    SB_ARG(neta >= 0 && etas && eigs && status && nred && iters);
    SB_ARG(geom->cs != nullptr);
    if (!(tol > 0)) tol = 2e-5;
    return sb::eta_sweep(g, geom->th_cents_host, etas, neta, tol, max_iter,
                         eigs, status, nred, iters, (cudaStream_t)stream);
}

int sb_thth_map(const sb_thth_geom* geom, double eta, int32_t hermitian,
                void* thth, int32_t* tau_inv, int32_t* fd_inv, uint8_t* pnts,
                uint8_t* th_pnts, int32_t* err, void* stream) {
    sb::StreamFence fence(stream);
    sb::ThthGeom g;
    int rc = sb::to_geom(geom, &g);
    if (rc) return rc;
    const bool wants_map = thth || tau_inv || fd_inv || pnts;
    SB_ARG(!wants_map || (err != nullptr && geom->cs != nullptr));
    return sb::thth_map(g, eta, hermitian, (float2*)thth, tau_inv, fd_inv,
                        pnts, th_pnts, err, (cudaStream_t)stream);
}

static int to_thin(const sb_thth_geom* geom, const double* th2, int32_t n2, double center_cut,
                   int32_t power, sb::ThinGeom* t) {
    int rc = sb::to_geom(geom, &t->g);
    if (rc) return rc;
    SB_ARG(geom->cs != nullptr && th2 != nullptr && n2 > 0);
    t->th2 = th2;
    t->n2 = n2;
    t->tau_max = geom->tau_absmax;     // carries tau.max() for the thin map
    t->center_cut = center_cut;
    t->power = power;
    return SB_OK;
}

int sb_thin_sweep(const sb_thth_geom* geom, const double* th2_cents, int32_t n_th2,
                  double center_cut, int32_t power, const double* eta1, const double* eta2,
                  int32_t neta, double tol, int32_t max_iter, double* svals,
                  int32_t* status, int32_t* n1_red, int32_t* n2_red, int32_t* iters,
                  void* stream) {
    sb::StreamFence fence(stream);
    sb::ThinGeom t;
    int rc = to_thin(geom, th2_cents, n_th2, center_cut, power, &t);
    if (rc) return rc;
    SB_ARG(neta >= 0 && eta1 && eta2 && svals && status && n1_red && n2_red && iters);
    if (!(tol > 0)) tol = 2e-5;
    return sb::thin_sweep(t, eta1, eta2, neta, tol, max_iter, svals, status, n1_red, n2_red,
                          iters, (cudaStream_t)stream);
}

int sb_thin_map(const sb_thth_geom* geom, const double* th2_cents, int32_t n_th2,
                int32_t power, double eta1, double eta2, void* thth, int32_t* err,
                void* stream) {
    sb::StreamFence fence(stream);
    sb::ThinGeom t;
    int rc = to_thin(geom, th2_cents, n_th2, 0.0, power, &t);
    if (rc) return rc;
    SB_ARG(thth && err);
    return sb::thin_map(t, eta1, eta2, (float2*)thth, err, (cudaStream_t)stream);
}

int sb_rev_map(const void* thth, int32_t n, const double* th_cents, double eta, double tau0,
               double dtau, int32_t ntau, double fd0, double dfd, int32_t nfd,
               int32_t hermitian, void* recov, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(thth && th_cents && recov && n >= 1 && ntau >= 1 && nfd >= 1);
    return sb::rev_map((const float2*)thth, n, th_cents, eta, tau0, dtau, ntau, fd0, dfd, nfd,
                       hermitian, (float2*)recov, (cudaStream_t)stream);
}

int sb_herm_eigvec(const void* a, int32_t n, int32_t ld, double tol, int32_t max_iter,
                   double* w, void* v, int32_t* info, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(a && w && v && info && n >= 1 && ld >= n);
    return sb::herm_eigvec((const float2*)a, n, ld, tol, max_iter, w, (float2*)v, info,
                           (cudaStream_t)stream);
}

int sb_ifft2_c2c_f32(const void* in, int32_t n0, int32_t n1, int32_t centred, int32_t crop0,
                     int32_t crop1, double scale, int32_t real_only, void* out, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(in && out);
    return sb::ifft2_c2c((const float2*)in, n0, n1, centred, crop0, crop1, scale, real_only,
                         out, (cudaStream_t)stream);
}

int sb_chisq_sweep(const sb_thth_geom* geom, const double* etas, int32_t neta,
                   const double* th_red, double dtau_bin, double dfd_bin, const float* dspec,
                   int32_t nf, int32_t nt, const uint8_t* mask, double tol, int32_t max_iter,
                   double* ssq, double* w, int32_t* status, int32_t* nred, int32_t* iters,
                   void* stream) {
    sb::StreamFence fence(stream);
    sb::ThthGeom g;
    int rc = sb::to_geom(geom, &g);
    if (rc) return rc;
    SB_ARG(neta >= 0 && etas && th_red && dspec && ssq && w && status && nred && iters);
    SB_ARG(geom->cs != nullptr);
    return sb::chisq_sweep(g, geom->th_cents_host, etas, neta, th_red, dtau_bin, dfd_bin, dspec,
                           mask, nf, nt, tol, max_iter, ssq, w, status, nred, iters,
                           (cudaStream_t)stream);
}

int sb_gerchberg_saxton_f32(void* wavefield, const float* amp, const uint8_t* rowmask,
                            int32_t n0, int32_t n1, int32_t niter, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(wavefield && amp && rowmask && niter >= 0);
    return sb::gerchberg_saxton((float2*)wavefield, amp, rowmask, n0, n1, niter,
                                (cudaStream_t)stream);
}

int sb_scale_dyn_lambda_f32(const float* dyn, int32_t nf, int32_t nt, int32_t flip_rows,
                            const float* a, const float* cp, const float* inv, const float* g,
                            float p0, float pn, const int32_t* idx, const float* w4,
                            int32_t nlam, float* out, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && a && cp && inv && g && idx && w4 && out && nt >= 1 && nlam >= 1);
    return sb::scale_dyn_lambda(dyn, nf, nt, flip_rows, a, cp, inv, g, p0, pn, idx,
                                (const float4*)w4, nlam, out, (cudaStream_t)stream);
}

int sb_norm_sspec_f32(const float* sspec, int32_t nr, int32_t nc, const double* fdop,
                      const double* tdel, double eta, double maxnormfac,
                      const double* fdopnew, int32_t nq, float* out, double* power,
                      void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(sspec && fdop && tdel && fdopnew && out && power && nr >= 1 && nc >= 2 && nq >= 1);
    return sb::norm_sspec_rows(sspec, nr, nc, fdop, tdel, eta, maxnormfac, fdopnew, nq, out,
                               power, (cudaStream_t)stream);
}

int sb_norm_sspec_avg_f32(const float* norm, int32_t nr, int32_t nq, const double* weights,
                          double* avg, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(norm && weights && avg && nr >= 1 && nq >= 1);
    return sb::norm_sspec_avg(norm, nr, nq, weights, avg, (cudaStream_t)stream);
}

int sb_sspec_f32(const float* dyn, int32_t nf, int32_t nt, const float* win_t,
                 const float* win_f, double sum_win_t, double sum_win_f,
                 int32_t prewhite, int32_t halve, int32_t db, const float* pd_fd,
                 const float* pd_td, float* sec, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && sec && nf >= 2 && nt >= 2);
    SB_ARG((win_t == nullptr) == (win_f == nullptr));
    SB_ARG(!prewhite || (halve && pd_fd && pd_td));
    return sb::sspec(dyn, nf, nt, win_t, win_f, sum_win_t, sum_win_f, prewhite,
                     halve, db, pd_fd, pd_td, sec, (cudaStream_t)stream);
}

int sb_acf_f32(const float* dyn, int32_t nf, int32_t nt, int32_t subtract_mean,
               int32_t normalise, float* acf, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && acf && nf >= 1 && nt >= 1);
    return sb::acf(dyn, nf, nt, subtract_mean, normalise, acf, (cudaStream_t)stream);
}

int sb_acf_sspec_f32(const float* dyn, int32_t nf, int32_t nt, const float* win_t,
                     const float* win_f, double sum_win_t, double sum_win_f,
                     int32_t normalise, float* acf, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && acf && nf >= 2 && nt >= 2);
    SB_ARG((win_t == nullptr) == (win_f == nullptr));
    return sb::acf_sspec(dyn, nf, nt, win_t, win_f, sum_win_t, sum_win_f, normalise,
                         acf, (cudaStream_t)stream);
}

int sb_sspec_tiles_f32(const float* dyn, int32_t nf, int32_t nt, int32_t fnum, int32_t tnum,
                       int32_t nfc, int32_t ntc, const float* win_t, const float* win_f,
                       double sum_win_t, double sum_win_f, float* sec, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && sec);
    SB_ARG((win_t == nullptr) == (win_f == nullptr));
    return sb::sspec_tiles(dyn, nf, nt, fnum, tnum, nfc, ntc, win_t, win_f, sum_win_t, sum_win_f,
                           sec, (cudaStream_t)stream);
}

int sb_acf_tiles_f32(const float* dyn, int32_t nf, int32_t nt, int32_t fnum, int32_t tnum,
                     int32_t nfc, int32_t ntc, float* acf, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dyn && acf);
    return sb::acf_tiles(dyn, nf, nt, fnum, tnum, nfc, ntc, acf, (cudaStream_t)stream);
}

int sb_cs_f32(const float* dspec, int32_t nf, int32_t nt, int32_t npad,
              float pad_value, const uint8_t* tau_rowmask, int32_t half_plane,
              int64_t cs_pitch, int32_t ncols_keep, void* cs, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dspec && cs && nf >= 1 && nt >= 1 && npad >= 0);
    SB_ARG(!half_plane || cs_pitch >= (int64_t)(npad + 1) * nt / 2 + 1);
    return sb::conj_spectrum(dspec, nf, nt, npad, pad_value, tau_rowmask,
                             half_plane, (long)cs_pitch, ncols_keep, (float2*)cs,
                             (cudaStream_t)stream);
}

int sb_cs_bound_f32(const float* dspec, int32_t nf, int32_t nt, int32_t npad, float pad_value,
                    float* bound_out, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(dspec && bound_out && nf >= 1 && nt >= 1 && npad >= 0);
    return sb::conj_spectrum_bound(dspec, nf, nt, npad, pad_value, bound_out, (cudaStream_t)stream);
}

int sb_cs_c2c_f32(const void* vis, int32_t nf, int32_t nt, int32_t npad, float pad_re,
                  float pad_im, const uint8_t* tau_rowmask, void* cs, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(vis && cs && nf >= 1 && nt >= 1 && npad >= 0);
    return sb::conj_spectrum_c2c((const float2*)vis, nf, nt, npad, pad_re, pad_im, tau_rowmask,
                                 (float2*)cs, (cudaStream_t)stream);
}

int sb_vlbi_retrieval(const sb_thth_geom* geom, const void* const* cs_list_host, int32_t n_dish,
                      double eta, const double* th_red, double dtau_bin, double dfd_bin,
                      int32_t nf, int32_t nt, double tol, int32_t max_iter, void* model_e,
                      double* w, void* v, int32_t* info, void* stream) {
    sb::StreamFence fence(stream);
    sb::ThthGeom g;
    int rc = sb::to_geom(geom, &g);
    if (rc) return rc;
    SB_ARG(cs_list_host && th_red && model_e && w && v && info);
    return sb::vlbi_retrieval(g, geom->th_cents_host, (const float2* const*)cs_list_host, n_dish,
                              eta, th_red, dtau_bin, dfd_bin, nf, nt, tol, max_iter,
                              (float2*)model_e, w, (float2*)v, info, (cudaStream_t)stream);
}

int sb_asymmetry_batch(const sb_thth_geom* geoms_host, int32_t nchunk, const double* etas,
                       double tol, int32_t max_iter, double* asym, double* w, int32_t* status,
                       int32_t* nred, int32_t* iters, void* v, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(nchunk >= 0 && (nchunk == 0 || geoms_host));
    SB_ARG(etas && asym && w && status && nred && iters);
    std::vector<sb::ThthGeom> g((size_t)nchunk);
    std::vector<const double*> th((size_t)nchunk);
    for (int k = 0; k < nchunk; ++k) {
        int rc = sb::to_geom(geoms_host + k, &g[k]);
        if (rc) return rc;
        th[k] = geoms_host[k].th_cents_host;
    }
    return sb::asymmetry_batch(g.data(), th.data(), nchunk, etas, tol, max_iter, asym, w, status,
                               nred, iters, (float2*)v, (cudaStream_t)stream);
}

int sb_mosaic_build(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                    const double* phi, const double* amp, void* wavefield, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(chunks && phi && wavefield);
    return sb::mosaic_build((const float2*)chunks, ncf, nct, cwf, cwt, phi, amp,
                            (float2*)wavefield, (cudaStream_t)stream);
}

int sb_mosaic_rot(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                  const double* phi, const void* wavefield, double* power, double* der,
                  void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(chunks && phi && wavefield && power && der);
    return sb::mosaic_rot((const float2*)chunks, ncf, nct, cwf, cwt, phi, (const float2*)wavefield,
                          power, der, (cudaStream_t)stream);
}

int sb_mosaic_overlap(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                      double* overlap, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(chunks && overlap);
    return sb::mosaic_overlap((const float2*)chunks, ncf, nct, cwf, cwt, overlap,
                              (cudaStream_t)stream);
}

int sb_mosaic_fit(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                  const double* phi, const double* amp, const void* wavefield, const float* dspec,
                  const float* noise, double* fit, double* grad, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(chunks && phi && amp && wavefield && dspec && noise && fit && grad);
    return sb::mosaic_fit((const float2*)chunks, ncf, nct, cwf, cwt, phi, amp,
                          (const float2*)wavefield, dspec, noise, fit, grad, (cudaStream_t)stream);
}

int sb_mosaic_hess(const void* chunks, int32_t ncf, int32_t nct, int32_t cwf, int32_t cwt,
                   const double* phi, const double* amp, const void* wavefield, const float* dspec,
                   const float* noise, int64_t* rows, int64_t* cols, double* vals, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(chunks && phi && amp && wavefield && dspec && noise && rows && cols && vals);
    return sb::mosaic_hess((const float2*)chunks, ncf, nct, cwf, cwt, phi, amp,
                           (const float2*)wavefield, dspec, noise, (long long*)rows,
                           (long long*)cols, vals, (cudaStream_t)stream);
}

int sb_sim_weights(const sb_sim_params* p, double* w, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(p && w);
    sb::SimParams q{p->nx, p->ny, p->dx, p->dy, p->alpha, p->ar, p->psi, p->inner, p->consp};
    return sb::sim_weights(q, w, (cudaStream_t)stream);
}

int sb_sim_screen(int32_t nx, int32_t ny, const double* w, const double* noise_re,
                  const double* noise_im, uint64_t seed, double* xyp, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(w && xyp && ((noise_re == nullptr) == (noise_im == nullptr)));
    return sb::sim_screen(nx, ny, w, noise_re, noise_im, seed, xyp, (cudaStream_t)stream);
}

int sb_sim_intensity(int32_t nx, int32_t ny, int32_t nf, const double* xyp,
                     const double* scales_host, double ffconx, double ffcony,
                     void* spe_t, float* xyi, void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(xyp && scales_host && spe_t && nf >= 1);
    return sb::sim_intensity(nx, ny, nf, xyp, scales_host, ffconx, ffcony,
                             (float2*)spe_t, xyi, (cudaStream_t)stream);
}

int sb_svd_topk(const float* A, int32_t nf, int32_t nt, int32_t k, double* V, double* s_host,
                double* res_host, double* gap_host, int32_t* info_host, void* stream) {
    sb::StreamFence fence(stream);
    return sb::svd_topk(A, nf, nt, k, V, s_host, res_host, gap_host, info_host,
                        (cudaStream_t)stream);
}

int sb_svd_apply(const float* A, int32_t nf, int32_t nt, int32_t k, const double* V, float* out,
                 float* model, void* stream) {
    sb::StreamFence fence(stream);
    return sb::svd_apply(A, nf, nt, k, V, out, model, (cudaStream_t)stream);
}

int sb_bandpass_rows(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan, double* mean,
                     void* stream) {
    sb::StreamFence fence(stream);
    return sb::bandpass_rows(A, nf, nt, zero_as_nan, mean, (cudaStream_t)stream);
}

int sb_bandpass_cols(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan,
                     const double* rowdiv, double* mean, void* stream) {
    sb::StreamFence fence(stream);
    return sb::bandpass_cols(A, nf, nt, zero_as_nan, rowdiv, mean, (cudaStream_t)stream);
}

int sb_bandpass_divide(const float* A, int32_t nf, int32_t nt, int32_t zero_as_nan,
                       const double* rowdiv, const double* coldiv, float* out, void* stream) {
    sb::StreamFence fence(stream);
    return sb::bandpass_divide(A, nf, nt, zero_as_nan, rowdiv, coldiv, out, (cudaStream_t)stream);
}

int sb_slow_ft_f32(const float* x, int32_t ntime, int32_t nfreq, const double* fscale, void* out,
                   void* stream) {
    sb::StreamFence fence(stream);
    SB_ARG(x && fscale && out);
    return sb::slow_ft(x, ntime, nfreq, fscale, (float2*)out, (cudaStream_t)stream);
}

int sb_inpaint_biharmonic_f64(const double* img, int32_t nf, int32_t nt, const int32_t* pix,
                              int32_t n, const double* tables, const uint8_t* rcls, int32_t nrc,
                              const uint8_t* ccls, int32_t ncc, double lo, double hi, double tol,
                              int32_t maxit, double* out, int32_t* info_host, double* resid_host,
                              void* stream) {
    sb::StreamFence fence(stream);
    return sb::inpaint_biharmonic(img, nf, nt, pix, n, tables, rcls, nrc, ccls, ncc, lo, hi, tol,
                                  maxit, out, info_host, resid_host, (cudaStream_t)stream);
}

int sb_medfilt_masked_f64(const double* img, int32_t nf, int32_t nt, const int32_t* pix, int32_t n,
                          int32_t kh, int32_t kw, double nan_value, double* out, void* stream) {
    sb::StreamFence fence(stream);
    return sb::medfilt_masked(img, nf, nt, pix, n, kh, kw, nan_value, out, (cudaStream_t)stream);
}

int sb_dyn_zero_counts_f64(const double* dyn, int32_t nf, int32_t nt, int32_t row0, int32_t row1,
                           int32_t* row_counts, int32_t* col_counts, void* stream) {
    sb::StreamFence fence(stream);
    return sb::dyn_zero_counts(dyn, nf, nt, row0, row1, row_counts, col_counts,
                               (cudaStream_t)stream);
}

int sb_zap_f64(double* dyn, int64_t n, double sigma, double* stats, void* stream) {
    sb::StreamFence fence(stream);
    return sb::zap(dyn, n, sigma, stats, (cudaStream_t)stream);
}

int sb_scint_fit_1d(const sb_scint_fit* fits, int32_t nfit, double* out, int32_t* info,
                    void* stream) {
    sb::StreamFence fence(stream);
    return sb::scint_fit_1d(fits, nfit, out, info, (cudaStream_t)stream);
}

int sb_scint_fit_2d(const sb_scint_fit* fits, int32_t nfit, double* out, int32_t* info,
                    void* stream) {
    sb::StreamFence fence(stream);
    return sb::scint_fit_2d(fits, nfit, out, info, (cudaStream_t)stream);
}

int sb_acf_model_f64(const sb_acf_model* m, double* acf, double* efield, void* stream) {
    sb::StreamFence fence(stream);
    return sb::acf_model(m, acf, efield, (cudaStream_t)stream);
}

int sb_brightness_f64(const sb_brightness* d, void* stream) {
    sb::StreamFence fence(stream);
    return sb::brightness(d, (cudaStream_t)stream);
}

int sb_scattered_image_f64(const sb_scatim* s, void* stream) {
    sb::StreamFence fence(stream);
    return sb::scattered_image(s, (cudaStream_t)stream);
}

int sb_convert_f64_f32(const double* src, float* dst, int64_t n, void* stream) {
    SB_ARG(src && dst && n >= 0);
    if (n == 0) return SB_OK;
    sb::convert_kernel<double, float><<<sb::num_sms() * 8, 256, 0, (cudaStream_t)stream>>>(src, dst, n);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
int sb_convert_f32_f64(const float* src, double* dst, int64_t n, void* stream) {
    SB_ARG(src && dst && n >= 0);
    if (n == 0) return SB_OK;
    sb::convert_kernel<float, double><<<sb::num_sms() * 8, 256, 0, (cudaStream_t)stream>>>(src, dst, n);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

}  // extern "C"
