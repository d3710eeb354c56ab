// Gap filling behind Dynspec.refill / dynspec.inpaint_biharmonic (include/scint_b200.h,
// sb_inpaint_biharmonic_f64 and sb_medfilt_masked_f64).  Everything is float64.
//
// Biharmonic inpainting.  One unknown per masked pixel, numbered in row-major order (the
// caller passes their pixel indices, pix).  Row k is the stencil S = laplace(laplace(e_p))
// of its pixel p on the 5x5 box around p clipped to the image (scipy.ndimage.laplace, mode
// 'reflect'): masked neighbours go into the matrix, known ones into the right-hand side
// b_k = -sum S(q) img(q).  The stencil depends only on the clipped box's extent and centre
// offset along each axis, so the host builds every variant with laplace itself: rcls[i] /
// ccls[j] name the class of row i / column j, and tables[rc][cc] is the 5x5 stencil of that
// class pair centred on the pixel (zero outside the box).  The device never holds the
// matrix: an image-sized int32 map (-1 for known pixels) and the tables apply it on the fly.
//
// Solver: BiCGSTAB with right Jacobi scaling (x = D^-1 u), so the recurrence residual is
// that of the unscaled system.  An iteration is three kernels over the unknowns:
//   A  p = r + beta (p - omega v), v = A D^-1 p        partial (rhat, v)
//   B  s = r - alpha v,           t = A D^-1 s        partials (t, s), (t, t), (s, s)
//   C  x += alpha D^-1 p + omega D^-1 s, r = s - omega t   partials (rhat, r), (r, r)
// Each kernel reduces the partials it needs itself: every block sums them in block order,
// so every block derives the same scalars and the same decisions, and repeated calls are
// bit-identical.  Block 0 records alpha / rho / omega of each step for the later kernels.
// p and v are double-buffered (kernel A reads the old ones at the neighbours).  The host
// enqueues INP_CHECK iterations at a time and reads the state once per batch.
//
// Stopping inside a batch.  Launch l = 3 it + {0, 1, 2} (kernels A, B, C of step it) of a
// run returns at once if state.stop_at < l, and the launch that decides to stop writes
// stop_at = l (block 0).  A block therefore never reads a stop written by its own launch:
// every block of the stopping launch applies the stop itself (kernel C's last x update
// included), whatever order the blocks run in, and every later launch skips.
//
// Stopping rule: ||r|| <= tol ||b|| on the recurrence residual (after kernel C, or on s
// after kernel B: the half step).  Then one more pass forms the true residual b - A x; if
// that misses the rule, BiCGSTAB restarts from x with rhat = r (at most INP_RESTARTS
// times).  Converged only if the true residual meets the rule.  A breakdown (rho, (rhat, v)
// or omega zero or not finite) ends the current run early and is handled the same way.
// The iteration cap counts every step of every run.
//
// Masked median.  One thread per masked pixel selects the element of rank kh kw / 2 of the
// zero-padded kh x kw window (scipy.signal.medfilt), NaN pixels read as nan_value; a
// median is one of the inputs, so the result is exact.
#include <math.h>

#ifndef SB_HOST_EMU
#include <vector>
#endif

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int INP_THREADS = 256;
constexpr int INP_MAX_NF = 32768;
constexpr int INP_MAX_NT = 16384;
constexpr int INP_MAX_CLASSES = 5;          // per axis: 2 leading, interior, 2 trailing
constexpr int INP_CHECK = 32;               // iterations per host check
constexpr int INP_RESTARTS = 3;
constexpr int MED_MAX_SIDE = 31;

struct InpSys {
    const int* pix;                 // [n] pixel of each unknown
    const int* map;                 // [nf nt] unknown of each pixel, -1 if known
    const unsigned char* rcls;      // [nf]
    const unsigned char* ccls;      // [nt]
    const double* tables;           // [nrc][ncc][25]
    const double* invd;             // [n] 1 / diagonal
    int nf, nt, n, ncc, ntab;
};

// scalars of the iteration, on the device
struct InpState {
    int stop_at;    // launch that stopped the current run, INP_RUNNING while it runs
    int conv;       // it stopped on the rule (1) or on a breakdown (0)
    int steps;      // steps of the current run
};
constexpr int INP_RUNNING = 0x7fffffff;

__device__ __forceinline__ double inp_block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    if (lane == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < nw; ++i) s += red[i];
    __syncthreads();
    return s;
}

// sum of part[0..G) in a fixed order; every thread of every block gets the same value
__device__ __forceinline__ double inp_reduce(const double* part, int G, double* red) {
    double s = 0.0;
    for (int b = threadIdx.x; b < G; b += blockDim.x) s += part[b];
    return inp_block_sum(s, red);
}

__device__ __forceinline__ void inp_load_tables(const InpSys& S, double* tab) {
    for (int e = threadIdx.x; e < S.ntab * 25; e += blockDim.x) tab[e] = S.tables[e];
    __syncthreads();
}

// f(q, c) for every pixel q with a non-zero coefficient c in row k, in a fixed order
template <class F>
__device__ __forceinline__ void inp_row(const InpSys& S, const double* tab, int k, F f) {
    const int p = S.pix[k];
    const int i = p / S.nt, j = p - i * S.nt;
    const double* T = tab + (S.rcls[i] * S.ncc + S.ccls[j]) * 25;
#pragma unroll
    for (int di = -2; di <= 2; ++di) {
        const int ii = i + di;
        if (ii < 0 || ii >= S.nf) continue;
#pragma unroll
        for (int dj = -2; dj <= 2; ++dj) {
            const int jj = j + dj;
            if (jj < 0 || jj >= S.nt) continue;
            const double c = T[(di + 2) * 5 + dj + 2];
            if (c != 0.0) f(ii * S.nt + jj, c);
        }
    }
}

__global__ void inp_map_kernel(const int* __restrict__ pix, int n, int* __restrict__ map) {
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
        map[pix[k]] = k;
}

// b_k = -sum over known q of S(q) img(q), invd_k = 1 / S(p), x = 0; partial ||b||^2
__global__ void __launch_bounds__(INP_THREADS)
inp_setup_kernel(InpSys S, const double* __restrict__ img, double* __restrict__ b,
                 double* __restrict__ invd, double* __restrict__ x, double* __restrict__ part_bb) {
    SB_SHARED double tab[INP_MAX_CLASSES * INP_MAX_CLASSES * 25];
    SB_SHARED double red[32];
    inp_load_tables(S, tab);
    double bb = 0.0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S.n; k += gridDim.x * blockDim.x) {
        const int p = S.pix[k];
        double s = 0.0, d = 0.0;
        inp_row(S, tab, k, [&](int q, double c) {
            if (q == p) d = c;
            else if (S.map[q] < 0) s -= c * img[q];
        });
        b[k] = s;
        invd[k] = d != 0.0 ? 1.0 / d : 1.0;     // a zero diagonal (tiny images): unscaled
        x[k] = 0.0;
        bb += s * s;
    }
    bb = inp_block_sum(bb, red);
    if (threadIdx.x == 0) part_bb[blockIdx.x] = bb;
}

// r = b - A x, rhat = r; partials (r, r) into both part_rr and part_rhr.  Also used for
// the true residual at the end of a run.
__global__ void __launch_bounds__(INP_THREADS)
inp_residual_kernel(InpSys S, const double* __restrict__ b, const double* __restrict__ x,
                    double* __restrict__ r, double* __restrict__ rhat, double* __restrict__ part_rr,
                    double* __restrict__ part_rhr, InpState* __restrict__ st) {
    SB_SHARED double tab[INP_MAX_CLASSES * INP_MAX_CLASSES * 25];
    SB_SHARED double red[32];
    inp_load_tables(S, tab);
    double rr = 0.0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S.n; k += gridDim.x * blockDim.x) {
        double ax = 0.0;
        inp_row(S, tab, k, [&](int q, double c) {
            const int u = S.map[q];
            if (u >= 0) ax += c * x[u];
        });
        const double v = b[k] - ax;
        if (r) {
            r[k] = v;
            rhat[k] = v;
        }
        rr += v * v;
    }
    rr = inp_block_sum(rr, red);
    if (threadIdx.x == 0) {
        part_rr[blockIdx.x] = rr;
        if (part_rhr) part_rhr[blockIdx.x] = rr;
    }
    if (st && blockIdx.x == 0 && threadIdx.x == 0) *st = InpState{INP_RUNNING, 0, 0};
}

struct InpIter {
    double* r;
    const double* rhat;
    double* x;
    double* s;
    double* t;
    double* rho;          // [maxit + 1] per step of the current run
    double* alpha;
    double* omega;
    double* part_rr;      // [G] each
    double* part_rhr;
    double* part_rv;
    double* part_ts;
    double* part_tt;
    double* part_ss;
    InpState* st;
    double thr;           // tol^2 ||b||^2
    int G;
};

__device__ __forceinline__ void inp_stop(InpState* st, int launch, int conv, int steps) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        st->stop_at = launch;
        st->conv = conv;
        st->steps = steps;
    }
}

// kernel A of step it
__global__ void __launch_bounds__(INP_THREADS)
inp_step_a_kernel(InpSys S, InpIter I, int it, const double* __restrict__ p_old,
                  const double* __restrict__ v_old, double* __restrict__ p, double* __restrict__ v) {
    if (I.st->stop_at < 3 * it) return;
    SB_SHARED double tab[INP_MAX_CLASSES * INP_MAX_CLASSES * 25];
    SB_SHARED double red[32];
    const double rr = inp_reduce(I.part_rr, I.G, red);
    const double rho = inp_reduce(I.part_rhr, I.G, red);
    if (rr <= I.thr) {
        inp_stop(I.st, 3 * it, 1, it);
        return;
    }
    if (!(rho != 0.0) || !isfinite(rho)) {
        inp_stop(I.st, 3 * it, 0, it);
        return;
    }
    double beta = 0.0, om = 0.0;
    if (it > 0) {
        om = I.omega[it - 1];
        beta = (rho / I.rho[it - 1]) * (I.alpha[it - 1] / om);
    }
    inp_load_tables(S, tab);
    const double* r = I.r;
    auto pnew = [&](int u) { return it > 0 ? r[u] + beta * (p_old[u] - om * v_old[u]) : r[u]; };
    double rv = 0.0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S.n; k += gridDim.x * blockDim.x) {
        double a = 0.0;
        inp_row(S, tab, k, [&](int q, double c) {
            const int u = S.map[q];
            if (u >= 0) a += c * (S.invd[u] * pnew(u));
        });
        p[k] = pnew(k);
        v[k] = a;
        rv += I.rhat[k] * a;
    }
    rv = inp_block_sum(rv, red);
    if (threadIdx.x == 0) I.part_rv[blockIdx.x] = rv;
    if (blockIdx.x == 0 && threadIdx.x == 0) I.rho[it] = rho;
}

// kernel B of step it
__global__ void __launch_bounds__(INP_THREADS)
inp_step_b_kernel(InpSys S, InpIter I, int it, const double* __restrict__ v) {
    if (I.st->stop_at < 3 * it + 1) return;
    SB_SHARED double tab[INP_MAX_CLASSES * INP_MAX_CLASSES * 25];
    SB_SHARED double red[32];
    const double alpha = I.rho[it] / inp_reduce(I.part_rv, I.G, red);
    if (!isfinite(alpha)) {
        inp_stop(I.st, 3 * it + 1, 0, it);
        return;
    }
    inp_load_tables(S, tab);
    const double* r = I.r;
    double ts = 0.0, tt = 0.0, ss = 0.0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S.n; k += gridDim.x * blockDim.x) {
        double a = 0.0;
        inp_row(S, tab, k, [&](int q, double c) {
            const int u = S.map[q];
            if (u >= 0) a += c * (S.invd[u] * (r[u] - alpha * v[u]));
        });
        const double sk = r[k] - alpha * v[k];
        I.s[k] = sk;
        I.t[k] = a;
        ts += a * sk;
        tt += a * a;
        ss += sk * sk;
    }
    ts = inp_block_sum(ts, red);
    tt = inp_block_sum(tt, red);
    ss = inp_block_sum(ss, red);
    if (threadIdx.x == 0) {
        I.part_ts[blockIdx.x] = ts;
        I.part_tt[blockIdx.x] = tt;
        I.part_ss[blockIdx.x] = ss;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) I.alpha[it] = alpha;
}

// kernel C of step it
__global__ void __launch_bounds__(INP_THREADS)
inp_step_c_kernel(InpSys S, InpIter I, int it, const double* __restrict__ p) {
    if (I.st->stop_at < 3 * it + 2) return;
    SB_SHARED double red[32];
    const double alpha = I.alpha[it];
    const double ss = inp_reduce(I.part_ss, I.G, red);
    const double ts = inp_reduce(I.part_ts, I.G, red);
    const double tt = inp_reduce(I.part_tt, I.G, red);
    const double omega = ts / tt;
    // the half step already meets the rule, or omega breaks down: x += alpha D^-1 p, stop
    const bool half = ss <= I.thr;
    const bool bad = !(omega != 0.0) || !isfinite(omega);
    double rr = 0.0, rhr = 0.0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S.n; k += gridDim.x * blockDim.x) {
        const double dk = S.invd[k];
        if (half || bad) {
            I.x[k] += alpha * (dk * p[k]);
            continue;
        }
        I.x[k] += alpha * (dk * p[k]) + omega * (dk * I.s[k]);
        const double rk = I.s[k] - omega * I.t[k];
        I.r[k] = rk;
        rr += rk * rk;
        rhr += I.rhat[k] * rk;
    }
    if (half || bad) {
        inp_stop(I.st, 3 * it + 2, half ? 1 : 0, it + 1);
        return;
    }
    rr = inp_block_sum(rr, red);
    rhr = inp_block_sum(rhr, red);
    if (threadIdx.x == 0) {
        I.part_rr[blockIdx.x] = rr;
        I.part_rhr[blockIdx.x] = rhr;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) I.omega[it] = omega;
}

// out_k = clip(x_k, lo, hi), NaN kept (np.clip)
__global__ void inp_clip_kernel(const double* __restrict__ x, int n, double lo, double hi,
                                double* __restrict__ out) {
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const double v = x[k];
        out[k] = v < lo ? lo : (v > hi ? hi : v);
    }
}

// ---- masked median ------------------------------------------------------------------------

// element of rank `rank` of a[0..m) (Hoare selection, in place)
__device__ __forceinline__ double med_select(double* a, int m, int rank) {
    int lo = 0, hi = m - 1;
    while (lo < hi) {
        const double piv = a[(lo + hi) >> 1];
        int i = lo, j = hi;
        while (i <= j) {
            while (a[i] < piv) ++i;
            while (piv < a[j]) --j;
            if (i <= j) {
                const double tmp = a[i];
                a[i] = a[j];
                a[j] = tmp;
                ++i;
                --j;
            }
        }
        if (rank <= j) hi = j;
        else if (rank >= i) lo = i;
        else return a[rank];
    }
    return a[rank];
}

template <int CAP>
__global__ void __launch_bounds__(128)
med_masked_kernel(const double* __restrict__ img, int nf, int nt, const int* __restrict__ pix,
                  int n, int kh, int kw, double nan_value, double* __restrict__ out) {
    double a[CAP];
    const int m = kh * kw, rh = kh / 2, rw = kw / 2;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int p = pix[k];
        const int i = p / nt, j = p - i * nt;
        int e = 0;
        for (int di = -rh; di <= rh; ++di) {
            const int ii = i + di;
            for (int dj = -rw; dj <= rw; ++dj) {
                const int jj = j + dj;
                double v = 0.0;
                if (ii >= 0 && ii < nf && jj >= 0 && jj < nt) {
                    v = img[(long long)ii * nt + jj];
                    if (isnan(v)) v = nan_value;
                }
                a[e++] = v;
            }
        }
        out[k] = med_select(a, m, m / 2);
    }
}

#ifndef SB_HOST_EMU

static unsigned inp_grid(long long n, int threads) {
    long long b = (n + threads - 1) / threads;
    const long long cap = (long long)num_sms() * 4;
    return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

static int inp_shape(const char* who, int nf, int nt) {
    SB_ARG(nf >= 1 && nt >= 1);
    if (nf > INP_MAX_NF || nt > INP_MAX_NT) {
        set_error("%s: %d x %d is outside the supported shapes (nf <= %d, nt <= %d)", who, nf, nt,
                  INP_MAX_NF, INP_MAX_NT);
        return SB_ERR_UNSUPPORTED;
    }
    return SB_OK;
}

int inpaint_biharmonic(const double* img, int nf, int nt, const int* pix, int n,
                       const double* tables, const unsigned char* rcls, int nrc,
                       const unsigned char* ccls, int ncc, double lo, double hi, double tol,
                       int maxit, double* out, int* info_host, double* resid_host,
                       cudaStream_t st) {
    int rc = inp_shape("sb_inpaint_biharmonic_f64", nf, nt);
    if (rc) return rc;
    SB_ARG(img && pix && tables && rcls && ccls && out && info_host && resid_host);
    SB_ARG(n >= 1 && (long long)n <= (long long)nf * nt);
    SB_ARG(nrc >= 1 && nrc <= INP_MAX_CLASSES && ncc >= 1 && ncc <= INP_MAX_CLASSES);
    SB_ARG(tol >= 0.0 && maxit >= 1);
    const int G = (int)inp_grid(n, INP_THREADS);
    const size_t npix = (size_t)nf * nt;
    // doubles: b invd x r rhat s t p[2] v[2] (11 n), rho alpha omega (3 (maxit + 1)),
    // partials (7 G), then the map (npix int32) and the state
    const size_t nd = 11 * (size_t)n + 3 * ((size_t)maxit + 1) + 7 * (size_t)G;
    const size_t bytes = nd * sizeof(double) + npix * sizeof(int) + sizeof(InpState) + 16;
    double* w = (double*)workspace(WS_PLANE0, bytes);
    if (!w) return SB_ERR_NOMEM;
    double* b = w;
    double* invd = b + n;
    double* x = invd + n;
    double* r = x + n;
    double* rhat = r + n;
    double* s = rhat + n;
    double* t = s + n;
    double* pb[2] = {t + n, t + 2 * (size_t)n};
    double* vb[2] = {t + 3 * (size_t)n, t + 4 * (size_t)n};
    double* rho = t + 5 * (size_t)n;
    double* alpha = rho + maxit + 1;
    double* omega = alpha + maxit + 1;
    double* part = omega + maxit + 1;
    int* map = (int*)(part + 7 * (size_t)G);
    InpState* state = (InpState*)(map + npix);

    InpSys S{pix, map, rcls, ccls, tables, invd, nf, nt, n, ncc, nrc * ncc};
    SB_CUDA(cudaMemsetAsync(map, 0xff, npix * sizeof(int), st));
    inp_map_kernel<<<inp_grid(n, 256), 256, 0, st>>>(pix, n, map);
    SB_LAUNCH_CHECK();
    double* part_bb = part;
    inp_setup_kernel<<<G, INP_THREADS, 0, st>>>(S, img, b, invd, x, part_bb);
    SB_LAUNCH_CHECK();
    std::vector<double> ph(G);
    SB_CUDA(cudaMemcpyAsync(ph.data(), part_bb, G * sizeof(double), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    double bb = 0.0;
    for (int i = 0; i < G; ++i) bb += ph[i];

    InpIter I{r, rhat, x, s, t, rho, alpha, omega, part, part + G, part + 2 * (size_t)G,
              part + 3 * (size_t)G, part + 4 * (size_t)G, part + 5 * (size_t)G, state,
              tol * tol * bb, G};
    int used = 0, restarts = 0;
    bool converged = false;
    double rr = 0.0;
    for (;;) {
        // a run of BiCGSTAB from x: r = b - A x, rhat = r
        inp_residual_kernel<<<G, INP_THREADS, 0, st>>>(S, b, x, r, rhat, I.part_rr, I.part_rhr,
                                                        state);
        SB_LAUNCH_CHECK();
        InpState h{INP_RUNNING, 0, 0};
        int it = 0;
        while (h.stop_at == INP_RUNNING && used + it < maxit) {
            const int stop = (used + it + INP_CHECK < maxit) ? it + INP_CHECK : maxit - used;
            for (; it < stop; ++it) {
                const int c = it & 1;
                inp_step_a_kernel<<<G, INP_THREADS, 0, st>>>(S, I, it, pb[c ^ 1], vb[c ^ 1], pb[c],
                                                              vb[c]);
                SB_LAUNCH_CHECK();
                inp_step_b_kernel<<<G, INP_THREADS, 0, st>>>(S, I, it, vb[c]);
                SB_LAUNCH_CHECK();
                inp_step_c_kernel<<<G, INP_THREADS, 0, st>>>(S, I, it, pb[c]);
                SB_LAUNCH_CHECK();
            }
            SB_CUDA(cudaMemcpyAsync(&h, state, sizeof(InpState), cudaMemcpyDeviceToHost, st));
            SB_CUDA(cudaStreamSynchronize(st));
        }
        used += h.stop_at != INP_RUNNING ? h.steps : it;
        // the true residual of x
        inp_residual_kernel<<<G, INP_THREADS, 0, st>>>(S, b, x, nullptr, nullptr, part + 6 * (size_t)G,
                                                        nullptr, nullptr);
        SB_LAUNCH_CHECK();
        SB_CUDA(cudaMemcpyAsync(ph.data(), part + 6 * (size_t)G, G * sizeof(double),
                                cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
        rr = 0.0;
        for (int i = 0; i < G; ++i) rr += ph[i];
        converged = rr <= I.thr;
        if (converged || used >= maxit || restarts >= INP_RESTARTS || !std::isfinite(rr)) break;
        ++restarts;
    }
    inp_clip_kernel<<<inp_grid(n, 256), 256, 0, st>>>(x, n, lo, hi, out);
    SB_LAUNCH_CHECK();
    info_host[0] = used;
    info_host[1] = converged ? 1 : 0;
    info_host[2] = restarts;
    *resid_host = bb > 0.0 ? sqrt(rr / bb) : sqrt(rr);
    return SB_OK;
}

int medfilt_masked(const double* img, int nf, int nt, const int* pix, int n, int kh, int kw,
                   double nan_value, double* out, cudaStream_t st) {
    int rc = inp_shape("sb_medfilt_masked_f64", nf, nt);
    if (rc) return rc;
    SB_ARG(img && pix && out && n >= 0 && (long long)n <= (long long)nf * nt);
    SB_ARG(kh >= 1 && kw >= 1 && (kh & 1) && (kw & 1));
    if (kh > MED_MAX_SIDE || kw > MED_MAX_SIDE) {
        set_error("sb_medfilt_masked_f64: kernel %d x %d is larger than %d x %d", kh, kw,
                  MED_MAX_SIDE, MED_MAX_SIDE);
        return SB_ERR_UNSUPPORTED;
    }
    if (n == 0) return SB_OK;
    const int m = kh * kw;
    const unsigned G = inp_grid(n, 128);
    if (m <= 25)
        med_masked_kernel<25><<<G, 128, 0, st>>>(img, nf, nt, pix, n, kh, kw, nan_value, out);
    else if (m <= 121)
        med_masked_kernel<121><<<G, 128, 0, st>>>(img, nf, nt, pix, n, kh, kw, nan_value, out);
    else
        med_masked_kernel<MED_MAX_SIDE * MED_MAX_SIDE><<<G, 128, 0, st>>>(img, nf, nt, pix, n, kh,
                                                                          kw, nan_value, out);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
