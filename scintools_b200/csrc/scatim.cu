// The scattered image of Dynspec.calc_scattered_image (include/scint_b200_scatim.h,
// sb_scattered_image_f64), batched over spectra that share a crop box.  Everything is
// float64.
//
// The reference fits scipy's RectBivariateSpline(tdel, fdop, 10**(sspec/10)) with s = 0:
// cubic B-splines on the knots [x0]*4 + x[2:-2] + [x_last]*4 of each axis, as many
// coefficients as data points, so the fit is the unique tensor-product interpolant
// Bx C By^T = Z.  Each collocation matrix is banded (two sub- and two superdiagonals) and
// totally positive, so Gaussian elimination without pivoting is stable (de Boor); the host
// factors each axis once (SB_SCATIM_NFAC tables) and the device solves:
//   linear   Z = 10**(sspec/10) of every crop box, read once at any row pitch
//   delay    forward and back substitution down every Doppler column, one thread per
//            column, so each row step is one coalesced load
//   doppler  the same along every delay row: a warp stages 32 rows x 32 columns in shared
//            memory with coalesced loads, then each lane runs its row through the tile
//   eval     FITPACK's fpbisp at every image point, in its operation order (the clamp to
//            [t_3, t_m], the interval search, fpbspl's recurrence, the 4 x 4 sum), times
//            fdop_y, written to both mirrored rows; each block writes its minimum
//   shift    image -= min(image); image += 1e-10, the blocks' minima reduced in a fixed
//            order (plot_scattered_image's in-place shift)
// Nothing is atomic and no item's arithmetic depends on another's, so an item's image is
// bit-identical alone, in any stack and on repeat.
#include <math.h>

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int SI_CHUNK = 8;     // rows a delay-pass thread loads before it steps through them
constexpr int SI_WARPS = 4;     // warps per Doppler-pass block, 32 rows each
constexpr int SI_THREADS = 256;

__device__ __forceinline__ double si_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// np.min's rule: any NaN wins
__device__ __forceinline__ double si_min(double a, double b) {
    return (a != a || b != b) ? si_nan() : (b < a ? b : a);
}

// w[z][i][j] = 10**(sspec[offset[z] + i pitch + j] / 10)
__global__ void si_linear_kernel(const double* __restrict__ sspec,
                                 const long long* __restrict__ offset, long long pitch, int nitem,
                                 int mx, int my, double* __restrict__ w) {
    const long long per = (long long)mx * my, m = per * nitem;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        const long long z = k / per, r = (k % per) / my, c = k % my;
        w[k] = exp10(__ddiv_rn(sspec[offset[z] + r * pitch + c], 10.0));
    }
}

// solves L U x = z in place down column j of item blockIdx.y (fac: SB_SCATIM_NFAC tables)
__global__ void si_delay_kernel(double* __restrict__ w, int mx, int my,
                                const double* __restrict__ fac) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= my) return;
    double* __restrict__ p = w + (long long)blockIdx.y * mx * my + j;
    const double *l2 = fac, *l1 = fac + mx, *dinv = fac + 2 * mx, *u1 = fac + 3 * mx,
                 *u2 = fac + 4 * mx;
    double a = 0.0, b = 0.0;    // the two previous results
    for (int i0 = 0; i0 < mx; i0 += SI_CHUNK) {
        const int n = mx - i0 < SI_CHUNK ? mx - i0 : SI_CHUNK;
        double z[SI_CHUNK];
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) z[q] = p[(long long)(i0 + q) * my];
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) {
                const int i = i0 + q;
                const double y = z[q] - l1[i] * b - l2[i] * a;
                z[q] = y;
                a = b;
                b = y;
            }
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) p[(long long)(i0 + q) * my] = z[q];
    }
    a = b = 0.0;
    for (int i1 = mx; i1 > 0; i1 -= SI_CHUNK) {
        const int n = i1 < SI_CHUNK ? i1 : SI_CHUNK;
        double z[SI_CHUNK];
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) z[q] = p[(long long)(i1 - 1 - q) * my];
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) {
                const int i = i1 - 1 - q;
                const double x = (z[q] - u1[i] * b - u2[i] * a) * dinv[i];
                z[q] = x;
                a = b;
                b = x;
            }
#pragma unroll
        for (int q = 0; q < SI_CHUNK; ++q)
            if (q < n) p[(long long)(i1 - 1 - q) * my] = z[q];
    }
}

// solves L U x = z in place along 32 rows per warp of item blockIdx.y, through a shared tile
__global__ void __launch_bounds__(32 * SI_WARPS)
si_doppler_kernel(double* __restrict__ w, int mx, int my, const double* __restrict__ fac) {
    SB_SHARED double tile[SI_WARPS][32][33];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int r0 = (blockIdx.x * SI_WARPS + wp) * 32;
    if (r0 >= mx) return;
    double(*t)[33] = tile[wp];
    double* __restrict__ base = w + (long long)blockIdx.y * mx * my + (long long)r0 * my;
    const double *l2 = fac, *l1 = fac + my, *dinv = fac + 2 * my, *u1 = fac + 3 * my,
                 *u2 = fac + 4 * my;
    const int nr = mx - r0 < 32 ? mx - r0 : 32, nch = (my + 31) / 32;
    double a = 0.0, b = 0.0;
    for (int ch = 0; ch < nch; ++ch) {
        const int c0 = ch * 32, nc = my - c0 < 32 ? my - c0 : 32;
        for (int rr = 0; rr < nr; ++rr)
            if (lane < nc) t[rr][lane] = base[(long long)rr * my + c0 + lane];
        __syncwarp();
        if (lane < nr)
            for (int cc = 0; cc < nc; ++cc) {
                const int j = c0 + cc;
                const double y = t[lane][cc] - l1[j] * b - l2[j] * a;
                t[lane][cc] = y;
                a = b;
                b = y;
            }
        __syncwarp();
        for (int rr = 0; rr < nr; ++rr)
            if (lane < nc) base[(long long)rr * my + c0 + lane] = t[rr][lane];
        __syncwarp();
    }
    a = b = 0.0;
    for (int ch = nch - 1; ch >= 0; --ch) {
        const int c0 = ch * 32, nc = my - c0 < 32 ? my - c0 : 32;
        for (int rr = 0; rr < nr; ++rr)
            if (lane < nc) t[rr][lane] = base[(long long)rr * my + c0 + lane];
        __syncwarp();
        if (lane < nr)
            for (int cc = nc - 1; cc >= 0; --cc) {
                const int j = c0 + cc;
                const double x = (t[lane][cc] - u1[j] * b - u2[j] * a) * dinv[j];
                t[lane][cc] = x;
                a = b;
                b = x;
            }
        __syncwarp();
        for (int rr = 0; rr < nr; ++rr)
            if (lane < nc) base[(long long)rr * my + c0 + lane] = t[rr][lane];
        __syncwarp();
    }
}

// fpbisp's clamp and interval: arg in [t_3, t_m], l the largest index in [3, m - 1] with
// t_l <= arg (a point on the last knot falls in the last interval); returns the clamped arg
__device__ __forceinline__ double si_interval(const double* __restrict__ t, int m, double arg,
                                              int& l) {
    if (arg < t[3]) arg = t[3];
    if (arg > t[m]) arg = t[m];
    int lo = 3, hi = m - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t[mid] <= arg) lo = mid;
        else hi = mid - 1;
    }
    l = lo;
    return arg;
}

// fpbspl: the four nonzero cubic B-splines at x in [t_l, t_l+1), de Boor-Cox's recurrence
__device__ __forceinline__ void si_bspl(const double* __restrict__ t, int l, double x,
                                        double h[4]) {
    double hh[3];
    h[0] = 1.0;
#pragma unroll
    for (int j = 1; j <= 3; ++j) {
#pragma unroll
        for (int i = 0; i < j; ++i) hh[i] = h[i];
        h[0] = 0.0;
#pragma unroll
        for (int i = 1; i <= j; ++i) {
            const double tr = t[l + i], tl = t[l + i - j];
            if (tr == tl) {
                h[i] = 0.0;
                continue;
            }
            const double f = __ddiv_rn(hh[i - 1], __dsub_rn(tr, tl));
            h[i - 1] = __dadd_rn(h[i - 1], __dmul_rn(f, __dsub_rn(tr, x)));
            h[i] = __dmul_rn(f, __dsub_rn(x, tl));
        }
    }
}

struct SiEval {
    const double *tx, *ty, *ax, *ay, *coef, *eta;
    double *image, *bmin;
    int mx, my, nx, ny;
};

// image[z][ny-1 +- i][c] = spline((ax[c]**2 + ay[i]**2) * eta, ax[c]) * ay[i]; the block's
// minimum to bmin[z][blockIdx.x]
__global__ void __launch_bounds__(SI_THREADS) si_eval_kernel(SiEval e) {
    SB_SHARED double red[SI_THREADS / 32];
    const long long z = blockIdx.y, per = (long long)e.ny * e.nx;
    const double eta = e.eta[z];
    const double* __restrict__ coef = e.coef + z * e.mx * e.my;
    double* __restrict__ img = e.image + z * e.nx * e.nx;
    double mn = INFINITY;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < per;
         k += (long long)gridDim.x * blockDim.x) {
        const int iy = (int)(k / e.nx), c = (int)(k % e.nx);
        const double fx = e.ax[c], fy = e.ay[iy];
        const double q = __dmul_rn(__dadd_rn(__dmul_rn(fx, fx), __dmul_rn(fy, fy)), eta);
        int lx, ly;
        const double qx = si_interval(e.tx, e.mx, q, lx);
        const double qy = si_interval(e.ty, e.my, fx, ly);
        double hx[4], hy[4];
        si_bspl(e.tx, lx, qx, hx);
        si_bspl(e.ty, ly, qy, hy);
        const double* cc = coef + (long long)(lx - 3) * e.my + (ly - 3);
        double sp = 0.0;
#pragma unroll
        for (int i1 = 0; i1 < 4; ++i1)
#pragma unroll
            for (int j1 = 0; j1 < 4; ++j1)
                sp = __dadd_rn(sp, __dmul_rn(__dmul_rn(cc[(long long)i1 * e.my + j1], hx[i1]),
                                             hy[j1]));
        const double v = __dmul_rn(sp, fy);
        const int s = e.ny - 1;
        img[(long long)(s + iy) * e.nx + c] = v;
        if (iy > 0) img[(long long)(s - iy) * e.nx + c] = v;
        mn = si_min(mn, v);
    }
    for (int o = 16; o > 0; o >>= 1) mn = si_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mn;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < SI_THREADS / 32; ++w) mn = si_min(mn, red[w]);
        e.bmin[z * gridDim.x + blockIdx.x] = mn;
    }
}

// image[z] = (image[z] - min(image[z])) + 1e-10, the minimum of the nb block minima
__global__ void si_shift_kernel(double* __restrict__ image, long long per,
                                const double* __restrict__ bmin, int nb) {
    SB_SHARED double s_min;
    const long long z = blockIdx.y;
    if (threadIdx.x < 32) {
        double mn = INFINITY;
        for (int t = threadIdx.x; t < nb; t += 32) mn = si_min(mn, bmin[z * nb + t]);
        for (int o = 16; o > 0; o >>= 1) mn = si_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        if (threadIdx.x == 0) s_min = mn;
    }
    __syncthreads();
    const double mn = s_min;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < per;
         k += (long long)gridDim.x * blockDim.x)
        image[z * per + k] = __dadd_rn(__dsub_rn(image[z * per + k], mn), 1e-10);
}

// blocks of an evaluation pass per item: fixed by the image size alone
inline int si_eval_blocks(int nx, int ny) {
    const long long b = ((long long)nx * ny + SI_THREADS - 1) / SI_THREADS;
    return (int)(b < 1024 ? b : 1024);
}

#ifndef SB_HOST_EMU

int scattered_image(const sb_scatim* s, cudaStream_t st) {
    SB_ARG(s != nullptr);
    if (s->nitem < 1 || s->nitem > 65535 || s->mx < SB_SCATIM_MIN_M ||
        s->mx > SB_SCATIM_MAX_MX || s->my < SB_SCATIM_MIN_M || s->my > SB_SCATIM_MAX_MY ||
        s->nx < 1 || s->nx > SB_SCATIM_MAX_NX || s->nx != 2 * s->ny - 1) {
        set_error("scattered_image: %d items (1..65535), crop %d x %d (%d..%d x %d..%d), "
                  "image %d x %d (nx = 2 ny - 1 <= %d)", s->nitem, s->mx, s->my,
                  SB_SCATIM_MIN_M, SB_SCATIM_MAX_MX, SB_SCATIM_MIN_M, SB_SCATIM_MAX_MY, s->nx,
                  s->ny, SB_SCATIM_MAX_NX);
        return SB_ERR_UNSUPPORTED;
    }
    SB_ARG(s->pitch >= s->my && s->sspec && s->offset && s->eta && s->tx && s->fx && s->ty &&
           s->fy && s->ax && s->ay && s->image);
    const int ni = s->nitem, mx = s->mx, my = s->my, nx = s->nx, ny = s->ny;
    const long long per = (long long)mx * my;
    const int nb = si_eval_blocks(nx, ny);
    double* w = (double*)workspace(WS_PLANE0, (size_t)per * ni * sizeof(double));
    double* bmin = (double*)workspace(WS_PLANE1, (size_t)nb * ni * sizeof(double));
    if (!w || !bmin) return SB_ERR_NOMEM;
    const long long ml = per * ni, bl = (ml + 255) / 256, cap = (long long)num_sms() * 16;
    si_linear_kernel<<<(unsigned)(bl < cap ? bl : cap), 256, 0, st>>>(
        s->sspec, (const long long*)s->offset, (long long)s->pitch, ni, mx, my, w);
    SB_LAUNCH_CHECK();
    si_delay_kernel<<<dim3((unsigned)((my + 127) / 128), (unsigned)ni), 128, 0, st>>>(w, mx, my,
                                                                                    s->fx);
    SB_LAUNCH_CHECK();
    si_doppler_kernel<<<dim3((unsigned)((mx + 32 * SI_WARPS - 1) / (32 * SI_WARPS)),
                             (unsigned)ni), 32 * SI_WARPS, 0, st>>>(w, mx, my, s->fy);
    SB_LAUNCH_CHECK();
    SiEval e{s->tx, s->ty, s->ax, s->ay, w, s->eta, s->image, bmin, mx, my, nx, ny};
    si_eval_kernel<<<dim3((unsigned)nb, (unsigned)ni), SI_THREADS, 0, st>>>(e);
    SB_LAUNCH_CHECK();
    if (s->shift) {
        const long long n2 = (long long)nx * nx, sb_ = (n2 + 2047) / 2048;
        si_shift_kernel<<<dim3((unsigned)(sb_ < 1024 ? sb_ : 1024), (unsigned)ni), 256, 0, st>>>(
            s->image, n2, bmin, nb);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
