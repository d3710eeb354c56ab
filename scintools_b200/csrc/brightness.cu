// The anisotropic brightness model of scint_sim.Brightness (include/scint_b200_brightness.h,
// sb_brightness_f64), batched over parameter sets.  Everything is float64.
//
// Three stages, each a fixed sequence of launches whatever the batch holds:
//   EFIELD  rho      the e-field ACF of every set, in the reference's operation order
//           gemm x2  B = |W rho W|: the 2-D DFT as two complex matrix products with the
//                    DFT matrix W, whose rows and columns carry the fftshift / ifftshift
//   SSPEC   query    thetax, thetay, the Jacobian and the unflipped SS of every (td, fd)
//           flip     SS[1:, 1:] += flip(SS[1:, 1:]) out of place, as numpy's overlap rule
//                    makes it, and LSS = 10 log10 SS
//   ACF     gemm x2  real(M1 SS M2^T) with the shifts folded into M1 and M2, and each output
//                    tile's maximum
//           norm     acf / max(acf)
//
// The DFTs are matrix products rather than FFTs because the sizes are mixed-radix (600,
// 2000 = 2^4 5^3, 1000) and B's tails sit about 1e-9 below its peak, which the fp32 FFT
// engine cannot resolve.  The products run on the FP64 tensor cores (mma.sync m8n8k4 .f64);
// the twiddle matrices are shared by every set of the batch.  Twiddles come from the exact
// integer phase (j k) mod n, so the shifts and odd sizes cost nothing.
//
// Interpolation: griddata's linear interpolant on the lattice meshgrid(x, x) is the
// barycentric interpolant on qhull's triangulation, in which every lattice cell is split by
// one of its diagonals.  The host finds which one once per lattice (diag bitmap); a query
// then needs its cell (binary search in x), the bit and three weights.  Like qhull's
// find_simplex, a query is inside when it is within 100 DBL_EPSILON of the lattice's
// bounding box, and NaN otherwise.
//
// Nothing is atomic and no set's arithmetic depends on another's, so a set's result is
// bit-identical alone, in any batch and on repeat.
#include <math.h>

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int BR_BM = 64;               // output rows per block
constexpr int BR_BN = 64;               // output columns per block
constexpr int BR_BK = 16;               // k per shared-memory stage
constexpr int BR_THREADS = 256;         // 8 warps, 2 x 4, each 32 x 16 outputs
constexpr int BR_LDA = BR_BK + 4;       // padded strides: no bank conflicts on the fragment
constexpr int BR_LDB = BR_BN + 4;       // loads of a half warp
constexpr double BR_HULL_EPS = 100 * 2.220446049250313e-16;

enum BrMode { BR_STORE = 0, BR_ABS = 1, BR_REAL = 2 };

#ifndef SB_HOST_EMU
// d += a b on one 8 x 8 x 4 tile of the FP64 tensor cores: lane l holds A[l / 4][l % 4],
// B[l % 4][l / 4] and D[l / 4][2 (l % 4) + {0, 1}]
__device__ __forceinline__ void br_mma(double2& d, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d.x), "+d"(d.y)
                 : "d"(a), "d"(b));
}
#endif

__device__ __forceinline__ double br_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// np.max's rule: any NaN wins
__device__ __forceinline__ double br_max(double a, double b) {
    return (a != a || b != b) ? br_nan() : (b > a ? b : a);
}

// W[r][c] = exp(-2 pi i p / n), p = ((r + ro) mod n) ((c + co) mod n) mod n
__global__ void br_twiddle_kernel(int n, int ro, int co, double* __restrict__ wr,
                                  double* __restrict__ wi) {
    const long long m = (long long)n * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        const long long r = (k / n + ro) % n, c = (k % n + co) % n;
        long long p = r * c % n;
        if (2 * p > n) p -= n;
        double s, cs;
        sincospi((double)(2 * p) / (double)n, &s, &cs);
        wr[k] = cs;
        wi[k] = -s;
    }
}

// numpy's array ** scalar takes exact shortcuts for these exponents
__device__ __forceinline__ double br_power(double q, double e) {
    if (e == 2.0) return __dmul_rn(q, q);
    if (e == 1.0) return q;
    if (e == 0.5) return __dsqrt_rn(q);
    return pow(q, e);
}

// rho[set][i][j] = exp(-0.5*(a*X**2 + b*Y**2 + c*X*Y)**(alpha/2)) at X = x[j], Y = x[i]
__global__ void br_rho_kernel(int nset, int n, const double* __restrict__ x,
                              const double* __restrict__ par, double* __restrict__ rho) {
    const long long n2 = (long long)n * n, m = n2 * nset;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        const double* p = par + (k / n2) * SB_BRIGHT_NPAR;
        const double X = x[k % n], Y = x[(k % n2) / n];
        const double q = __dadd_rn(__dadd_rn(__dmul_rn(p[0], __dmul_rn(X, X)),
                                             __dmul_rn(p[1], __dmul_rn(Y, Y))),
                                   __dmul_rn(__dmul_rn(p[2], X), Y));
        rho[k] = exp(__dmul_rn(-0.5, br_power(q, p[3])));
    }
}

// C[z] = A[z] B[z], complex, planar; a batch stride of 0 shares the operand.  BIM: B has an
// imaginary part (else it is real).  MODE: BR_STORE writes C, BR_ABS |C| to cr, BR_REAL
// re(C) to cr and the block's maximum to cmax[z][tile].
struct BrGemm {
    const double *ar, *ai, *br, *bi;
    double *cr, *ci, *cmax;
    long long sa, sb, sc;
    int M, N, K;
};

template <bool BIM, int MODE>
__global__ void __launch_bounds__(BR_THREADS) br_gemm_kernel(BrGemm g) {
    SB_SHARED double Ar[BR_BM][BR_LDA], Ai[BR_BM][BR_LDA];
    SB_SHARED double Br[BR_BK][BR_LDB], Bi[BR_BK][BR_LDB];
    SB_SHARED double red[BR_THREADS / 32];
    const long long z = blockIdx.z;
    const double* __restrict__ ar = g.ar + z * g.sa;
    const double* __restrict__ ai = g.ai + z * g.sa;
    const double* __restrict__ br = g.br + z * g.sb;
    const double* __restrict__ bi = BIM ? g.bi + z * g.sb : nullptr;
    const int m0 = blockIdx.y * BR_BM, n0 = blockIdx.x * BR_BN;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16, gr = lane >> 2, tg = lane & 3;
    double2 cr[4][2], ci[4][2];
    for (int p = 0; p < 4; ++p)
        for (int q = 0; q < 2; ++q) cr[p][q] = ci[p][q] = make_double2(0.0, 0.0);
    for (int k0 = 0; k0 < g.K; k0 += BR_BK) {
        for (int e = tid; e < BR_BM * BR_BK; e += BR_THREADS) {
            const int r = e / BR_BK, c = e % BR_BK;
            const bool in = m0 + r < g.M && k0 + c < g.K;
            const long long o = (long long)(m0 + r) * g.K + k0 + c;
            Ar[r][c] = in ? ar[o] : 0.0;
            Ai[r][c] = in ? ai[o] : 0.0;
        }
        for (int e = tid; e < BR_BK * BR_BN; e += BR_THREADS) {
            const int r = e / BR_BN, c = e % BR_BN;
            const bool in = k0 + r < g.K && n0 + c < g.N;
            const long long o = (long long)(k0 + r) * g.N + n0 + c;
            Br[r][c] = in ? br[o] : 0.0;
            if (BIM) Bi[r][c] = in ? bi[o] : 0.0;
        }
        __syncthreads();
        for (int kk = 0; kk < BR_BK; kk += 4) {
            double fr[4], fi[4], hr[2], hi[2];
            for (int p = 0; p < 4; ++p) {
                fr[p] = Ar[wm + 8 * p + gr][kk + tg];
                fi[p] = Ai[wm + 8 * p + gr][kk + tg];
            }
            for (int q = 0; q < 2; ++q) {
                hr[q] = Br[kk + tg][wn + 8 * q + gr];
                hi[q] = BIM ? Bi[kk + tg][wn + 8 * q + gr] : 0.0;
            }
            for (int p = 0; p < 4; ++p)
                for (int q = 0; q < 2; ++q) {
                    br_mma(cr[p][q], fr[p], hr[q]);
                    if (BIM) br_mma(cr[p][q], -fi[p], hi[q]);
                    if (MODE != BR_REAL) {
                        br_mma(ci[p][q], fi[p], hr[q]);
                        if (BIM) br_mma(ci[p][q], fr[p], hi[q]);
                    }
                }
        }
        __syncthreads();
    }
    double mx = -INFINITY;
    for (int p = 0; p < 4; ++p)
        for (int q = 0; q < 2; ++q)
            for (int h = 0; h < 2; ++h) {
                const int row = m0 + wm + 8 * p + gr, col = n0 + wn + 8 * q + 2 * tg + h;
                if (row >= g.M || col >= g.N) continue;
                const long long o = z * g.sc + (long long)row * g.N + col;
                const double re = h ? cr[p][q].y : cr[p][q].x, im = h ? ci[p][q].y : ci[p][q].x;
                if (MODE == BR_STORE) {
                    g.cr[o] = re;
                    g.ci[o] = im;
                } else if (MODE == BR_ABS) {
                    g.cr[o] = hypot(re, im);
                } else {
                    g.cr[o] = re;
                    mx = br_max(mx, re);
                }
            }
    if (MODE == BR_REAL) {
        for (int o = 16; o > 0; o >>= 1) mx = br_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) red[warp] = mx;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < BR_THREADS / 32; ++w) mx = br_max(mx, red[w]);
            g.cmax[z * gridDim.x * gridDim.y + blockIdx.y * gridDim.x + blockIdx.x] = mx;
        }
    }
}

// largest j in [0, n - 2] with x[j] <= q (0 below the lattice, n - 2 above it)
__device__ __forceinline__ int br_cell(const double* __restrict__ x, int n, double q) {
    int lo = 0, hi = n - 2;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (x[mid] <= q) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// griddata(..., method='linear') of B on meshgrid(x, x) at (qx, qy)
__device__ double br_interp(const double* __restrict__ x, int n, const unsigned char* diag,
                            const double* __restrict__ B, double qx, double qy) {
    const double lo = x[0] - BR_HULL_EPS, hi = x[n - 1] + BR_HULL_EPS;
    if (!(qx >= lo && qx <= hi && qy >= lo && qy <= hi)) return br_nan();
    const int j = br_cell(x, n, qx), i = br_cell(x, n, qy);
    const double u = (qx - x[j]) / (x[j + 1] - x[j]), v = (qy - x[i]) / (x[i + 1] - x[i]);
    const double* b = B + (long long)i * n + j;
    const double f00 = b[0], f10 = b[1], f01 = b[n], f11 = b[n + 1];
    const long long k = (long long)i * (n - 1) + j;
    if ((diag[k >> 3] >> (7 - (k & 7))) & 1) {      // split along (x[j], x[i])-(x[j+1], x[i+1])
        return u >= v ? (1 - u) * f00 + (u - v) * f10 + v * f11
                      : (1 - v) * f00 + (v - u) * f01 + u * f11;
    }
    return u + v <= 1 ? (1 - u - v) * f00 + u * f10 + v * f01
                      : (u + v - 1) * f11 + (1 - v) * f10 + (1 - u) * f01;
}

struct BrQuery {
    const double *x, *td, *colx, *colq, *par, *B;
    const unsigned char* diag;
    double *thetax, *thetay, *jac, *pre;
    int nset, n, ntd, nfd;
    double half_df, jac_cap, jac_out;
};

// calc_SS's loop body per (set, itd, ifd), in the reference's IEEE order, and the two
// interpolations at (thetax, +-thetay) times the Jacobian, summed: SS before the flip
__global__ void br_query_kernel(BrQuery a) {
    const long long nq = (long long)a.ntd * a.nfd, m = nq * a.nset;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        const long long z = k / nq;
        const int r = (int)((k % nq) / a.nfd), c = (int)(k % a.nfd);
        const double* p = a.par + z * SB_BRIGHT_NPAR;
        const double thx = a.colx[z * a.nfd + c];
        // td - (thetax + thetagx)**2 + thetarx**2 + thetary**2
        const double s = __dadd_rn(__dadd_rn(__dsub_rn(a.td[r], a.colq[z * a.nfd + c]), p[5]),
                                   p[6]);
        double thy = 0.0, amp;
        if (s > 0) {
            const double t = __dsqrt_rn(s);
            thy = __dadd_rn(0.0, __dsub_rn(t, p[4]));
            amp = t < a.half_df ? a.jac_cap : __ddiv_rn(1.0, t);
        } else {
            amp = a.jac_out;
        }
        const double* B = a.B + z * (long long)a.n * a.n;
        const double g1 = br_interp(a.x, a.n, a.diag, B, thx, thy);
        const double g2 = br_interp(a.x, a.n, a.diag, B, thx, -thy);
        a.thetax[k] = thx;
        a.thetay[k] = thy;
        a.jac[k] = amp;
        a.pre[k] = __dadd_rn(__dmul_rn(g1, amp), __dmul_rn(g2, amp));
    }
}

// SS[1:, 1:] = pre[1:, 1:] + flip(pre[1:, 1:]); LSS = 10*log10(SS)
__global__ void br_flip_kernel(int nset, int ntd, int nfd, const double* __restrict__ pre,
                               double* __restrict__ ss, double* __restrict__ lss) {
    const long long nq = (long long)ntd * nfd, m = nq * nset;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        const long long z = k / nq;
        const int r = (int)((k % nq) / nfd), c = (int)(k % nfd);
        double v = pre[k];
        if (r > 0 && c > 0) v = __dadd_rn(v, pre[z * nq + (long long)(ntd - r) * nfd + (nfd - c)]);
        ss[k] = v;
        lss[k] = __dmul_rn(10.0, log10(v));
    }
}

// acf[z] /= max(acf[z]): the set's tile maxima in a fixed order (max is exact), then the
// correctly rounded division numpy does
__global__ void br_normalise_kernel(double* __restrict__ acf, long long nq,
                                    const double* __restrict__ cmax, int ntile) {
    SB_SHARED double s_max;
    const long long z = blockIdx.y;
    if (threadIdx.x < 32) {
        double mx = -INFINITY;
        for (int t = threadIdx.x; t < ntile; t += 32) mx = br_max(mx, cmax[z * ntile + t]);
        for (int o = 16; o > 0; o >>= 1) mx = br_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (threadIdx.x == 0) s_max = mx;
    }
    __syncthreads();
    const double mx = s_max;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nq;
         k += (long long)gridDim.x * blockDim.x)
        acf[z * nq + k] = __ddiv_rn(acf[z * nq + k], mx);
}

#ifndef SB_HOST_EMU

static unsigned br_blocks(long long m) {
    const long long b = (m + 255) / 256, cap = (long long)num_sms() * 16;
    return (unsigned)(b < cap ? (b > 0 ? b : 1) : cap);
}

static dim3 br_grid(int M, int N, int nset) {
    return dim3((unsigned)((N + BR_BN - 1) / BR_BN), (unsigned)((M + BR_BM - 1) / BR_BM),
                (unsigned)nset);
}

int brightness(const sb_brightness* d, cudaStream_t st) {
    SB_ARG(d != nullptr);
    const int stg = d->stages;
    SB_ARG(stg >= 1 && stg <= 7);
    if (d->nset < 1 || d->nset > 65535 || d->n < 2 || d->n > SB_BRIGHT_MAX_N || d->ntd < 1 ||
        d->ntd > SB_BRIGHT_MAX_Q || d->nfd < 1 || d->nfd > SB_BRIGHT_MAX_Q) {
        set_error("brightness: %d sets (1..65535), lattice %d (2..%d), %d x %d queries "
                  "(1..%d each)", d->nset, d->n, SB_BRIGHT_MAX_N, d->ntd, d->nfd,
                  SB_BRIGHT_MAX_Q);
        return SB_ERR_UNSUPPORTED;
    }
    SB_ARG(!(stg & SB_BRIGHT_EFIELD) || (d->x && d->par && d->rho && d->B));
    SB_ARG(!(stg & SB_BRIGHT_SSPEC) || (d->x && d->diag && d->td && d->par && d->colx &&
                                        d->colq && d->B && d->thetax && d->thetay && d->jac &&
                                        d->ss && d->lss));
    SB_ARG(!(stg & SB_BRIGHT_ACF) || (d->ss && d->acf));
    const int n = d->n, ntd = d->ntd, nfd = d->nfd, ns = d->nset;
    const long long n2 = (long long)n * n, nq = (long long)ntd * nfd;
    if (stg & SB_BRIGHT_EFIELD) {
        double* w = (double*)workspace(WS_PLANE0, 2 * n2 * sizeof(double));
        double* t = (double*)workspace(WS_PLANE1, 2 * n2 * ns * sizeof(double));
        if (!w || !t) return SB_ERR_NOMEM;
        br_rho_kernel<<<br_blocks(n2 * ns), 256, 0, st>>>(ns, n, d->x, d->par, d->rho);
        SB_LAUNCH_CHECK();
        // B[i][k] = |sum W^((i+h)(m1+h)) W^((k+h)(m2+h)) rho[m1][m2]|: W is symmetric
        br_twiddle_kernel<<<br_blocks(n2), 256, 0, st>>>(n, n / 2, n / 2, w, w + n2);
        SB_LAUNCH_CHECK();
        BrGemm g1{w, w + n2, d->rho, nullptr, t, t + n2 * ns, nullptr, 0, n2, n2, n, n, n};
        br_gemm_kernel<false, BR_STORE><<<br_grid(n, n, ns), BR_THREADS, 0, st>>>(g1);
        SB_LAUNCH_CHECK();
        BrGemm g2{t, t + n2 * ns, w, w + n2, d->B, nullptr, nullptr, n2, 0, n2, n, n, n};
        br_gemm_kernel<true, BR_ABS><<<br_grid(n, n, ns), BR_THREADS, 0, st>>>(g2);
        SB_LAUNCH_CHECK();
    }
    if (stg & SB_BRIGHT_SSPEC) {
        double* pre = (double*)workspace(WS_PLANE2, nq * ns * sizeof(double));
        if (!pre) return SB_ERR_NOMEM;
        BrQuery a{d->x, d->td, d->colx, d->colq, d->par, d->B, d->diag, d->thetax, d->thetay,
                  d->jac, pre, ns, n, ntd, nfd, d->half_df, d->jac_cap, d->jac_out};
        br_query_kernel<<<br_blocks(nq * ns), 256, 0, st>>>(a);
        SB_LAUNCH_CHECK();
        br_flip_kernel<<<br_blocks(nq * ns), 256, 0, st>>>(ns, ntd, nfd, pre, d->ss, d->lss);
        SB_LAUNCH_CHECK();
    }
    if (stg & SB_BRIGHT_ACF) {
        const long long m1 = (long long)ntd * ntd, m2 = (long long)nfd * nfd;
        const dim3 grid = br_grid(ntd, nfd, ns);
        const int ntile = (int)(grid.x * grid.y);
        double* w = (double*)workspace(WS_PLANE0, 2 * (m1 + m2) * sizeof(double));
        double* t = (double*)workspace(WS_PLANE1, 2 * nq * ns * sizeof(double));
        double* cmax = (double*)workspace(WS_PLANE3, (size_t)ntile * ns * sizeof(double));
        if (!w || !t || !cmax) return SB_ERR_NOMEM;
        double *w1 = w, *w2 = w + 2 * m1;
        const int h1 = ntd / 2, h2 = nfd / 2;
        // acf[i][k] = re sum W1^((i-h1)(m1+h1)) W2^((k-h2)(m2+h2)) ss[m1][m2]; the second
        // factor is stored transposed, [m2][k]
        br_twiddle_kernel<<<br_blocks(m1), 256, 0, st>>>(ntd, ntd - h1, h1, w1, w1 + m1);
        SB_LAUNCH_CHECK();
        br_twiddle_kernel<<<br_blocks(m2), 256, 0, st>>>(nfd, h2, nfd - h2, w2, w2 + m2);
        SB_LAUNCH_CHECK();
        BrGemm g1{w1, w1 + m1, d->ss, nullptr, t, t + nq * ns, nullptr, 0, nq, nq, ntd, nfd, ntd};
        br_gemm_kernel<false, BR_STORE><<<grid, BR_THREADS, 0, st>>>(g1);
        SB_LAUNCH_CHECK();
        BrGemm g2{t, t + nq * ns, w2, w2 + m2, d->acf, nullptr, cmax, nq, 0, nq, ntd, nfd, nfd};
        br_gemm_kernel<true, BR_REAL><<<grid, BR_THREADS, 0, st>>>(g2);
        SB_LAUNCH_CHECK();
        const long long per = (nq + 2047) / 2048;
        br_normalise_kernel<<<dim3((unsigned)(per < 1024 ? per : 1024), (unsigned)ns), 256, 0,
                              st>>>(d->acf, nq, cmax, ntile);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
