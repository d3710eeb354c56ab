// scint_sim.Simulation on the device (reference: scintools/scint_sim.py).
//
//   screen   : w (spectral amplitude, :169-198 + swdsp :276-292) in fp64,
//              xyp = real(fft2(w * (n1 + i n2))) in fp64 (:201-204)
//   intensity: per frequency s: E = exp(i xyp s) -> fft2 -> Fresnel filter
//              (frfilt3 :294-311) -> ifft2 -> column ny/2 (:226-230).
//              Only column ny/2 of the inverse transform is used, and
//              exp(2 pi i ky (ny/2)/ny) = (-1)^ky, so the inverse collapses to a
//              filtered, sign-alternating sum over ky followed by ONE 1-D
//              inverse FFT over kx.  The transform order is x (strided axis,
//              four-step tiles, exp(i phi s) fused into the first load) then
//              y (contiguous rows in shared memory, reduction fused into the
//              epilogue), so the 8192^2 field makes 2.5 HBM round trips per
//              frequency instead of 6.  The last frequency also produces
//              xyi = |ifft2(.)|^2 (:232) through the full inverse.
#include <math.h>

#include "fft_kernels.cuh"

namespace sb {

struct SimParams {
    int nx, ny;
    double dx, dy, alpha, ar, psi, inner, consp;
};

// ------------------------------------------------------------------ weights
__device__ __forceinline__ double swdsp(const SimParams& p, double kx, double ky) {
    const double pi = 3.14159265358979323846;
    const double cs = cos(p.psi * pi / 180), sn = sin(p.psi * pi / 180);
    const double r = p.ar;
    const double con = sqrt(p.consp);
    const double alf = -(p.alpha + 2) / 4;
    const double a = (cs * cs) / r + r * sn * sn;
    const double b = r * cs * cs + sn * sn / r;
    const double c = 2 * cs * sn * (1 / r - r);
    const double q2 = a * kx * kx + b * ky * ky + c * kx * ky;
    return con * pow(q2, alf) * exp(-(kx * kx + ky * ky) * p.inner * p.inner / 2);
}

// closed form of the quadrant-mirroring loops of get_screen (:178-198),
// including the ky=0 off-by-one (:185) and the overwrite order at c = ny/2.
__global__ void sim_weights_kernel(SimParams p, double* __restrict__ w) {
    const long total = (long)p.nx * p.ny;
    const double pi = 3.14159265358979323846;
    const double dqx = 2 * pi / (p.dx * p.nx), dqy = 2 * pi / (p.dy * p.ny);
    const int nx = p.nx, ny = p.ny, hx = nx / 2, hy = ny / 2;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / ny), c = (int)(i % ny);
        double v;
        if (c == 0) {
            if (r == 0 || r == hx) v = 0.0;
            else if (r < hx) v = swdsp(p, r * dqx, 0.0);
            else v = swdsp(p, (nx + 1 - r) * dqx, 0.0);
        } else if (r == 0) {
            v = swdsp(p, 0.0, (c <= hy ? c : ny - c) * dqy);
        } else if (c < hy) {
            v = swdsp(p, (r <= hx ? r : -(nx - r)) * dqx, c * dqy);
        } else if (c == hy) {
            v = swdsp(p, (r <= hx ? r : nx - r) * dqx, hy * dqy);
        } else {
            v = swdsp(p, (r >= hx ? nx - r : -r) * dqx, (ny - c) * dqy);
        }
        w[i] = v;
    }
}

// --------------------------------------------------------------- device RNG
// Philox4x32-10 counter RNG + Box-Muller: statistically equivalent noise for
// throughput runs.  (Parity runs pass the legacy MT19937 fields from the host.)
__device__ __forceinline__ void philox_round(unsigned (&c)[4], unsigned k0, unsigned k1) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * c[0];
    const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * c[2];
    const unsigned n0 = (unsigned)(p1 >> 32) ^ c[1] ^ k0;
    const unsigned n1 = (unsigned)p1;
    const unsigned n2 = (unsigned)(p0 >> 32) ^ c[3] ^ k1;
    const unsigned n3 = (unsigned)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ __forceinline__ void philox4(unsigned long long ctr, unsigned long long seed,
                                        unsigned (&out)[4]) {
    unsigned c[4] = {(unsigned)ctr, (unsigned)(ctr >> 32), 0u, 0u};
    unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}
__device__ __forceinline__ double2 gauss_pair(unsigned long long idx, unsigned long long seed) {
    unsigned r[4];
    philox4(idx, seed, r);
    const double u1 = ((double)r[0] * 4294967296.0 + (double)r[1] + 0.5) * (1.0 / 18446744073709551616.0);
    const double u2 = ((double)r[2] * 4294967296.0 + (double)r[3] + 0.5) * (1.0 / 18446744073709551616.0);
    const double rad = sqrt(-2.0 * log(u1));
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    return make_double2(rad * c, rad * s);
}

// ------------------------------------------------------------ screen (fp64)
struct ScreenRowLoad {   // z[x][y] = w * (n1 + i n2)
    const double* w;
    const double* n1;
    const double* n2;
    unsigned long long seed;
    int ny;
    __device__ __forceinline__ double2 operator()(long row, int n) const {
        const size_t i = (size_t)row * ny + n;
        const double ww = w[i];
        double2 g = n1 ? make_double2(n1[i], n2[i]) : gauss_pair(i, seed);
        return make_double2(ww * g.x, ww * g.y);
    }
};
struct RealPartStore {   // xyp[k][c] = Re X[k][c], k = k1 + R1 k2
    double* out;
    long pitch;
    int R1;
    __device__ __forceinline__ void operator()(int y, int k, int c, double2 v) const {
        out[(size_t)(y + R1 * k) * pitch + c] = v.x;
    }
};

int sim_weights(const SimParams& p, double* w, cudaStream_t st) {
    if (p.nx < 4 || p.ny < 4 || (p.nx & 1) || (p.ny & 1)) {
        set_error("Simulation: nx, ny must be even and >= 4");
        return SB_ERR_UNSUPPORTED;
    }
    sim_weights_kernel<<<num_sms() * 8, 256, 0, st>>>(p, w);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// xyp = real(fft2(w * noise)), all fp64
int sim_screen(int nx, int ny, const double* w, const double* n1, const double* n2,
               unsigned long long seed, double* xyp, cudaStream_t st) {
    ProfScope prof(PROF_SIM_SCREEN, st);
    if (!is_pow2(nx) || !is_pow2(ny) || ny < 8 || ny > 8192 || nx < 4 || nx > 65536) {
        set_error("Simulation screen: %dx%d unsupported (powers of two, nx 4..65536, ny 8..8192)",
                  nx, ny);
        return SB_ERR_UNSUPPORTED;
    }
    double2* B1 = (double2*)workspace(3, (size_t)nx * ny * sizeof(double2));
    double2* B2 = (double2*)workspace(4, (size_t)nx * ny * sizeof(double2));
    if (!B1 || !B2) return SB_ERR_NOMEM;
    ScreenRowLoad ld{w, n1, n2, seed, ny};
    PlainRowStore<double2> rs{B1, ny};
    int rc = SB_OK;
    SB_ROW_DISPATCH(ny, rc = (launch_row_c2c<double, N1, N2, -1>(ld, rs, nx, st)));
    if (rc) return rc;
    int R1, R2;
    split_len(nx, &R1, &R2);
    StrideALoad<double2> la{B1, ny, R2};
    RealPartStore sb{xyp, ny, R1};
    return cols_generic<double, -1>(la, B2, ny, nx, ny, sb, st);
}

// ------------------------------------------------------- intensity (fp32)
struct FieldALoad {   // exp(i * xyp * scale), x-axis pass A: y = r2, i = r1
    const double* xyp;
    long pitch;
    int R2;
    double scale;
    __device__ __forceinline__ float2 operator()(int y, int i, int c) const {
        const double phi = xyp[(size_t)(i * R2 + y) * pitch + c] * scale;
        // range-reduce in fp64, evaluate in fp32
        const double t = phi * 0.15915494309189533577;   // / 2 pi
        const float r = (float)((t - rint(t)) * 6.28318530717958647692);
        float s, cc;
        sincosf(r, &s, &cc);
        return make_float2(cc, s);
    }
};

// Fresnel filter tables for one frequency (frfilt3 :294-311):
//   fx[kx] = exp(-i s ffconx kx'^2), kx' = min(kx, nx - kx)
//   fy[ky] = exp(-i s ffcony ky'^2) * (-1)^ky   (sign = column ny/2 of the inverse)
//   fyp[ky] = same without the sign (full inverse of the last frequency)
__global__ void sim_filter_kernel(int nx, int ny, double scale, double ffconx,
                                  double ffcony, float2* __restrict__ fx,
                                  float2* __restrict__ fy, float2* __restrict__ fyp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nx) {
        const double k = (double)(i <= nx / 2 ? i : nx - i);
        double s, c;
        sincos(k * k * scale * ffconx, &s, &c);
        fx[i] = make_float2((float)c, (float)-s);
    }
    if (i < ny) {
        const double k = (double)(i <= ny / 2 ? i : ny - i);
        double s, c;
        sincos(ffcony * (k * k) * scale, &s, &c);
        const float sg = (i & 1) ? -1.f : 1.f;
        fyp[i] = make_float2((float)c, (float)-s);
        fy[i] = make_float2(sg * (float)c, sg * (float)-s);
    }
}

// y-axis FFT of one row kx, then g[kx] = fx[kx] * sum_ky X[kx][ky] fy[ky]
template <int N1, int N2>
__global__ void __launch_bounds__(1024)
sim_row_reduce_kernel(const float2* __restrict__ in, long pitch,
                      const float2* __restrict__ fx, const float2* __restrict__ fy,
                      float2* __restrict__ g, float2* __restrict__ full,
                      const float2* __restrict__ fyp, RowTables<float> tabs) {
    using C = float2;
    constexpr int N = N1 * N2, RS = N2 + 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    C* tw1 = s + N1 * RS; C* tw2 = tw1 + N1; C* twl = tw2 + N2;
    __shared__ float redx[32], redy[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    const long row = blockIdx.x;
    row_load_tables<float, N1, N2, -1>(tw1, tw2, twl, tabs.wN, tid, nt);
    for (int n = tid; n < N; n += nt) s[row_in_pos<float, N1, N2>(n)] = in[row * pitch + n];
    __syncthreads();
    row_fft_smem<float, N1, N2, -1>(s, tw1, tw2, twl, tid, nt);
    const C fxr = fx[row];
    float ax = 0.f, ay = 0.f;
    for (int k = tid; k < N; k += nt) {
        const C v = s[row_out_pos<float, N1, N2>(k)];
        const C f = fy[k];
        ax += v.x * f.x - v.y * f.y;
        ay += v.x * f.y + v.y * f.x;
        if (full) full[row * pitch + k] = cmul(cmul(v, fyp[k]), fxr);
    }
    ax = warp_sum(ax);
    ay = warp_sum(ay);
    if ((tid & 31) == 0) { redx[tid >> 5] = ax; redy[tid >> 5] = ay; }
    __syncthreads();
    if (tid == 0) {
        float sx = 0.f, sy = 0.f;
        for (int k = 0; k < (nt + 31) / 32; ++k) { sx += redx[k]; sy += redy[k]; }
        g[row] = cmul(make_float2(sx, sy), fxr);
    }
}

struct GRowLoad {
    const float2* g;
    int nx;
    __device__ __forceinline__ float2 operator()(long row, int n) const {
        return g[(size_t)row * nx + n];
    }
};
struct SpeRowStore {   // spe_t[f][x] = z / (nx ny)
    float2* spe;
    int nx;
    float scale;
    __device__ __forceinline__ void operator()(long row, int k, float2 v) const {
        spe[(size_t)row * nx + k] = make_float2(v.x * scale, v.y * scale);
    }
};
struct PowerBStore {     // xyi[k][c] = |v|^2 * scale^2
    float* out;
    long pitch;
    int R1;
    float scale2;
    __device__ __forceinline__ void operator()(int y, int k, int c, float2 v) const {
        out[(size_t)(y + R1 * k) * pitch + c] = (v.x * v.x + v.y * v.y) * scale2;
    }
};

// spe_t [nf][nx] complex64 (= reference spe transposed), xyi [nx][ny] or null
int sim_intensity(int nx, int ny, int nf, const double* xyp, const double* scales_host,
                  double ffconx, double ffcony, float2* spe_t, float* xyi,
                  cudaStream_t st) {
    if (!is_pow2(nx) || !is_pow2(ny) || ny < 8 || ny > 16384 || nx < 8 || nx > 16384) {
        set_error("Simulation intensity: %dx%d unsupported (powers of two, 8..16384)", nx, ny);
        return SB_ERR_UNSUPPORTED;
    }
    const size_t fld = (size_t)nx * ny * sizeof(float2);
    float2* B1 = (float2*)workspace(5, fld);
    float2* B2 = (float2*)workspace(6, fld);
    float2* tabs_ = (float2*)workspace(7, (size_t)(nx + 2 * ny + (size_t)nf * nx) * sizeof(float2));
    if (!B1 || !B2 || !tabs_) return SB_ERR_NOMEM;
    float2* fx = tabs_;
    float2* fy = fx + nx;
    float2* fyp = fy + ny;
    float2* G = fyp + ny;           // [nf][nx]
    int R1, R2;
    split_len(nx, &R1, &R2);
    RowTables<float> rt;
    rt.wN = twiddle_table<float>(ny, -1, st);
    rt.w2N = nullptr;
    if (!rt.wN) return SB_ERR_NOMEM;
    for (int f = 0; f < nf; ++f) {
        ProfScope prof(PROF_SIM_FREQ, st);
        const double scale = scales_host[f];
        const bool last = (f == nf - 1) && xyi != nullptr;
        sim_filter_kernel<<<(max(nx, ny) + 255) / 256, 256, 0, st>>>(nx, ny, scale, ffconx,
                                                                     ffcony, fx, fy, fyp);
        SB_LAUNCH_CHECK();
        // x axis (strided): exp(i phi s) fused into the first load
        FieldALoad la{xyp, ny, R2, scale};
        NaturalBStore<float2> nb{B2, ny, R1};
        int rc = cols_generic<float, -1>(la, B1, ny, nx, ny, nb, st);
        if (rc) return rc;
        // y axis (contiguous) + filtered reduction over ky
        SB_ROW_DISPATCH(ny, {
            auto kern = sim_row_reduce_kernel<N1, N2>;
            const size_t smem = RowSmem<float, N1, N2>::bytes;
            SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<nx, row_threads(ny), smem, st>>>(B2, ny, fx, fy, G + (size_t)f * nx,
                                                    last ? B1 : nullptr, fyp, rt);
        });
        SB_LAUNCH_CHECK();
        if (last) {
            // full inverse of the filtered spectrum (in B1): rows then columns
            PitchRowLoad<float2> fl{B1, ny};
            PlainRowStore<float2> ps{B2, ny};
            SB_ROW_DISPATCH(ny, rc = (launch_row_c2c<float, N1, N2, +1>(fl, ps, nx, st)));
            if (rc) return rc;
            StrideALoad<float2> sl{B2, ny, R2};
            const float sc = 1.0f / ((float)nx * (float)ny);
            PowerBStore pb{xyi, ny, R1, sc * sc};
            rc = cols_generic<float, +1>(sl, B1, ny, nx, ny, pb, st);
            if (rc) return rc;
        }
    }
    // spe[:, f] = ifft over kx of g_f  (batched rows of length nx)
    GRowLoad gl{G, nx};
    SpeRowStore ss{spe_t, nx, 1.0f / ((float)nx * (float)ny)};
    int rc = SB_OK;
    SB_ROW_DISPATCH(nx, rc = (launch_row_c2c<float, N1, N2, +1>(gl, ss, nf, st)));
    return rc;
}

}  // namespace sb
