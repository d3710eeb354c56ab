// The theoretical intensity ACF of scint_sim.ACF (include/scint_b200.h, sb_acf_model_f64).
// Everything is float64.
//
// For a time lag s (positions sx, sy) and a frequency lag nu > 0 the reference sums, over the
// tensor grid (x, y) = (snp[j], snp[i]),
//     S = sum_{i,j} G[i][j] exp(i ((x - sx)^2 + (y - sy)^2) / (2 nu))
// with G the e-field ACF.  The exponential factors into ex[j] = exp(i (snp[j] - sx)^2 / (2 nu))
// and ey[i] = exp(i (snp[i] - sy)^2 / (2 nu)), so S = ey^T G ex: 2n sincos per lag instead of
// n^2, and the rest is a real-times-complex matrix product.
//
// Three launches:
//   gauss     G on the main grid (into `efield`) and on the core grid (workspace)
//   contract  one block per (column, lag tile, row-tile range) of a host-built table: for its
//             AM_TS lags and its AM_TI-row tiles, T = G[rows][:] ex (ex made on the fly, one
//             AM_TJ chunk at a time), then the partial ey^T T over its rows
//   finish    one thread per (lag, column): column 0 in closed form (+ wn/amp at the
//             reference's rows), the others as the sum of their partials in table order, then
//             amp |gamma|^2 written to every position the reference's mirroring puts it
// No atomics, and the table depends on the shapes only, so a repeated call is bit-identical.
#include <math.h>

#include <vector>

#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int AM_TI = 64;              // grid rows per tile
constexpr int AM_TS = 32;              // lags per tile
constexpr int AM_TJ = 32;              // grid columns per chunk
constexpr int AM_THREADS = 256;        // 16 x 16: 4 rows x 2 lags per thread
constexpr int AM_TARGET_BLOCKS = 1056; // enough blocks for 8 per SM on 132 SMs

struct AmBlock {
    int col, lt, i0, i1;               // column >= 1, lag tile, row tiles [i0, i1)
};

// The contract table: main-grid columns split their row tiles into P1 ranges so the launch
// has about AM_TARGET_BLOCKS blocks; the core column (1) into as many as give its blocks the
// work of a main-grid block.  range[(col - 1) * nst + lt] = {first block, count}.
struct AmPlan {
    std::vector<AmBlock> blocks;
    std::vector<int2> range;
};

inline void am_plan(int n1, int n2, int ndnun, int nsn, AmPlan& p) {
    const long long nst = (nsn + AM_TS - 1) / AM_TS;
    const long long it1 = (n1 + AM_TI - 1) / AM_TI, it2 = (n2 + AM_TI - 1) / AM_TI;
    long long p1 = (AM_TARGET_BLOCKS + (ndnun - 1) * nst - 1) / ((ndnun - 1) * nst);
    p1 = p1 < 1 ? 1 : (p1 > it1 ? it1 : p1);
    const long long work = (it1 + p1 - 1) / p1 * n1;       // one main-grid block's row work
    long long p2 = (it2 * n2 + work - 1) / work;
    p2 = p2 < 1 ? 1 : (p2 > it2 ? it2 : p2);
    p.blocks.clear();
    p.range.assign((size_t)((ndnun - 1) * nst), make_int2(0, 0));
    for (int col = 1; col < ndnun; ++col) {
        const long long it = col == 1 ? it2 : it1, pp = col == 1 ? p2 : p1;
        for (int lt = 0; lt < (int)nst; ++lt) {
            p.range[(size_t)((col - 1) * nst + lt)] = make_int2((int)p.blocks.size(), (int)pp);
            for (long long g = 0; g < pp; ++g)
                p.blocks.push_back(AmBlock{col, lt, (int)(g * it / pp), (int)((g + 1) * it / pp)});
        }
    }
}

// exp(-0.5 ((x / sqrtar)^2 + (y sqrtar)^2)^alph2), in the reference's order of operations
__device__ __forceinline__ double am_gauss(double x, double y, double sqrtar, double alph2) {
    const double a = x / sqrtar, b = __dmul_rn(y, sqrtar);
    return exp(-0.5 * pow(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), alph2));
}

// G[i][j] = am_gauss(snp[j], snp[i]) on both grids: flat index k < n1^2 the main grid, the
// rest the core grid
__global__ void am_gauss_kernel(const double* __restrict__ snp, int n1,
                                const double* __restrict__ snp2, int n2, double sqrtar,
                                double alph2, double* __restrict__ g1, double* __restrict__ g2) {
    const long long m1 = (long long)n1 * n1, m = m1 + (long long)n2 * n2;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m;
         k += (long long)gridDim.x * blockDim.x) {
        if (k < m1)
            g1[k] = am_gauss(snp[k % n1], snp[k / n1], sqrtar, alph2);
        else
            g2[k - m1] = am_gauss(snp2[(k - m1) % n2], snp2[(k - m1) / n2], sqrtar, alph2);
    }
}

// the lag position moved by the phase gradient, sn - 2 sig dnun (scint_sim.py:639-640,
// 646-647); with phasegrad == 0, sig is +-0 and the position is unchanged
__device__ __forceinline__ double am_shift(double sn, double sig, double nu) {
    return __dsub_rn(sn, __dmul_rn(2.0 * sig, nu));
}

// exp(i (p - s)^2 / (2 nu))
__device__ __forceinline__ double2 am_chirp(double p, double s, double twonu) {
    const double d = p - s;
    double sn, cs;
    sincos(__dmul_rn(d, d) / twonu, &sn, &cs);
    return make_double2(cs, sn);
}

struct AmArgs {
    const double *snp1, *snp2, *g1, *g2, *dnun, *snx, *sny;
    int n1, n2, nsn;
    double sigxn, sigyn;
};

// part[block][AM_TS]: the block's share of S for each lag of its tile
__global__ void __launch_bounds__(AM_THREADS)
am_contract_kernel(AmArgs a, const AmBlock* __restrict__ table, double2* __restrict__ part) {
    SB_SHARED double Gs[AM_TI][AM_TJ + 1];
    SB_SHARED double2 Es[AM_TJ][AM_TS];
    SB_SHARED double2 red[AM_THREADS / 16][AM_TS];
    const AmBlock b = table[blockIdx.x];
    const bool core = b.col == 1;
    const int n = core ? a.n2 : a.n1;
    const double* __restrict__ snp = core ? a.snp2 : a.snp1;
    const double* __restrict__ G = core ? a.g2 : a.g1;
    const double nu = a.dnun[b.col], twonu = 2.0 * nu;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int s0 = b.lt * AM_TS;
    // the y positions of this thread's two lags (lags past nsn have zero ex, so zero sums)
    double sy[2];
    for (int q = 0; q < 2; ++q) {
        const int s = s0 + tx + 16 * q < a.nsn ? s0 + tx + 16 * q : a.nsn - 1;
        sy[q] = am_shift(a.sny[s], a.sigyn, nu);
    }
    double2 tot[2] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0)};
    for (int itile = b.i0; itile < b.i1; ++itile) {
        const int r0 = itile * AM_TI;
        double2 acc[4][2];
        for (int p = 0; p < 4; ++p)
            for (int q = 0; q < 2; ++q) acc[p][q] = make_double2(0.0, 0.0);
        for (int j0 = 0; j0 < n; j0 += AM_TJ) {
            for (int e = tid; e < AM_TI * AM_TJ; e += AM_THREADS) {
                const int r = e / AM_TJ, c = e % AM_TJ;
                Gs[r][c] = (r0 + r < n && j0 + c < n) ? G[(long long)(r0 + r) * n + j0 + c] : 0.0;
            }
            for (int e = tid; e < AM_TJ * AM_TS; e += AM_THREADS) {
                const int c = e / AM_TS, l = e % AM_TS, s = s0 + l;
                Es[c][l] = (j0 + c < n && s < a.nsn)
                               ? am_chirp(snp[j0 + c], am_shift(a.snx[s], a.sigxn, nu), twonu)
                               : make_double2(0.0, 0.0);
            }
            __syncthreads();
            for (int c = 0; c < AM_TJ; ++c) {
                double g[4];
                double2 e[2];
                for (int p = 0; p < 4; ++p) g[p] = Gs[ty + 16 * p][c];
                for (int q = 0; q < 2; ++q) e[q] = Es[c][tx + 16 * q];
                for (int p = 0; p < 4; ++p)
                    for (int q = 0; q < 2; ++q) {
                        acc[p][q].x = fma(g[p], e[q].x, acc[p][q].x);
                        acc[p][q].y = fma(g[p], e[q].y, acc[p][q].y);
                    }
            }
            __syncthreads();
        }
        // ey^T T over this tile's rows
        for (int p = 0; p < 4; ++p) {
            const int i = r0 + ty + 16 * p;
            if (i >= n) continue;
            for (int q = 0; q < 2; ++q) {
                const double2 ey = am_chirp(snp[i], sy[q], twonu);
                tot[q].x += ey.x * acc[p][q].x - ey.y * acc[p][q].y;
                tot[q].y += ey.x * acc[p][q].y + ey.y * acc[p][q].x;
            }
        }
    }
    for (int q = 0; q < 2; ++q) red[ty][tx + 16 * q] = tot[q];
    __syncthreads();
    if (tid < AM_TS) {
        double2 s = make_double2(0.0, 0.0);
        for (int r = 0; r < AM_THREADS / 16; ++r) {
            s.x += red[r][tid].x;
            s.y += red[r][tid].y;
        }
        part[(long long)blockIdx.x * AM_TS + tid] = s;
    }
}

struct AmFinish {
    const double *dnun, *snx, *sny;
    const double2* part;
    const int2* range;
    int ndnun, nsn, quadrant;
    double sqrtar, alph2, step1, step2, wn_amp, amp;
};

// acf [2 ndnun - 1][nt_out]: nt_out = 2 nsn - 1 (quadrant, scint_sim.py:611-622) or nsn
// (half plane, :659-663)
__global__ void am_finish_kernel(AmFinish f, double* __restrict__ acf) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)f.nsn * f.ndnun) return;
    const int r = (int)(k / f.ndnun), c = (int)(k % f.ndnun);
    double v;
    if (c == 0) {
        double g = am_gauss(f.snx[r], f.sny[r], f.sqrtar, f.alph2);
        if (f.quadrant ? r == 0 : f.snx[r] == 0.0) g += f.wn_amp;
        v = g * g;
    } else {
        const int nst = (f.nsn + AM_TS - 1) / AM_TS;
        const int2 rg = f.range[(long long)(c - 1) * nst + r / AM_TS];
        double2 s = make_double2(0.0, 0.0);
        for (int b = 0; b < rg.y; ++b) {
            const double2 p = f.part[(long long)(rg.x + b) * AM_TS + r % AM_TS];
            s.x += p.x;
            s.y += p.y;
        }
        // -1j ((dsp / fac)^2 sum / ((2 pi) dnun)); |.|^2
        const double h = c == 1 ? f.step2 : f.step1;
        const double den = 6.283185307179586 * f.dnun[c];
        const double re = h * h * s.x / den, im = h * h * s.y / den;
        v = re * re + im * im;
    }
    v *= f.amp;
    const int nc = f.ndnun;
    if (f.quadrant) {
        const int nr = f.nsn, nt = 2 * nr - 1;
        for (int sf = -1; sf <= 1; sf += 2)
            for (int st = -1; st <= 1; st += 2)
                acf[(long long)(nc - 1 + sf * c) * nt + (nr - 1 + st * r)] = v;
    } else {
        const int nt = f.nsn;
        acf[(long long)(nc - 1 + c) * nt + r] = v;
        if (c > 0) acf[(long long)(nc - 1 - c) * nt + (nt - 1 - r)] = v;
    }
}

#ifndef SB_HOST_EMU

int acf_model(const sb_acf_model* m, double* acf, double* efield, cudaStream_t st) {
    SB_ARG(m && acf && efield && m->snp && m->snp2 && m->dnun && m->snx && m->sny);
    if (m->n1 < 1 || m->n1 > 16384 || m->n2 < 1 || m->n2 > 16384 || m->ndnun < 2 ||
        m->ndnun > 4096 || m->nsn < 1 || m->nsn > 8191) {
        set_error("acf_model: grids %d, %d (1..16384), %d frequency lags (2..4096), %d time "
                  "lags (1..8191)", m->n1, m->n2, m->ndnun, m->nsn);
        return SB_ERR_UNSUPPORTED;
    }
    AmPlan plan;
    am_plan(m->n1, m->n2, m->ndnun, m->nsn, plan);
    const size_t nb = plan.blocks.size(), nr = plan.range.size();
    const size_t bytes = (size_t)m->n2 * m->n2 * sizeof(double) + nb * AM_TS * sizeof(double2) +
                         nb * sizeof(AmBlock) + nr * sizeof(int2) + 4 * 16;
    char* w = (char*)workspace(WS_PLANE0, bytes);
    if (!w) return SB_ERR_NOMEM;
    auto take = [&](size_t b) { char* p = w; w += (b + 15) & ~size_t(15); return p; };
    double* g2 = (double*)take((size_t)m->n2 * m->n2 * sizeof(double));
    double2* part = (double2*)take(nb * AM_TS * sizeof(double2));
    AmBlock* d_blocks = (AmBlock*)take(nb * sizeof(AmBlock));
    int2* d_range = (int2*)take(nr * sizeof(int2));
    SB_CUDA(cudaMemcpyAsync(d_blocks, plan.blocks.data(), nb * sizeof(AmBlock),
                            cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemcpyAsync(d_range, plan.range.data(), nr * sizeof(int2),
                            cudaMemcpyHostToDevice, st));
    am_gauss_kernel<<<num_sms() * 8, 256, 0, st>>>(m->snp, m->n1, m->snp2, m->n2, m->sqrtar,
                                                   m->alph2, efield, g2);
    SB_LAUNCH_CHECK();
    AmArgs a{m->snp, m->snp2, efield, g2, m->dnun, m->snx, m->sny, m->n1, m->n2, m->nsn,
             m->sigxn, m->sigyn};
    am_contract_kernel<<<(unsigned)nb, AM_THREADS, 0, st>>>(a, d_blocks, part);
    SB_LAUNCH_CHECK();
    AmFinish f{m->dnun, m->snx, m->sny, part, d_range, m->ndnun, m->nsn, m->quadrant != 0,
               m->sqrtar, m->alph2, m->step1, m->step2, m->wn_amp, m->amp};
    const long long nk = (long long)m->nsn * m->ndnun;
    am_finish_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(f, acf);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
