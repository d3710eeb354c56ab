// Wavefield mosaic of half-overlapping chunks: the stacking, coherence and chi-square
// passes behind ththmod.rotInit / rotMos / rotFit / rotDer / fullMos / fullMosFit /
// fullMosGrad / fullMosHess (include/scint_b200.h, sb_mosaic_*).
//
// Geometry.  ncf x nct chunks of cwf x cwt (float2 [P][cwf][cwt], k = cf * nct + ct).
// Chunk (cf, ct) covers mosaic rows cf*hf .. cf*hf+cwf and columns ct*ht .. ct*ht+cwt
// with hf = cwf/2, ht = cwt/2; an axis with one chunk has no overlap and its tile extent
// is the whole width.  The mosaic splits into tf x tt half-tiles of hf x ht pixels
// (tf = ncf+1, or 1 for a single chunk).  Tile (a, b) is covered by at most four chunks,
// slot s = 2*si + sj holding chunk (a-1+si, b-1+sj); slot order is chunk order.
// Chunk cf's weight on its first half is the rising sin^2 ramp (if cf > 0), on its second
// half one minus that ramp (if cf < ncf-1), separably in time: the ramps of overlapping
// chunks add up to one.
//
// Every pass is one thread block per tile (grid-stride over tiles, 128 threads, pixels
// strided over the threads).  The ramps are evaluated in float64 once per block and
// rounded to float32; each pixel is float32 arithmetic; every thread accumulates in
// float64, the block reduces in a fixed order and writes the tile's partial sums.  A
// second kernel adds each chunk's (or pair's) partials from its at most four tiles in a
// fixed order, so every result is deterministic.  Counts live in grid.x or in loops.
#include "common.cuh"
#include "drivers.cuh"

namespace sb {

constexpr int MOS_THREADS = 128;
constexpr int MOS_MAX_TILE = 2048;   // tile extent per axis (ramps live in shared memory)

enum MosMode { MOS_BUILD = 0, MOS_ROT = 1, MOS_OVERLAP = 2, MOS_FIT = 3, MOS_HESS = 4 };

// partial sums per tile
template <int MODE> struct MosNq { static constexpr int value = 1; };
template <> struct MosNq<MOS_ROT> { static constexpr int value = 5; };       // sum|W|^2, Im(conj W y_s)
template <> struct MosNq<MOS_OVERLAP> { static constexpr int value = 12; };  // 6 pairs, re / im
template <> struct MosNq<MOS_FIT> { static constexpr int value = 9; };       // chi2, gA_s, gP_s
template <> struct MosNq<MOS_HESS> { static constexpr int value = 44; };     // 6 pairs x 4 + 4 x 5

struct MosGeom {
    int ncf, nct, cwf, cwt;
    int hf, ht, tf, tt;
    long long nF, nT;      // mosaic rows / columns
    long long ntiles;
};

// index of the slot pair (u < v) in a tile
__device__ __forceinline__ int mos_pair_index(int u, int v) {
    return u == 0 ? v - 1 : (u == 1 ? v + 1 : 5);
}

__device__ __forceinline__ float mos_fac(int s_hi, int c, int n, const float* up, const float* dn,
                                         int i) {
    // s_hi: the tile is the chunk's first half (1) or second half (0)
    if (s_hi) return c > 0 ? up[i] : 1.0f;
    return c < n - 1 ? dn[i] : 1.0f;
}

template <int NQ>
__device__ __forceinline__ void mos_block_store(double (&acc)[NQ], double* out) {
    SB_SHARED double red[MOS_THREADS / 32][NQ];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        const double v = warp_sum(acc[q]);
        if (lane == 0) red[w][q] = v;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < NQ; q += blockDim.x) {
        double v = red[0][q];
        for (int ww = 1; ww < MOS_THREADS / 32; ++ww) v += red[ww][q];
        out[q] = v;
    }
    __syncthreads();
}

// One pass over the half-tiles.  chunks float2 [P][cwf][cwt]; phi, amp float64 [P] (amp
// NULL: all ones); W float2 [nF][nT] (written by MOS_BUILD, read by ROT / FIT / HESS);
// dspec, noise float32 [nF][nT] (FIT / HESS); part float64 [ntiles][NQ].
template <int MODE>
__global__ void __launch_bounds__(MOS_THREADS)
mosaic_tile_kernel(MosGeom g, const float2* __restrict__ chunks, const double* __restrict__ phi,
                   const double* __restrict__ amp, float2* __restrict__ W,
                   const float* __restrict__ dspec, const float* __restrict__ noise,
                   double* __restrict__ part) {
    constexpr int NQ = MosNq<MODE>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* upf = reinterpret_cast<float*>(smem_raw);
    float* dnf = upf + g.hf;
    float* upt = dnf + g.hf;
    float* dnt = upt + g.ht;
    SB_SHARED float2 rot_s[4];
    SB_SHARED float amp_s[4];
    SB_SHARED int valid_s[4];
    // the reference's mask_func(h) = sin((pi/2) * i / h)^2 and 1 - mask_func(h), in float64
    for (int i = threadIdx.x; i < g.hf + g.ht; i += blockDim.x) {
        const int h = i < g.hf ? g.hf : g.ht;
        const int x = i < g.hf ? i : i - g.hf;
        const double s = sin((M_PI / 2) * (double)x / (double)h);
        const double up = s * s;
        if (i < g.hf) { upf[x] = (float)up; dnf[x] = (float)(1.0 - up); }
        else { upt[x] = (float)up; dnt[x] = (float)(1.0 - up); }
    }
    const int npx = g.hf * g.ht;
    for (long long tile = blockIdx.x; tile < g.ntiles; tile += gridDim.x) {
        const int a = (int)(tile / g.tt), b = (int)(tile % g.tt);
        __syncthreads();
        if (threadIdx.x < 4) {
            const int s = threadIdx.x;
            const int cf = a - 1 + (s >> 1), ct = b - 1 + (s & 1);
            const int ok = cf >= 0 && cf < g.ncf && ct >= 0 && ct < g.nct;
            valid_s[s] = ok;
            float2 r = make_float2(1.0f, 0.0f);
            float A = 1.0f;
            if (ok && MODE != MOS_OVERLAP) {
                const long long k = (long long)cf * g.nct + ct;
                const double p = phi[k];
                r = make_float2((float)cos(p), (float)sin(p));   // e^{i phi} in float64
                if (amp) A = (float)amp[k];
            }
            rot_s[s] = r;
            amp_s[s] = A;
        }
        __syncthreads();
        double acc[NQ];
#pragma unroll
        for (int q = 0; q < NQ; ++q) acc[q] = 0.0;
        for (int px = threadIdx.x; px < npx; px += blockDim.x) {
            const int i = px / g.ht, j = px - (px / g.ht) * g.ht;
            float2 y[4];
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                y[s] = make_float2(0.0f, 0.0f);
                if (!valid_s[s]) continue;
                const int si = s >> 1, sj = s & 1;
                const int cf = a - 1 + si, ct = b - 1 + sj;
                const long long k = (long long)cf * g.nct + ct;
                const int r = (1 - si) * g.hf + i, c = (1 - sj) * g.ht + j;
                const float2 v = chunks[(k * g.cwf + r) * g.cwt + c];
                const float m = mos_fac(si, cf, g.ncf, upf, dnf, i) * mos_fac(sj, ct, g.nct, upt, dnt, j);
                const float2 e = rot_s[s];
                // m * chunk * e^{i phi}
                const float zr = v.x * e.x - v.y * e.y, zi = v.x * e.y + v.y * e.x;
                y[s] = make_float2(m * zr, m * zi);
            }
            const long long o = ((long long)a * g.hf + i) * g.nT + (long long)b * g.ht + j;
            if (MODE == MOS_BUILD) {
                float wr = 0.0f, wi = 0.0f;
#pragma unroll
                for (int s = 0; s < 4; ++s) { wr += amp_s[s] * y[s].x; wi += amp_s[s] * y[s].y; }
                W[o] = make_float2(wr, wi);
            } else if (MODE == MOS_OVERLAP) {
                // C[v][u] += y_u conj(y_v): earlier chunk u against later chunk v
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int v = u + 1; v < 4; ++v) {
                        const int pi = mos_pair_index(u, v);
                        acc[2 * pi] += (double)(y[u].x * y[v].x + y[u].y * y[v].y);
                        acc[2 * pi + 1] += (double)(y[u].y * y[v].x - y[u].x * y[v].y);
                    }
            } else {
                const float2 w = W[o];
                if (MODE == MOS_ROT) {
                    acc[0] += (double)(w.x * w.x + w.y * w.y);
#pragma unroll
                    for (int s = 0; s < 4; ++s) acc[1 + s] += (double)(w.x * y[s].y - w.y * y[s].x);
                } else {
                    const float d = dspec[o], nn = noise[o];
                    const float wt = (w.x * w.x + w.y * w.y) - d;
                    const float n2 = nn * nn;
                    // t_s = y_s conj(W)
                    float tr[4], ti[4];
#pragma unroll
                    for (int s = 0; s < 4; ++s) {
                        tr[s] = y[s].x * w.x + y[s].y * w.y;
                        ti[s] = y[s].y * w.x - y[s].x * w.y;
                    }
                    if (MODE == MOS_FIT) {
                        const float chi = wt * wt / n2;
                        if (!isnan(chi)) acc[0] += (double)chi;
                        const float f4 = 4.0f * wt;
#pragma unroll
                        for (int s = 0; s < 4; ++s) {
                            const float gr = f4 * tr[s] / n2, gi = f4 * ti[s] / n2;
                            if (!isnan(gr) && !isnan(gi)) {   // nansum of a complex term
                                acc[1 + s] += (double)gr;
                                acc[5 + s] += (double)gi;
                            }
                        }
                    } else {   // MOS_HESS
                        const float f4 = 4.0f * wt;
#pragma unroll
                        for (int u = 0; u < 4; ++u)
#pragma unroll
                            for (int v = u + 1; v < 4; ++v) {
                                const int pi = mos_pair_index(u, v);
                                // gy = y_u conj(y_v)
                                const float gyr = y[u].x * y[v].x + y[u].y * y[v].y;
                                const float gyi = y[u].y * y[v].x - y[u].x * y[v].y;
                                acc[4 * pi + 0] += (double)((8.0f * tr[u] * tr[v] + f4 * gyr) / n2);
                                acc[4 * pi + 1] += (double)((-8.0f * ti[v] * tr[u] + f4 * gyi) / n2);
                                acc[4 * pi + 2] += (double)((-8.0f * ti[u] * tr[v] - f4 * gyi) / n2);
                                acc[4 * pi + 3] += (double)((8.0f * ti[u] * ti[v] + f4 * gyr) / n2);
                            }
#pragma unroll
                        for (int s = 0; s < 4; ++s) {
                            const float yy = y[s].x * y[s].x + y[s].y * y[s].y;
                            acc[24 + 5 * s + 0] += (double)((8.0f * tr[s] * tr[s] + f4 * yy) / n2);
                            acc[24 + 5 * s + 1] += (double)((-8.0f * ti[s] * tr[s]) / n2);
                            acc[24 + 5 * s + 2] += (double)((-f4 * ti[s]) / n2);
                            acc[24 + 5 * s + 3] += (double)((8.0f * ti[s] * ti[s] + f4 * yy) / n2);
                            acc[24 + 5 * s + 4] += (double)((-f4 * tr[s]) / n2);
                        }
                    }
                }
            }
        }
        if (MODE != MOS_BUILD) mos_block_store<NQ>(acc, part + tile * NQ);
    }
}

// Sum of a per-slot quantity q0 + slot over the (up to four) tiles of chunk k.
template <int NQ>
__device__ __forceinline__ double mos_chunk_sum(const MosGeom& g, const double* part, int cf, int ct,
                                                int q0) {
    double v = 0.0;
    for (int i = 0; i < 2; ++i) {
        const int a = cf + i;
        if (a >= g.tf) continue;
        for (int j = 0; j < 2; ++j) {
            const int b = ct + j;
            if (b >= g.tt) continue;
            const int s = 2 * (1 - i) + (1 - j);
            v += part[((long long)a * g.tt + b) * NQ + q0 + s];
        }
    }
    return v;
}

// Sum over the tiles that chunks u (earlier) and v (later) share; for u == v the per-slot
// quantity at qdiag + stride * slot, else the per-pair one at qpair + stride * pair.
template <int NQ>
__device__ __forceinline__ double mos_pair_sum(const MosGeom& g, const double* part, int uf, int ut,
                                               int vf, int vt, int qpair, int qdiag, int stride) {
    double v = 0.0;
    const int a0 = max(uf, vf), a1 = min(min(uf, vf) + 1, g.tf - 1);
    const int b0 = max(ut, vt), b1 = min(min(ut, vt) + 1, g.tt - 1);
    for (int a = a0; a <= a1; ++a)
        for (int b = b0; b <= b1; ++b) {
            const int su = 2 * (uf - a + 1) + (ut - b + 1);
            const int sv = 2 * (vf - a + 1) + (vt - b + 1);
            const int q = su == sv ? qdiag + stride * su : qpair + stride * mos_pair_index(su, sv);
            v += part[((long long)a * g.tt + b) * NQ + q];
        }
    return v;
}

// ROT: der[k] = 2 sum Im(conj(W) y_k).  FIT: grad[k] = (sum 4 wt Re t_k / N^2,
// -A_k sum 4 wt Im t_k / N^2), NaN terms skipped.
template <int MODE>
__global__ void mosaic_chunk_kernel(MosGeom g, const double* __restrict__ part,
                                    const double* __restrict__ amp, double* __restrict__ out) {
    constexpr int NQ = MosNq<MODE>::value;
    const long long P = (long long)g.ncf * g.nct;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < P;
         k += (long long)gridDim.x * blockDim.x) {
        const int cf = (int)(k / g.nct), ct = (int)(k % g.nct);
        if (MODE == MOS_ROT) {
            out[k] = 2.0 * mos_chunk_sum<NQ>(g, part, cf, ct, 1);
        } else {
            const double A = amp ? amp[k] : 1.0;
            out[2 * k] = mos_chunk_sum<NQ>(g, part, cf, ct, 1);
            out[2 * k + 1] = -A * mos_chunk_sum<NQ>(g, part, cf, ct, 5);
        }
    }
}

// out[0] = sum over tiles of part[tile][0] (fixed order: thread-strided, then a tree)
template <int NQ>
__global__ void mosaic_total_kernel(long long ntiles, const double* __restrict__ part,
                                    double* __restrict__ out) {
    SB_SHARED double red[256];
    double v = 0.0;
    for (long long t = threadIdx.x; t < ntiles; t += blockDim.x) v += part[t * NQ];
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = red[0];
}

// earlier neighbour e of chunk (cf, ct): (cf-1, ct-1), (cf-1, ct), (cf-1, ct+1), (cf, ct-1)
__device__ __forceinline__ void mos_earlier(int e, int cf, int ct, int* jf, int* jt) {
    *jf = e < 3 ? cf - 1 : cf;
    *jt = e == 0 || e == 3 ? ct - 1 : (e == 1 ? ct : ct + 1);
}

// OVERLAP: C float64 complex [P][4]: C[k][e] = sum mask_j chunk_j conj(mask_k chunk_k) over the
// overlap with earlier neighbour j = e (zero where there is none).
__global__ void mosaic_overlap_kernel(MosGeom g, const double* __restrict__ part,
                                      double* __restrict__ C) {
    constexpr int NQ = MosNq<MOS_OVERLAP>::value;
    const long long n = (long long)g.ncf * g.nct * 4;
    for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < n;
         x += (long long)gridDim.x * blockDim.x) {
        const long long k = x >> 2;
        const int e = (int)(x & 3);
        const int cf = (int)(k / g.nct), ct = (int)(k % g.nct);
        int jf, jt;
        mos_earlier(e, cf, ct, &jf, &jt);
        double re = 0.0, im = 0.0;
        if (jf >= 0 && jt >= 0 && jt < g.nct) {
            re = mos_pair_sum<NQ>(g, part, jf, jt, cf, ct, 0, 0, 2);
            im = mos_pair_sum<NQ>(g, part, jf, jt, cf, ct, 1, 1, 2);
        }
        C[2 * x] = re;
        C[2 * x + 1] = im;
    }
}

// HESS: COO triplets, 8 per (chunk N, forward neighbour e): e = 0 N itself, 1 (cf, ct+1),
// 2 (cf+1, ct-1), 3 (cf+1, ct), 4 (cf+1, ct+1).  Parameter index of phi_k is k-1 (k > 0),
// of A_k is k + P - 1.  Unused slots have row = col = -1.
__global__ void mosaic_hess_kernel(MosGeom g, const double* __restrict__ part,
                                   const double* __restrict__ amp, long long* __restrict__ rows,
                                   long long* __restrict__ cols, double* __restrict__ vals) {
    constexpr int NQ = MosNq<MOS_HESS>::value;
    const long long P = (long long)g.ncf * g.nct;
    for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < P * 5;
         x += (long long)gridDim.x * blockDim.x) {
        const long long u = x / 5;
        const int e = (int)(x - u * 5);
        const int uf = (int)(u / g.nct), ut = (int)(u % g.nct);
        const int vf = e < 2 ? uf : uf + 1;
        const int vt = e == 0 || e == 3 ? ut : (e == 2 ? ut - 1 : ut + 1);
        long long* R = rows + x * 8;
        long long* Cc = cols + x * 8;
        double* V = vals + x * 8;
        int n = 0;
        auto put = [&](long long r, long long c, double v) { R[n] = r; Cc[n] = c; V[n] = v; ++n; };
        if (vf < g.ncf && vt >= 0 && vt < g.nct) {
            const long long v = (long long)vf * g.nct + vt;
            const double Au = amp[u], Av = amp[v];
            const long long aU = u + P - 1, aV = v + P - 1, pU = u - 1, pV = v - 1;
            if (e == 0) {
                double d[5];
                for (int q = 0; q < 5; ++q) d[q] = mos_pair_sum<NQ>(g, part, uf, ut, uf, ut, 0, 24 + q, 5);
                put(aU, aU, d[0]);
                if (u > 0) {
                    const double ap = Au * d[1] + d[2];
                    put(aU, pU, ap);
                    put(pU, aU, ap);
                    put(pU, pU, Au * Au * d[3] + Au * d[4]);
                }
            } else {
                double q[4];
                for (int i = 0; i < 4; ++i) q[i] = mos_pair_sum<NQ>(g, part, uf, ut, vf, vt, i, 0, 4);
                put(aU, aV, q[0]);
                put(aV, aU, q[0]);
                put(aU, pV, Av * q[1]);
                put(pV, aU, Av * q[1]);
                if (u > 0) {
                    put(aV, pU, Au * q[2]);
                    put(pU, aV, Au * q[2]);
                    put(pU, pV, Au * Av * q[3]);
                    put(pV, pU, Au * Av * q[3]);
                }
            }
        }
        for (; n < 8; ++n) { R[n] = -1; Cc[n] = -1; V[n] = 0.0; }
    }
}

// tile geometry of ncf x nct chunks of cwf x cwt (widths already checked)
inline void mos_geom_fill(int ncf, int nct, int cwf, int cwt, MosGeom* g) {
    g->ncf = ncf; g->nct = nct; g->cwf = cwf; g->cwt = cwt;
    g->hf = ncf > 1 ? cwf / 2 : cwf;
    g->ht = nct > 1 ? cwt / 2 : cwt;
    g->tf = ncf > 1 ? ncf + 1 : 1;
    g->tt = nct > 1 ? nct + 1 : 1;
    g->nF = (long long)g->tf * g->hf;
    g->nT = (long long)g->tt * g->ht;
    g->ntiles = (long long)g->tf * g->tt;
}

#ifndef SB_HOST_EMU

static int mosaic_geom(int ncf, int nct, int cwf, int cwt, MosGeom* g) {
    SB_ARG(ncf >= 1 && nct >= 1 && cwf >= 1 && cwt >= 1);
    SB_ARG(ncf == 1 || (cwf >= 2 && cwf % 2 == 0));
    SB_ARG(nct == 1 || (cwt >= 2 && cwt % 2 == 0));
    mos_geom_fill(ncf, nct, cwf, cwt, g);
    if (g->hf > MOS_MAX_TILE || g->ht > MOS_MAX_TILE || g->nF > INT32_MAX || g->nT > INT32_MAX ||
        (long long)ncf * nct > INT32_MAX / 8) {
        set_error("mosaic: %d x %d chunks of %d x %d outside the supported geometry (tile "
                  "extent <= %d, mosaic sides < 2^31, fewer than 2^28 chunks)",
                  ncf, nct, cwf, cwt, MOS_MAX_TILE);
        return SB_ERR_UNSUPPORTED;
    }
    return SB_OK;
}

static unsigned mos_grid(long long n, long long per_block) {
    long long b = (n + per_block - 1) / per_block;
    if (b > (1LL << 20)) b = 1LL << 20;
    return (unsigned)(b < 1 ? 1 : b);
}

template <int MODE>
static int mosaic_tiles(const MosGeom& g, const float2* chunks, const double* phi, const double* amp,
                        float2* W, const float* dspec, const float* noise, double** part,
                        cudaStream_t st) {
    constexpr int NQ = MosNq<MODE>::value;
    double* p = nullptr;
    if (MODE != MOS_BUILD) {
        p = (double*)workspace(WS_TABLE, (size_t)g.ntiles * NQ * sizeof(double));
        if (!p) return SB_ERR_NOMEM;
    }
    const size_t smem = (size_t)2 * (g.hf + g.ht) * sizeof(float);
    ProfScope prof(PROF_MOSAIC_TILE, st);
    mosaic_tile_kernel<MODE><<<mos_grid(g.ntiles, 1), MOS_THREADS, smem, st>>>(
        g, chunks, phi, amp, W, dspec, noise, p);
    SB_LAUNCH_CHECK();
    if (part) *part = p;
    return SB_OK;
}

int mosaic_build(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
                 const double* amp, float2* W, cudaStream_t st) {
    MosGeom g;
    int rc = mosaic_geom(ncf, nct, cwf, cwt, &g);
    if (rc) return rc;
    return mosaic_tiles<MOS_BUILD>(g, chunks, phi, amp, W, nullptr, nullptr, nullptr, st);
}

int mosaic_rot(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
               const float2* W, double* power, double* der, cudaStream_t st) {
    MosGeom g;
    int rc = mosaic_geom(ncf, nct, cwf, cwt, &g);
    if (rc) return rc;
    double* part = nullptr;
    rc = mosaic_tiles<MOS_ROT>(g, chunks, phi, nullptr, const_cast<float2*>(W), nullptr, nullptr,
                               &part, st);
    if (rc) return rc;
    ProfScope prof(PROF_MOSAIC_REDUCE, st);
    const long long P = (long long)ncf * nct;
    mosaic_chunk_kernel<MOS_ROT><<<mos_grid(P, 256), 256, 0, st>>>(g, part, nullptr, der);
    SB_LAUNCH_CHECK();
    mosaic_total_kernel<MosNq<MOS_ROT>::value><<<1, 256, 0, st>>>(g.ntiles, part, power);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int mosaic_overlap(const float2* chunks, int ncf, int nct, int cwf, int cwt, double* C,
                   cudaStream_t st) {
    MosGeom g;
    int rc = mosaic_geom(ncf, nct, cwf, cwt, &g);
    if (rc) return rc;
    double* part = nullptr;
    rc = mosaic_tiles<MOS_OVERLAP>(g, chunks, nullptr, nullptr, nullptr, nullptr, nullptr, &part, st);
    if (rc) return rc;
    ProfScope prof(PROF_MOSAIC_REDUCE, st);
    mosaic_overlap_kernel<<<mos_grid((long long)ncf * nct * 4, 256), 256, 0, st>>>(g, part, C);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int mosaic_fit(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
               const double* amp, const float2* W, const float* dspec, const float* noise,
               double* fit, double* grad, cudaStream_t st) {
    MosGeom g;
    int rc = mosaic_geom(ncf, nct, cwf, cwt, &g);
    if (rc) return rc;
    double* part = nullptr;
    rc = mosaic_tiles<MOS_FIT>(g, chunks, phi, amp, const_cast<float2*>(W), dspec, noise, &part, st);
    if (rc) return rc;
    ProfScope prof(PROF_MOSAIC_REDUCE, st);
    const long long P = (long long)ncf * nct;
    mosaic_chunk_kernel<MOS_FIT><<<mos_grid(P, 256), 256, 0, st>>>(g, part, amp, grad);
    SB_LAUNCH_CHECK();
    mosaic_total_kernel<MosNq<MOS_FIT>::value><<<1, 256, 0, st>>>(g.ntiles, part, fit);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int mosaic_hess(const float2* chunks, int ncf, int nct, int cwf, int cwt, const double* phi,
                const double* amp, const float2* W, const float* dspec, const float* noise,
                long long* rows, long long* cols, double* vals, cudaStream_t st) {
    MosGeom g;
    int rc = mosaic_geom(ncf, nct, cwf, cwt, &g);
    if (rc) return rc;
    double* part = nullptr;
    rc = mosaic_tiles<MOS_HESS>(g, chunks, phi, amp, const_cast<float2*>(W), dspec, noise, &part,
                                st);
    if (rc) return rc;
    ProfScope prof(PROF_MOSAIC_REDUCE, st);
    const long long P = (long long)ncf * nct;
    mosaic_hess_kernel<<<mos_grid(P * 5, 256), 256, 0, st>>>(g, part, amp, rows, cols, vals);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

#endif  // SB_HOST_EMU

}  // namespace sb
