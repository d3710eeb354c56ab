// Hand-written radix-2/4/8/16 FFT building blocks for sm_90a.
//
// Everything here works on a shared-memory array viewed as [fft index][batch]:
// element (i, b) lives at s[i * fstride + b * bstride].  Lanes always run over
// the batch index, so every shared-memory access of a warp is a run of
// consecutive (or odd-stride padded) elements: no bank conflicts by
// construction.  Passes are in place:
//   DIF (decimation in frequency): natural input  -> digit-reversed output
//   DIT (decimation in time):      digit-reversed input -> natural output
// with the SAME position map digit_pos<L>() for both.
#pragma once
#include "common.cuh"

namespace sb {

template <typename T> struct CxT;
template <> struct CxT<float> { using type = float2; };
template <> struct CxT<double> { using type = double2; };
template <typename T> using cx = typename CxT<T>::type;

template <typename T> __host__ __device__ __forceinline__ cx<T> mkc(T x, T y) {
    cx<T> r; r.x = x; r.y = y; return r;
}
template <typename C> __device__ __forceinline__ C cadd(C a, C b) { a.x += b.x; a.y += b.y; return a; }
template <typename C> __device__ __forceinline__ C csub(C a, C b) { a.x -= b.x; a.y -= b.y; return a; }
template <typename C> __device__ __forceinline__ C cmul(C a, C b) {
    C r; r.x = a.x * b.x - a.y * b.y; r.y = a.x * b.y + a.y * b.x; return r;
}
template <typename C> __device__ __forceinline__ C cconj(C a) { a.y = -a.y; return a; }
// multiply by (DIR * i): DIR=-1 -> -i (forward), DIR=+1 -> +i (inverse)
template <int DIR, typename C> __device__ __forceinline__ C mul_i(C a) {
    C r;
    if (DIR < 0) { r.x = a.y; r.y = -a.x; } else { r.x = -a.y; r.y = a.x; }
    return r;
}
// multiply by exp(DIR * i * pi/4) = (1 + DIR i)/sqrt2
template <int DIR, typename C> __device__ __forceinline__ C mul_w8(C a) {
    const auto h = (decltype(a.x))0.70710678118654752440;
    C r;
    if (DIR < 0) { r.x = (a.x + a.y) * h; r.y = (a.y - a.x) * h; }
    else { r.x = (a.x - a.y) * h; r.y = (a.y + a.x) * h; }
    return r;
}
// multiply by exp(DIR * i * theta) given cos, sin of theta
template <int DIR, typename C, typename T>
__device__ __forceinline__ C mul_cs(C a, T c, T s) {
    C r;
    if (DIR < 0) { r.x = a.x * c + a.y * s; r.y = a.y * c - a.x * s; }
    else { r.x = a.x * c - a.y * s; r.y = a.y * c + a.x * s; }
    return r;
}

// ---- fp32 complex arithmetic with a fixed rounding sequence ----------------
// A complex multiply is b * a.x + (-b.y, b.x) * a.y: one rounded multiply and one
// fused multiply-add per component.  The _rn intrinsics keep the compiler from
// contracting or reordering these, so every fp32 transform rounds the same way
// whatever the optimisation level.  These overloads are picked over the generic
// templates above for every fp32 transform; the fp64 paths are unchanged.
#ifndef SB_HOST_EMU
__device__ __forceinline__ float2 cadd(float2 a, float2 b) {
    return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 csub(float2 a, float2 b) {
    return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
}
// a * (s, s)
__device__ __forceinline__ float2 f2_scale(float2 a, float s) {
    return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s));
}
// a * (s, s) + c
__device__ __forceinline__ float2 f2_fma(float2 a, float s, float2 c) {
    return make_float2(__fmaf_rn(a.x, s, c.x), __fmaf_rn(a.y, s, c.y));
}
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return f2_fma(make_float2(-b.y, b.x), a.y, f2_scale(b, a.x));
}
template <int DIR> __device__ __forceinline__ float2 mul_w8(float2 a) {
    const float2 r = DIR < 0 ? make_float2(a.y, -a.x) : make_float2(-a.y, a.x);
    return f2_scale(cadd(a, r), 0.70710678118654752440f);
}
template <int DIR> __device__ __forceinline__ float2 mul_cs(float2 a, float c, float s) {
    const float2 r = DIR < 0 ? make_float2(a.y, -a.x) : make_float2(-a.y, a.x);
    return f2_fma(r, s, f2_scale(a, c));
}
#endif  // SB_HOST_EMU

// ---- in-register DFTs, natural order in and out --------------------------
template <int DIR, typename C> __device__ __forceinline__ void dft2(C& a, C& b) {
    C t = a; a = cadd(t, b); b = csub(t, b);
}
template <int DIR, typename C>
__device__ __forceinline__ void dft4(C& a0, C& a1, C& a2, C& a3) {
    C t0 = cadd(a0, a2), t1 = csub(a0, a2);
    C t2 = cadd(a1, a3), t3 = mul_i<DIR>(csub(a1, a3));
    a0 = cadd(t0, t2); a2 = csub(t0, t2);
    a1 = cadd(t1, t3); a3 = csub(t1, t3);
}
template <int R, int DIR, typename C> struct Dft;
template <int DIR, typename C> struct Dft<2, DIR, C> {
    static __device__ __forceinline__ void run(C (&a)[2]) { dft2<DIR>(a[0], a[1]); }
};
template <int DIR, typename C> struct Dft<4, DIR, C> {
    static __device__ __forceinline__ void run(C (&a)[4]) { dft4<DIR>(a[0], a[1], a[2], a[3]); }
};
template <int DIR, typename C> struct Dft<8, DIR, C> {
    static __device__ __forceinline__ void run(C (&a)[8]) {
        // 8 = 2 x 4 (DIF split): u -> even outputs, v -> odd outputs
        C u0 = cadd(a[0], a[4]), v0 = csub(a[0], a[4]);
        C u1 = cadd(a[1], a[5]), v1 = mul_w8<DIR>(csub(a[1], a[5]));
        C u2 = cadd(a[2], a[6]), v2 = mul_i<DIR>(csub(a[2], a[6]));
        C u3 = cadd(a[3], a[7]), v3 = mul_i<DIR>(mul_w8<DIR>(csub(a[3], a[7])));
        dft4<DIR>(u0, u1, u2, u3);
        dft4<DIR>(v0, v1, v2, v3);
        a[0] = u0; a[2] = u1; a[4] = u2; a[6] = u3;
        a[1] = v0; a[3] = v1; a[5] = v2; a[7] = v3;
    }
};
template <int DIR, typename C> struct Dft<16, DIR, C> {
    static __device__ __forceinline__ void run(C (&a)[16]) {
        using T = decltype(a[0].x);
        const T c1 = (T)0.92387953251128675613, s1 = (T)0.38268343236508977173;
        // 16 = 4 x 4: columns j (stride 4), then twiddle w16^(j r'), then rows
#pragma unroll
        for (int j = 0; j < 4; ++j) dft4<DIR>(a[j], a[j + 4], a[j + 8], a[j + 12]);
        // b[j][r'] sits in a[j + 4 r']; multiply by w16^(j r')
        a[5] = mul_cs<DIR>(a[5], c1, s1);          // j=1 r'=1 : w^1
        a[9] = mul_w8<DIR>(a[9]);                  // j=1 r'=2 : w^2
        a[13] = mul_cs<DIR>(a[13], s1, c1);        // j=1 r'=3 : w^3
        a[6] = mul_w8<DIR>(a[6]);                  // j=2 r'=1 : w^2
        a[10] = mul_i<DIR>(a[10]);                 // j=2 r'=2 : w^4
        a[14] = mul_i<DIR>(mul_w8<DIR>(a[14]));    // j=2 r'=3 : w^6
        a[7] = mul_cs<DIR>(a[7], s1, c1);          // j=3 r'=1 : w^3
        a[11] = mul_i<DIR>(mul_w8<DIR>(a[11]));    // j=3 r'=2 : w^6
        a[15] = mul_i<DIR>(mul_i<DIR>(mul_cs<DIR>(a[15], c1, s1)));  // w^9 = w^8 w^1
        // rows: X[4 k' + r'] = dft4 over j of a[j + 4 r']
        C o[16];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            C x0 = a[4 * r], x1 = a[4 * r + 1], x2 = a[4 * r + 2], x3 = a[4 * r + 3];
            dft4<DIR>(x0, x1, x2, x3);
            o[r] = x0; o[4 + r] = x1; o[8 + r] = x2; o[12 + r] = x3;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) a[k] = o[k];
    }
};

// radix schedule: outermost radix for a sub-transform of length n
__host__ __device__ constexpr int pick_radix(int n) {
    return (n >= 16 && n != 32 && n != 64) ? 16 : (n >= 8 ? 8 : n);
}

// position of logical index idx inside an in-place transform of length L
template <int L> __host__ __device__ __forceinline__ int digit_pos(int idx) {
    int pos = 0, n = L;
#pragma unroll
    for (int guard = 0; guard < 8; ++guard) {
        if (n <= 1) break;
        const int R = pick_radix(n);
        const int d = idx % R;
        idx /= R;
        n /= R;
        pos += d * n;
    }
    return pos;
}

// one in-place radix-R pass over sub-blocks of length n (n | L).
// tw[i] = exp(DIR * 2 pi i * i / L), i < L (shared memory).
template <typename T, int R, int DIR, bool DIT>
__device__ __forceinline__ void fft_pass(cx<T>* s, int n, int L, int fstride,
                                         int log2batch, int bstride,
                                         const cx<T>* tw, int tid, int nthreads) {
    using C = cx<T>;
    const int m = n / R;
    const int items = (L / R) << log2batch;
    const int twstep = L / n;
    const int bmask = (1 << log2batch) - 1;
    for (int it = tid; it < items; it += nthreads) {
        const int b = it & bmask;
        const int bf = it >> log2batch;
        const int j = bf % m;
        const int o = (bf / m) * n;
        C* p = s + (size_t)(o + j) * fstride + (size_t)b * bstride;
        const int es = m * fstride;
        C a[R];
#pragma unroll
        for (int r = 0; r < R; ++r) a[r] = p[r * es];
        if (DIT && m > 1) {
#pragma unroll
            for (int r = 1; r < R; ++r) a[r] = cmul(a[r], tw[j * r * twstep]);
        }
        Dft<R, DIR, C>::run(a);
        if (!DIT && m > 1) {
#pragma unroll
            for (int r = 1; r < R; ++r) a[r] = cmul(a[r], tw[j * r * twstep]);
        }
#pragma unroll
        for (int r = 0; r < R; ++r) p[r * es] = a[r];
    }
}

template <typename T, int L, int N, int DIR> struct DifPasses {
    static __device__ __forceinline__ void run(cx<T>* s, int fs, int lb, int bs,
                                               const cx<T>* tw, int tid, int nt) {
        constexpr int R = pick_radix(N);
        fft_pass<T, R, DIR, false>(s, N, L, fs, lb, bs, tw, tid, nt);
        __syncthreads();
        DifPasses<T, L, N / R, DIR>::run(s, fs, lb, bs, tw, tid, nt);
    }
};
template <typename T, int L, int DIR> struct DifPasses<T, L, 1, DIR> {
    static __device__ __forceinline__ void run(cx<T>*, int, int, int, const cx<T>*, int, int) {}
};
template <typename T, int L, int N, int DIR> struct DitPasses {
    static __device__ __forceinline__ void run(cx<T>* s, int fs, int lb, int bs,
                                               const cx<T>* tw, int tid, int nt) {
        constexpr int R = pick_radix(N);
        DitPasses<T, L, N / R, DIR>::run(s, fs, lb, bs, tw, tid, nt);
        fft_pass<T, R, DIR, true>(s, N, L, fs, lb, bs, tw, tid, nt);
        __syncthreads();
    }
};
template <typename T, int L, int DIR> struct DitPasses<T, L, 1, DIR> {
    static __device__ __forceinline__ void run(cx<T>*, int, int, int, const cx<T>*, int, int) {}
};

// In-place length-L transform along the strided axis for 2^log2batch
// independent batch entries.  Caller syncs before; a sync follows each pass.
template <typename T, int L, int DIR, bool DIT>
__device__ __forceinline__ void fft_axis(cx<T>* s, int fstride, int log2batch,
                                         int bstride, const cx<T>* tw, int tid,
                                         int nthreads) {
    if (DIT) DitPasses<T, L, L, DIR>::run(s, fstride, log2batch, bstride, tw, tid, nthreads);
    else DifPasses<T, L, L, DIR>::run(s, fstride, log2batch, bstride, tw, tid, nthreads);
}

}  // namespace sb
