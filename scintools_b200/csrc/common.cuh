// Shared helpers for libscint_b200 (sm_90a only).
#pragma once
#ifndef SB_HOST_EMU            // tests/host_emu compiles the device code for the CPU
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/scint_b200.h"

namespace sb {

void set_error(const char* fmt, ...);
const char* last_error();

// grow-only per-process device workspace (one CUDA context per process,
// one caller thread at a time; see include/scint_b200.h)
void* workspace(int slot, size_t bytes);
void workspace_release();
int num_sms();

// optional per-kernel timing with CUDA events on the launching stream
// (sb_profile_enable / sb_profile_collect); ids below
enum ProfId { PROF_CS_ROWS = 0, PROF_CS_COLA, PROF_CS_COLB, PROF_THTH_PREP,
              PROF_THTH_BUILD, PROF_THTH_EIG, PROF_SSPEC, PROF_ACF, PROF_SIM_SCREEN,
              PROF_SIM_FREQ, PROF_MOSAIC_TILE, PROF_MOSAIC_REDUCE, PROF_SVD_GRAM,
              PROF_SVD_APPLY, PROF_SFT_DOPPLER, PROF_SFT_DELAY, PROF_COUNT };
void prof_begin(int id, cudaStream_t st);
void prof_end(int id, cudaStream_t st);
struct ProfScope {
    int id; cudaStream_t st;
    ProfScope(int i, cudaStream_t s) : id(i), st(s) { prof_begin(id, st); }
    ~ProfScope() { prof_end(id, st); }
};

#define SB_CUDA(call)                                                        \
    do {                                                                     \
        cudaError_t _e = (call);                                             \
        if (_e != cudaSuccess) {                                             \
            sb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call,       \
                          cudaGetErrorString(_e));                           \
            return SB_ERR_CUDA;                                              \
        }                                                                    \
    } while (0)

void count_launch();

#define SB_LAUNCH_CHECK()                                                    \
    do {                                                                     \
        sb::count_launch();                                                  \
        cudaError_t _e = cudaGetLastError();                                 \
        if (_e != cudaSuccess) {                                             \
            sb::set_error("%s:%d launch -> %s", __FILE__, __LINE__,          \
                          cudaGetErrorString(_e));                           \
            return SB_ERR_CUDA;                                              \
        }                                                                    \
    } while (0)

#define SB_ARG(cond)                                                         \
    do {                                                                     \
        if (!(cond)) {                                                       \
            sb::set_error("%s:%d bad argument: %s", __FILE__, __LINE__,      \
                          #cond);                                            \
            return SB_ERR_ARG;                                               \
        }                                                                    \
    } while (0)

}  // namespace sb
#endif  // SB_HOST_EMU

// statically sized shared arrays: one per block on the device, one function-local
// static shared by all fibers under tests/host_emu
#ifdef SB_HOST_EMU
#define SB_SHARED static
#else
#define SB_SHARED __shared__
#endif

namespace sb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Exact floor(a / b) for finite doubles -- the value numpy's floor_divide
// (npy_divmod: fmod, (a-mod)/b, snap) returns.  Inputs must be bit-identical
// to the host's; callers build them with __dmul_rn/__dadd_rn (no FMA
// contraction).  Reference use: ththmod.py:94-97.
__device__ __forceinline__ double floor_div_exact(double a, double b) {
    if (b > 0.0 && isfinite(a)) {
        double q = floor(__ddiv_rn(a, b));
        double r = __fma_rn(-q, b, a);  // sign-exact remainder
        if (r < 0.0) q -= 1.0;
        else if (r >= b) q += 1.0;
        return q;
    }
    // literal npy_divmod for the unusual sign / non-finite cases
    if (b == 0.0) return __ddiv_rn(a, b);
    double mod = fmod(a, b);
    double div = __ddiv_rn(__dsub_rn(a, mod), b);
    if (mod != 0.0) {
        if ((b < 0.0) != (mod < 0.0)) div -= 1.0;
    }
    if (div != 0.0) {
        double fl = floor(div);
        if (div - fl > 0.5) fl += 1.0;
        return fl;
    }
    return copysign(0.0, __ddiv_rn(a, b));
}

// Same exact floor through a reciprocal: floor(a * (1/b)) is off by at most
// one for |a/b| < 2^50 and the FMA remainder fixes it.
__device__ __forceinline__ double floor_div_fast(double a, double b, double inv_b) {
    double q = floor(a * inv_b);
    if (b > 0.0 && fabs(q) < 1.0e15) {
        double r = __fma_rn(-q, b, a);
        if (r < 0.0) q -= 1.0;
        else if (r >= b) q += 1.0;
        return q;
    }
    return floor_div_exact(a, b);
}

}  // namespace sb
