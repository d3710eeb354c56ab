// Shared helpers for libscint_b200 (sm_90a only).
#pragma once
#ifndef SB_HOST_EMU            // tests/host_emu compiles the device code for the CPU
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/scint_b200.h"

namespace sb {

void set_error(const char* fmt, ...);
const char* last_error();

// Grow-only per-process device workspace (one CUDA context per process, one caller thread
// at a time; see include/scint_b200.h).  A request larger than a slot's size frees the slot
// and allocates it again, so a pointer taken earlier from that slot dangles: a driver must
// not hold a buffer in a slot that a driver it calls takes.
//
//   slot          takers
//   WS_SCALARS    the ScalarBlock below
//   WS_INDEX      index tables of eta_sweep, thin_sweep, chisq_sweep; rev_map's bin counts;
//                 vlbi_retrieval's and asymmetry_batch's per-call arrays; the chirp-z result
//                 of conj_spectrum_c2c; the per-tile sums of sspec_tiles and acf_tiles;
//                 zap's select state and digit histogram
//   WS_BATCH      the batch slab of eta_sweep, thin_sweep, chisq_sweep, vlbi_retrieval,
//                 asymmetry_batch; herm_eigvec's basis; the padded chunk of
//                 conj_spectrum_c2c; gerchberg_saxton; svd_topk; zap's candidate keys
//   WS_PLANE0..4  the FFT engine: chirp_fft2 takes all five (through ifft2_chirp,
//                 ifft2_planes, ifft2_conj_any and the chirp-z conj_spectrum); the radix
//                 2-D transforms of sspec, acf, acf_sspec, sspec_tiles, acf_tiles,
//                 conj_spectrum, ifft2_planes,
//                 conj_spectrum_c2c and gerchberg_saxton take PLANE0..2.  Drivers that
//                 call neither use them too: sim_screen, sim_intensity, slow_ft,
//                 inpaint_biharmonic, scint_fit, acf_model, scale_dyn_lambda, brightness
//                 (PLANE0..3), scattered_image (PLANE0..1); eta_sweep
//                 keeps its fp16 copy in PLANE3, eig_half_launch its Lanczos basis in PLANE4
//   WS_TABLE      the column table and compact copy of thth_gather_source; the partial
//                 sums of svd_topk, bandpass_cols and the mosaic tiles
//
// Nesting rule: a driver that calls the FFT engine keeps its own buffers in WS_SCALARS,
// WS_INDEX, WS_BATCH and WS_TABLE only (chisq_sweep, vlbi_retrieval, conj_spectrum_c2c,
// gerchberg_saxton, conj_spectrum).  Likewise acf_sspec holds PLANE2 across sspec, and
// eta_sweep holds PLANE3 across eig_half_launch.
enum WsSlot {
    WS_SCALARS = 0,
    WS_INDEX = 1,
    WS_BATCH = 2,
    WS_PLANE0 = 3,
    WS_PLANE1 = 4,
    WS_PLANE2 = 5,
    WS_PLANE3 = 6,
    WS_PLANE4 = 7,
    WS_TABLE = 8,
    WS_COUNT = 9
};
void* workspace(WsSlot slot, size_t bytes);
void workspace_release();

// The device scalars in WS_SCALARS.  Kernels take plain pointers to the fields.
struct ScalarBlock {
    union {
        double stats[8];      // stats_pass (dynspec.cu): sums [0..3], means [4..6], ACF power [7]
        double c2c_sum[2];    // conj_spectrum_c2c: sum of the chunk's re, im
    };
    float acf_factor;         // acf: the factor of the final row pass
    float pad0[15];
    unsigned sweep_scale;     // eta_sweep: scale of the fp16 copy (the bits of a float)
    unsigned pad1[15];
    double l1;                // conj_spectrum_bound: L1 norm accumulator
    double pad2[7];
    double acf_part[32];      // acf: partial power sums (acf_tiles: written, not read)
};
static_assert(offsetof(ScalarBlock, stats) == 0, "ScalarBlock layout");
static_assert(offsetof(ScalarBlock, c2c_sum) == 0, "ScalarBlock layout");
static_assert(offsetof(ScalarBlock, acf_factor) == 8 * sizeof(double), "ScalarBlock layout");
static_assert(offsetof(ScalarBlock, sweep_scale) == 16 * sizeof(double), "ScalarBlock layout");
static_assert(offsetof(ScalarBlock, l1) == 24 * sizeof(double), "ScalarBlock layout");
static_assert(offsetof(ScalarBlock, acf_part) == 32 * sizeof(double), "ScalarBlock layout");
static_assert(sizeof(ScalarBlock) == 64 * sizeof(double), "ScalarBlock fills its allocation");

inline ScalarBlock* scalar_block() {
    return (ScalarBlock*)workspace(WS_SCALARS, sizeof(ScalarBlock));
}
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
