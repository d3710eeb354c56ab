// CPU run of the device code of the cleaning passes (csrc/clean.cu, sources unchanged) under
// the SIMT emulator: the zero-count kernel on a 2-D grid of blocks, and the zap kernels
// launched in the order of sb::zap with G blocks of `threads` threads for the grid-wide
// passes.  The blocks of a launch run one after another.  The candidate buffer's capacity is
// an argument, so the compaction can be made to happen at any digit or never.
// TEST INFRASTRUCTURE (tests/test_clean_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
    unsigned long long o = *p;
    *p = o + v;
    return o;
}
static inline long long __double_as_longlong(double x) { long long v; std::memcpy(&v, &x, 8); return v; }
namespace sb {
alignas(128) unsigned char smem_raw[128 * 1024];
}

#include "../../scintools_b200/csrc/clean.cu"

namespace {
using namespace sb;

void grid(unsigned G, int threads, const std::function<void()>& body) {
    for (unsigned x = 0; x < G; ++x)
        emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, 0, 0},
                       emu::Dim3{G, 1, 1}, body);
}
}  // namespace

extern "C" int emu_zero_counts(const double* dyn, int nf, int nt, int row0, int row1,
                               int* row_counts, int* col_counts) {
    if (row_counts) std::memset(row_counts, 0, sizeof(int) * (row1 - row0));
    if (col_counts) std::memset(col_counts, 0, sizeof(int) * nt);
    const unsigned gx = (nt + ZC_THREADS - 1) / ZC_THREADS, gy = (row1 - row0 + ZC_ROWS - 1) / ZC_ROWS;
    for (unsigned y = 0; y < gy; ++y)
        for (unsigned x = 0; x < gx; ++x)
            emu::run_block(emu::Dim3{ZC_THREADS, 1, 1}, emu::Dim3{x, y, 0},
                           emu::Dim3{gx, gy, 1},
                           [&]() { zero_counts_kernel(dyn, nt, row0, row1, row_counts, col_counts); });
    (void)nf;
    return 0;
}

// sb::zap with cap = the buffer capacity (<= 0: the driver's); info[2 pass + 0/1]: the
// buffer's fill and the digit after which it was filled (-1: never)
extern "C" int emu_zap(double* x, long long n, double sigma, double* stats, int threads,
                       int G, long long cap, long long* info) {
    if (cap <= 0) cap = zap_cap(n);
    std::vector<unsigned long long> hist(ZP_BINS0), buf(cap > 0 ? cap : 1);
    ZapState state;
    ZapArgs a{x, n, nullptr, buf.data(), buf.data(), &state, hist.data()};
    for (int pass = 0; pass < 2; ++pass) {
        a.med = pass ? stats : nullptr;
        grid(1, 64, [&]() { zap_init_kernel(a, cap); });
        info[2 * pass] = 0;
        info[2 * pass + 1] = -1;
        for (int L = 0; L < ZP_LEVELS; ++L) {
            grid(G, threads, [&]() { zap_hist_kernel(a, L); });
            grid(1, ZP_SCAN, [&]() { zap_scan_kernel(a, L); });
            if (L + 1 < ZP_LEVELS) {
                const bool now = state.compact_now && !state.empty;
                grid(G, threads, [&]() { zap_compact_kernel(a); });
                if (now) {
                    info[2 * pass] = state.nbuf;
                    info[2 * pass + 1] = L;
                }
            }
        }
        grid(1, 1, [&]() { zap_final_kernel(a, stats + pass); });
    }
    if (n > 0) grid(G, threads, [&]() { zap_apply_kernel(x, n, sigma, stats); });
    return 0;
}
