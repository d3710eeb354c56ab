// CPU run of the device code of the theoretical intensity ACF (csrc/acf_model.cu, sources
// unchanged) under the SIMT emulator: the contraction table of am_plan, then the gauss,
// contract and finish kernels in the order of sb::acf_model.  The blocks of a launch run one
// after another in block order.
// TEST INFRASTRUCTURE (tests/test_acf_model_emu_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

struct int2 { int x, y; };
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }

#include "../../scintools_b200/csrc/acf_model.cu"

namespace {
using namespace sb;

void grid(unsigned G, int threads, const std::function<void()>& body) {
    for (unsigned x = 0; x < G; ++x)
        emu::run_block(emu::Dim3{(unsigned)threads, 1, 1}, emu::Dim3{x, 0, 0},
                       emu::Dim3{G, 1, 1}, body);
}
}  // namespace

// returns the number of contraction blocks
extern "C" int emu_acf_model(const double* snp, int n1, const double* snp2, int n2,
                             const double* dnun, int ndnun, const double* snx,
                             const double* sny, int nsn, int quadrant, double sigxn,
                             double sigyn, double sqrtar, double alph2, double step1,
                             double step2, double wn_amp, double amp, double* acf,
                             double* efield) {
    AmPlan plan;
    am_plan(n1, n2, ndnun, nsn, plan);
    std::vector<double> g2((size_t)n2 * n2);
    std::vector<double2> part(plan.blocks.size() * AM_TS);
    grid(3, 64, [&]() { am_gauss_kernel(snp, n1, snp2, n2, sqrtar, alph2, efield, g2.data()); });
    AmArgs a{snp, snp2, efield, g2.data(), dnun, snx, sny, n1, n2, nsn, sigxn, sigyn};
    grid((unsigned)plan.blocks.size(), AM_THREADS,
         [&]() { am_contract_kernel(a, plan.blocks.data(), part.data()); });
    AmFinish f{dnun, snx, sny, part.data(), plan.range.data(), ndnun, nsn, quadrant,
               sqrtar, alph2, step1, step2, wn_amp, amp};
    const long long nk = (long long)nsn * ndnun;
    grid((unsigned)((nk + 255) / 256), 256, [&]() { am_finish_kernel(f, acf); });
    return (int)plan.blocks.size();
}
