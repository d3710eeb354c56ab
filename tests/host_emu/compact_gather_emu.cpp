// CPU run of the curvature-sweep gather of csrc/thth.cu from both of its sources, under
// the SIMT emulator: thth_prep_kernel, the table of reached columns (thth_colmark_kernel,
// thth_colslots_kernel), cs_compact_kernel and thth_build_copy_kernel reading the compact copy,
// against thth_build_kernel reading the spectrum itself and against thth_herm_upper.
// Every buffer a kernel receives has exactly the size sb::eta_sweep / sb::thth_gather_source
// give it and ends at an inaccessible page, with another one in front of it: an access
// outside it stops the process.  TEST INFRASTRUCTURE (tests/test_compact_gather_cpu.py).
#define SB_HOST_EMU 1
#include "simt.h"

#include <float.h>
#include <limits.h>
#include <sys/mman.h>
#include <unistd.h>

namespace sb {
alignas(128) unsigned char smem_raw[256 * 1024];
}
#include "../../scintools_b200/csrc/thth.cu"
#include "gather_src_emu.h"

namespace {
// count elements of T whose last byte is followed by a PROT_NONE page; PROT_NONE page before
// the mapping's first data page too
template <typename T>
struct Guarded {
    unsigned char* map = nullptr;
    size_t map_bytes = 0;
    T* p = nullptr;
    size_t count = 0;
    explicit Guarded(size_t n, int fill = 0) : count(n) {
        const size_t page = (size_t)sysconf(_SC_PAGESIZE);
        const size_t bytes = n * sizeof(T);
        const size_t data_pages = (bytes + page - 1) / page + (bytes == 0);
        map_bytes = (data_pages + 2) * page;
        map = (unsigned char*)mmap(nullptr, map_bytes, PROT_READ | PROT_WRITE,
                                   MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (map == MAP_FAILED) abort();
        std::memset(map, fill, map_bytes);
        mprotect(map, page, PROT_NONE);
        mprotect(map + (data_pages + 1) * page, page, PROT_NONE);
        p = reinterpret_cast<T*>(map + (data_pages + 1) * page - bytes);
    }
    ~Guarded() { munmap(map, map_bytes); }
    Guarded(const Guarded&) = delete;
    Guarded& operator=(const Guarded&) = delete;
};
}  // namespace

// M_cmp / M_dir / M_ref: float2 [neta][ld][ld] (compact copy, spectrum, thth_herm_upper on
// the cropped grid; the first two start as NaN junk, M_ref as zeros); Mb_cmp / Mb_dir:
// unsigned [neta][ld][ld / 2 ... ] as the build kernel lays the fp16 copy out (pack != 0);
// slot_of_col / col_of_slot: int [ncols]; info: {nslots from the device, nslots counted by
// a plain host loop over the pairs, error word after the gathers, ncols}.
extern "C" int emu_compact_gather(const float* cs_in, long long ntau, long long nfd,
                                  long long cs_pitch, int cs_half, double tau0, double dtau,
                                  double tau_absmax, double fd0, double dfd, double fd_half,
                                  const double* th_in, int n_th, int coherent,
                                  const double* etas_in, int neta, int pack, float* M_cmp,
                                  float* M_dir, float* M_ref, unsigned* Mb_cmp, unsigned* Mb_dir,
                                  int* nred_out, int* status_out, int* slot_of_col,
                                  int* col_of_slot, int* info) {
    using namespace sb;
    const long long pitch = cs_half ? cs_pitch : (cs_pitch > 0 ? cs_pitch : nfd);
    Guarded<float2> cs((size_t)ntau * pitch);
    std::memcpy(cs.p, cs_in, cs.count * sizeof(float2));
    Guarded<double> th(n_th), etas(neta);
    std::memcpy(th.p, th_in, n_th * sizeof(double));
    std::memcpy(etas.p, etas_in, neta * sizeof(double));
    ThthGeom g;
    g.cs = cs.p;
    g.ntau = ntau; g.nfd = nfd;
    g.tau0 = tau0; g.dtau = dtau; g.half_dtau = dtau / 2; g.tau_absmax = tau_absmax;
    g.fd0 = fd0; g.dfd = dfd; g.half_dfd = dfd / 2; g.fd_half = fd_half;
    g.inv_dtau = 1.0 / dtau; g.inv_dfd = 1.0 / dfd;
    g.th = th.p; g.n = n_th; g.coherent = coherent; g.cs_half = cs_half; g.cs_valid_cols = 0;
    g.cs_bound = nullptr;
    g.cs_pitch = pitch;
    const int ld = (n_th + 31) / 32 * 32;
    if (ld > 512) return -1;
    Guarded<int> idx((size_t)neta * ld), nred(neta), status(neta);
    for (int e = 0; e < neta; ++e)
        emu::run_block(emu::Dim3{32, 1, 1}, emu::Dim3{(unsigned)e, 0, 0},
                       emu::Dim3{(unsigned)neta, 1, 1},
                       [&]() { thth_prep_kernel(g, etas.p, neta, ld, idx.p, nred.p); });
    for (int e = 0; e < neta; ++e)
        for (unsigned bx = 0; bx < 4; ++bx)
            emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, (unsigned)e, 0},
                           emu::Dim3{4, (unsigned)neta, 1},
                           [&]() { thth_indexerr_kernel(g, etas.p, status.p); });
    std::memcpy(nred_out, nred.p, neta * sizeof(int));
    std::memcpy(status_out, status.p, neta * sizeof(int));

    // table: first uncapped (the launcher's first call of a geometry), then capped by the
    // count it read back
    const int ncols = thth_ncols(g);
    Guarded<int> tab(emu_table_ints(ncols));
    const int nslots = emu_col_table(g, tab.p, ncols, INT_MAX);
    if (nslots <= 0 || nslots > ncols) return -2;
    if (emu_col_table(g, tab.p, ncols, nslots) != nslots) return -3;
    Guarded<float2> C((size_t)nslots * emu_tau_pitch(g), 0xff);
    const ThthCopy copy = emu_compact(g, tab.p, ncols, nslots, C.p);
    std::memcpy(slot_of_col, tab.p + ncols, ncols * sizeof(int));
    std::memcpy(col_of_slot, tab.p + 2 * (size_t)ncols, ncols * sizeof(int));
    {   // the same marks by a plain loop over the pairs
        std::vector<char> mark(ncols, 0);
        for (int i = 0; i < n_th; ++i)
            for (int j = i + 1; j < n_th; ++j) {
                if (i + j == n_th - 1) continue;
                bool mirrored;
                const int c = thth_pair_column(g, th.p[j], th.p[i], &mirrored);
                if (c >= ncols) return -4;
                if (c >= 0) mark[c] = 1;
            }
        int cnt = 0;
        for (int c = 0; c < ncols; ++c) cnt += mark[c];
        info[1] = cnt;
    }
    info[0] = nslots;
    info[3] = ncols;

    float m = 0.f;
    for (long long r = 0; r < ntau; ++r)
        for (long long c = 0; c < (cs_half ? nfd / 2 + 1 : nfd); ++c) {
            const float2 q = g.cs[r * g.cs_pitch + c];
            m = std::fmax(std::fmax(std::fabs(q.x), std::fabs(q.y)), m);
        }
    Guarded<unsigned> absmax(1);
    absmax.p[0] = __float_as_uint(m);
    double tmin = th.p[0], tmax = th.p[0];
    for (int k = 1; k < n_th; ++k) {
        tmin = th.p[k] < tmin ? th.p[k] : tmin;
        tmax = th.p[k] > tmax ? th.p[k] : tmax;
    }
    const float span = (float)((tmax - tmin) * 1.0001);
    const int T = ld / 32, npairs = T * (T + 1) / 2;
    const unsigned gx = (unsigned)((neta + SB_BUILD_EB - 1) / SB_BUILD_EB);
    const size_t mat = (size_t)neta * ld * ld;
    for (int pass = 0; pass < 2; ++pass) {
        Guarded<float2> M(mat, 0xff);                       // NaN junk, like a fresh slab
        Guarded<unsigned> Mb(pack ? mat : 0, 0xff);
        for (unsigned bx = 0; bx < gx; ++bx)
            for (unsigned by = 0; by < (unsigned)npairs; ++by)
                emu::run_block(emu::Dim3{32, 8, 1}, emu::Dim3{bx, by, 0},
                               emu::Dim3{gx, (unsigned)npairs, 1}, [&]() {
                                   unsigned* mb = pack ? Mb.p : nullptr;
                                   const unsigned* am = pack ? absmax.p : nullptr;
                                   if (pack && pass)
                                       thth_build_kernel<2, unsigned>(g, etas.p, 0, neta, ld, idx.p,
                                                                      nred.p, M.p, mb, am, span);
                                   else if (pack)
                                       thth_build_copy_kernel<2, unsigned>(g, etas.p, 0, neta, ld,
                                                                           idx.p, nred.p, M.p, mb, am,
                                                                           span, copy);
                                   else if (pass)
                                       thth_build_kernel<0, size_t>(g, etas.p, 0, neta, ld, idx.p,
                                                                    nred.p, M.p, nullptr, nullptr, 0.f);
                                   else
                                       thth_build_copy_kernel<0, size_t>(g, etas.p, 0, neta, ld, idx.p,
                                                                         nred.p, M.p, nullptr, nullptr,
                                                                         0.f, copy);
                               });
        std::memcpy(pass ? M_dir : M_cmp, M.p, mat * sizeof(float2));
        if (pack) std::memcpy(pass ? Mb_dir : Mb_cmp, Mb.p, mat * sizeof(unsigned));
    }
    info[2] = *copy.err;
    float2* R = reinterpret_cast<float2*>(M_ref);
    for (int e = 0; e < neta; ++e) {
        const int n = nred.p[e];
        const int* id = idx.p + (size_t)e * ld;
        for (int a = 0; a < n; ++a)
            for (int b = a + 1; b < n; ++b)
                R[((size_t)e * ld + a) * ld + b] = thth_herm_upper(g, etas.p[e], id[a], id[b]);
    }
    return 0;
}
