// The kernels behind sb::thth_gather_source (csrc/thth.cu) under the SIMT emulator, launch
// geometry and buffer layout as there: the table of reached columns and the compact,
// delay-contiguous copy of those columns.  Include after thth.cu.  TEST INFRASTRUCTURE.
#pragma once

namespace sb {

// ints of the table buffer: [mark | slot_of_col | col_of_slot | nslots, err]
inline size_t emu_table_ints(int ncols) { return 3 * (size_t)ncols + 2; }

// thth_colmark_kernel + thth_colslots_kernel into tab (emu_table_ints(ncols) ints);
// returns the slot count the device wrote
inline int emu_col_table(const ThthGeom& g, int* tab, int ncols, int cap) {
    std::memset(tab, 0, emu_table_ints(ncols) * sizeof(int));
    const long long pairs = (long long)g.n * g.n;
    unsigned blocks = (unsigned)((pairs + 255) / 256);
    if (blocks > 8) blocks = 8;
    for (unsigned bx = 0; bx < blocks; ++bx)
        emu::run_block(emu::Dim3{256, 1, 1}, emu::Dim3{bx, 0, 0}, emu::Dim3{blocks, 1, 1},
                       [&]() { thth_colmark_kernel(g, tab); });
    int* tail = tab + 3 * (size_t)ncols;
    emu::run_block(emu::Dim3{SLOT_THREADS, 1, 1}, emu::Dim3{0, 0, 0}, emu::Dim3{1, 1, 1}, [&]() {
        thth_colslots_kernel(tab, ncols, cap, tab + ncols, tab + 2 * (size_t)ncols, tail, tail + 1);
    });
    return tail[0];
}

inline long long emu_tau_pitch(const ThthGeom& g) { return (g.ntau + 3) / 4 * 4; }

// cs_compact_kernel into C (nslots * emu_tau_pitch(g) elements); the copy the gather
// then reads
inline ThthCopy emu_compact(const ThthGeom& g, int* tab, int ncols, int nslots, float2* C) {
    const long long tau_pitch = emu_tau_pitch(g);
    const unsigned gx = (unsigned)((g.ntau + 31) / 32), gy = (unsigned)((nslots + 31) / 32);
    for (unsigned bx = 0; bx < gx; ++bx)
        for (unsigned by = 0; by < gy; ++by)
            emu::run_block(emu::Dim3{32, 8, 1}, emu::Dim3{bx, by, 0}, emu::Dim3{gx, gy, 1}, [&]() {
                cs_compact_kernel(g.cs, g.ntau, g.cs_pitch, tab + 2 * (size_t)ncols, nslots,
                                  tau_pitch, C);
            });
    return ThthCopy{C, tau_pitch, nslots, tab + ncols, tab + 3 * (size_t)ncols + 1};
}

}  // namespace sb
