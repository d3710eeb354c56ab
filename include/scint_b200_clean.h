/* libscint_b200 -- the cleaning passes of Dynspec: trim_edges's zero counts and zap
 * (reference scintools/dynspec.py:259-328, :3856-3870).
 *
 * Declared apart from include/scint_b200.h so that header keeps the entry points of ABI
 * version 8 exactly; the conventions of scint_b200.h hold here too (status codes,
 * sb_last_error, device pointers, caller stream, calls ordered across streams).
 */
#ifndef SCINT_B200_CLEAN_H
#define SCINT_B200_CLEAN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The statistics of Dynspec.trim_edges (dynspec.py:259-328): over rows row0 .. row1 - 1 of
 * dyn float64 [nf][nt], row_counts int32 [row1 - row0] holds each row's number of entries
 * that are 0 or NaN, and col_counts int32 [nt] each column's number over those rows.  Either
 * output may be NULL; both are overwritten (row0 == row1: every column count is 0).  Exact.
 * 0 <= row0 <= row1 <= nf, else SB_ERR_ARG; more than 4194240 rows in one call:
 * SB_ERR_UNSUPPORTED. */
int sb_dyn_zero_counts_f64(const double* dyn, int32_t nf, int32_t nt, int32_t row0, int32_t row1,
                           int32_t* row_counts, int32_t* col_counts, void* stream);

/* Dynspec.zap (dynspec.py:3856-3870) in place on dyn float64 [n]:
 *   med = np.median(dyn[~isnan(dyn)]); d = |dyn - med|; mdev = np.median(d[~isnan(d)]);
 *   dyn[d / mdev > sigma] = NaN.
 * A median is the middle value, or the mean (a + b) / 2 of the two middle values, of the
 * values that are not NaN (+-inf included), NaN when there is none.  Both are selections
 * (radix select on the values' ordered bit patterns), so stats float64 [2] = {med, mdev}
 * and the mask are numpy's exactly.  Workspace: 256 KiB and a buffer of n/8 keys. */
int sb_zap_f64(double* dyn, int64_t n, double sigma, double* stats, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCINT_B200_CLEAN_H */
