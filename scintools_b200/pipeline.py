"""Whole arc-measurement pipeline for a batch of dynamic spectra
(BASELINE.json config 5: secondary spectrum + ACF + theta-theta curvature per
dynspec, dynspecs block-partitioned over ranks, one all-gather of the fitted
curvatures at the end).

This is the GPU counterpart of the reference's only parallel mode,
``pool.map(thth.single_search, pars)`` over independent chunks
(scintools/dynspec.py:1715-1719): one process per GPU instead of a fork pool.
"""
import numpy as np

from . import sharding
from . import ththmod as thth
from .dynspec import BasicDyn, Dynspec


def arc_pipeline(dyn, freqs, times, etas, edges, fw=0.1, npad=3, coher=True,
                 tau_mask=0.0, want_sspec=True, want_acf=True, dtype=np.float32):
    """calc_sspec + calc_acf + single_search for one dynamic spectrum.
    Returns a dict with eta_fit, eta_sig, eigs and (optionally) sspec / acf."""
    freqs = np.asarray(freqs, dtype=np.float64)
    times = np.asarray(times, dtype=np.float64)
    out = {}
    if want_sspec or want_acf:
        ds = Dynspec(dyn=BasicDyn(dyn, times=times, freqs=freqs,
                                  dt=times[1] - times[0], df=freqs[1] - freqs[0]),
                     verbose=False)
        if want_sspec:
            ds.calc_sspec(dtype=dtype)
            out.update(sspec=ds.sspec, fdop=ds.fdop, tdel=ds.tdel)
        if want_acf:
            ds.calc_acf(dtype=dtype)
            out["acf"] = ds.acf
    d0 = np.asarray(dyn, dtype=np.float64)
    d0 = np.nan_to_num(d0 - np.nanmean(d0))         # dynspec.py:1691-1693
    res = thth.single_search([d0, freqs, times, etas, edges, None, False, fw,
                              npad, coher, tau_mask, False])
    out.update(eta_fit=float(np.asarray(res[0])), eta_sig=float(np.asarray(res[1])),
               eigs=res[4])
    return out


def batch_arc_pipeline(dyns, freqs, times, etas, edges, group=None, device=None,
                       **kw):
    """Run arc_pipeline on this rank's block of ``dyns`` (a sequence of 2-D
    arrays) and all-gather (eta_fit, eta_sig) over the process group.
    Returns two float64 arrays of length len(dyns), identical on every rank."""
    n = len(dyns)
    rank, world = sharding.world_info(group)
    lo, hi = sharding.block_range(n, rank, world)
    fit = np.full(hi - lo, np.nan)
    sig = np.full(hi - lo, np.nan)
    want_sspec = kw.pop("want_sspec", True)
    want_acf = kw.pop("want_acf", True)
    for k, i in enumerate(range(lo, hi)):
        r = arc_pipeline(dyns[i], freqs, times, etas, edges, want_sspec=want_sspec,
                         want_acf=want_acf, **kw)
        fit[k], sig[k] = r["eta_fit"], r["eta_sig"]
    return (sharding.all_gather_blocks(fit, n, group, device),
            sharding.all_gather_blocks(sig, n, group, device))
