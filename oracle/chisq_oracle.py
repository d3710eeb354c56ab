"""Unit-free CPU restatement of ththmod.chisq_calc (ththmod.py:330-368).

TEST INFRASTRUCTURE (see oracle/__init__.py).  float64 numpy, built from the
gather, rev_map, scipy eigsh and numpy ifft2 of oracle/thth_oracle.py (its
``modeler``).  Units as there: tau [us], fd / edges [mHz], eta [s^3].
"""
import numpy as np

from oracle import thth_oracle as TO


def chisq_calc(dspec, CS, tau, fd, eta, edges, N, mask=None):
    """ththmod.py:330-368: sum over the mask (default: finite dspec) of the
    squared residual of the rank-1 model, divided by N (not N**2)."""
    dspec = np.asarray(dspec)
    if mask is None:
        mask = np.isfinite(dspec)
    model = TO.modeler(CS, tau, fd, eta, edges)[3][:dspec.shape[0], :dspec.shape[1]]
    return np.sum((model - dspec)[mask] ** 2) / N
