"""Classical arc fit: Dynspec.norm_sspec / Dynspec.fit_arc on the GPU path
(reference scintools/dynspec.py:1920-2183 and :970-1346, SURVEY.md 8f rank 2).

The device does the heavy part -- every delay row of the secondary spectrum
resampled with numpy.interp semantics on the normalised Doppler axis, the masked
power per row and the delay-scrunched, weighted profile
(``sb_norm_sspec_f32`` / ``sb_norm_sspec_avg_f32``, csrc/normsspec.cu).  What is
left here is the reference's scalar bookkeeping: axis construction, weights,
Savitzky-Golay smoothing, the window walk around the peak and the (log-)parabola
fit.  That glue follows the reference's control flow and expressions line by
line on purpose -- the drop-in contract is "same attributes, same numbers"
(``eta / etaerr / etaerr2``, ``betaeta...``, ``norm_sspec_avg``, ``eta_array``,
``noise``, ``prob_eta_peak``, ``normsspec*``, ``powerspectrum``) -- with the
plotting branches removed and astropy / lmfit out of the picture.

Mixed into ``scintools_b200.dynspec.Dynspec`` (class ArcFitMixin).
"""
from copy import deepcopy as cp

import numpy as np
from scipy.signal import savgol_filter

from . import _device as D
from . import _lib


def is_valid(array):
    """scint_utils.is_valid (scint_utils.py:87-91)."""
    return np.isfinite(array) * (~np.isnan(array))


def fit_parabola(x, y):
    """scint_models.fit_parabola (scint_models.py:300-326): peak and its error
    from a quadratic polyfit on a rescaled abscissa."""
    ptp = np.ptp(x)
    x = x * (1000 / ptp)
    params, pcov = np.polyfit(x, y, 2, cov=True)
    yfit = params[0] * np.power(x, 2) + params[1] * x + params[2]
    errors = [np.absolute(pcov[i][i]) ** 0.5 for i in range(len(params))]
    peak = -params[1] / (2 * params[0])
    peak_error = np.sqrt((errors[1] ** 2) * ((1 / (2 * params[0])) ** 2) +
                         (errors[0] ** 2) * ((params[1] / 2) ** 2))
    return yfit, peak * (ptp / 1000), peak_error * (ptp / 1000)


def fit_log_parabola(x, y):
    """scint_models.fit_log_parabola (scint_models.py:329-347)."""
    logx = np.log(x)
    ptp = np.ptp(logx)
    x = logx * (1000 / ptp)
    yfit, peak, peak_error = fit_parabola(x, y)
    frac_error = peak_error / peak
    peak = np.e ** (peak * ptp / 1000)
    return yfit, peak, frac_error * peak


def norm_rows_device(sspec, fdop, tdel, eta, maxnormfac, fdopnew, weights_fn, want_2d=True):
    """Resample + scrunch on the GPU.  ``weights_fn(power) -> weights [nr]`` runs on
    the host between the two kernels (the reference derives the weights from the
    per-row power spectrum); it may return ``(weights, rows)`` instead, a boolean
    selection of the rows that enter the average (the others are left out, not given
    a zero weight, which would turn a +-inf sample into NaN).  Returns (norm [nr][nq]
    float64 with NaN where masked or None, power [nr], avg [nq] with NaN where the
    weights sum to zero)."""
    import torch
    sspec = np.ascontiguousarray(sspec)
    nr, nc = sspec.shape
    nq = int(np.shape(fdopnew)[0])
    # np.interp raises on a row with no selected sample (a NaN sqrt(tdel / eta), e.g. the
    # delay-zero row at eta = 0); the kernel would return it fully masked instead
    imax = maxnormfac * np.sqrt(np.asarray(tdel, dtype=np.float64) / eta)
    if not np.all(np.min(np.abs(fdop)) <= imax):
        raise ValueError("array of sample points is empty")
    d_s = D.upload_f32(sspec)
    d_fd = D.upload(np.ascontiguousarray(fdop, dtype=np.float64))
    d_td = D.upload(np.ascontiguousarray(tdel, dtype=np.float64))
    d_fn = D.upload(np.ascontiguousarray(fdopnew, dtype=np.float64))
    d_out = D.empty((nr, nq), torch.float32)
    d_pow = D.empty((nr,), torch.float64)
    _lib.check(_lib.lib.sb_norm_sspec_f32(d_s.data_ptr(), nr, nc, d_fd.data_ptr(),
                                          d_td.data_ptr(), float(eta), float(maxnormfac),
                                          d_fn.data_ptr(), nq, d_out.data_ptr(),
                                          d_pow.data_ptr(), D.stream_ptr()))
    power = d_pow.cpu().numpy()
    weights, rows = weights_fn(power), None
    if isinstance(weights, tuple):
        weights, rows = weights
    weights = np.ascontiguousarray(weights, dtype=np.float64)
    if weights.shape != (nr,):
        raise ValueError("norm_sspec: weights must have one entry per delay row")
    d_in = d_out
    if rows is not None:
        rows = np.asarray(rows, dtype=bool)
        if not rows.all():          # the rows the average reads, gathered in order
            d_in = d_out.index_select(0, torch.as_tensor(np.flatnonzero(rows),
                                                         device=d_out.device))
            weights = np.ascontiguousarray(weights[rows])
    if d_in.shape[0] == 0:          # no row: every weight sum is zero
        avg = np.full(nq, np.nan)
    else:
        d_w = D.upload(weights)
        d_avg = D.empty((nq,), torch.float64)
        _lib.check(_lib.lib.sb_norm_sspec_avg_f32(d_in.data_ptr(), d_in.shape[0], nq,
                                                  d_w.data_ptr(), d_avg.data_ptr(),
                                                  D.stream_ptr()))
        avg = d_avg.cpu().numpy()
    norm = d_out.cpu().numpy().astype(np.float64) if want_2d else None
    return norm, power, avg


# tests replace this with a numpy stand-in to exercise the host glue without a GPU
_norm_rows = norm_rows_device


class ArcFitMixin:
    """Dynspec.norm_sspec and Dynspec.fit_arc (see the module docstring)."""

    # ------------------------------------------------------------------
    def norm_sspec(self, eta=None, delmax=None, plot=False, startbin=1,
                   maxnormfac=5, minnormfac=0, cutmid=0, lamsteps=True,
                   scrunched=True, plot_fit=True, ref_freq=1400,
                   velocity=False, numsteps=None, filename=None, display=True,
                   weighted=True, unscrunched=True, logsteps=False,
                   powerspec=True, interp_nan=False, fit_spectrum=False,
                   powerspec_cut=False, figsize=(9, 9),
                   subtract_artefacts=False, dpi=200):
        """Normalise the Doppler axis with the arc curvature and scrunch over
        delay (reference dynspec.py:1920-2183) -> self.normsspec (masked 2-D),
        normsspecavg, normsspec_tdel, normsspec_fdop, powerspectrum, mask, weights."""
        if plot:
            raise NotImplementedError("plotting is outside the GPU hot path")
        if velocity or logsteps or interp_nan or fit_spectrum or minnormfac > 0:
            raise NotImplementedError(
                "norm_sspec on the GPU path: velocity, logsteps, interp_nan, "
                "fit_spectrum (lmfit) and minnormfac > 0 are not part of this version")
        delmax = np.max(self.tdel) if delmax is None else delmax
        if lamsteps:
            if not hasattr(self, 'lamsspec'):
                self.calc_sspec(lamsteps=lamsteps)
            yaxis = cp(self.beta)
            sspec = cp(self.lamsspec)
            if not hasattr(self, 'betaeta') and eta is None:
                self.fit_arc(lamsteps=lamsteps, delmax=delmax, plot=plot, startbin=startbin)
        else:
            if not hasattr(self, 'sspec'):
                self.calc_sspec()
            sspec = cp(self.sspec)
            yaxis = cp(self.tdel)
            if not hasattr(self, 'eta') and eta is None:
                self.fit_arc(lamsteps=lamsteps, delmax=delmax, plot=plot, startbin=startbin)
        if eta is None:
            eta = self.betaeta if lamsteps else self.eta
        elif not lamsteps:      # convert to beta (dynspec.py:2026-2030)
            c = 299792458.0
            beta_to_eta = c * 1e6 / ((ref_freq * 10 ** 6) ** 2)
            eta = eta / (self.freq / ref_freq) ** 2
            eta = eta * beta_to_eta

        ind = np.argmin(abs(self.tdel - delmax))
        sspec = np.array(sspec[startbin:ind, :], dtype=np.float64)
        nr, nc = np.shape(sspec)
        sspec[:, int(nc / 2 - np.floor(cutmid / 2)):int(nc / 2 + np.floor(cutmid / 2))] = np.nan
        tdel = yaxis[startbin:ind]
        if subtract_artefacts:
            delay_response = np.nanmean(sspec[:, np.argwhere(
                np.abs(self.fdop) > 0.9 * np.max(self.fdop))], axis=1)
            delay_response -= np.median(delay_response)
            sspec = np.subtract(sspec, delay_response)
        fdop = self.fdop
        maxfdop = maxnormfac * np.sqrt(tdel[-1] / eta)
        if maxfdop > max(fdop):
            maxfdop = max(fdop)
        nfdop = 2 * len(fdop[abs(fdop) <= maxfdop]) if numsteps is None else numsteps
        if nfdop % 2 != 0:
            nfdop += 1
        fdopnew = np.linspace(-maxnormfac, maxnormfac, int(nfdop))

        state = {}

        def weights_fn(power):
            # dynspec.py:2120-2157 with fit_spectrum=False, the reference's expressions
            ps = np.ma.masked_invalid(power)
            state["powerspectrum"] = ps
            xdata = np.sqrt(tdel)
            ydata = np.sqrt(tdel) * ps
            xdata = xdata[~np.isnan(xdata)]
            ydata = ydata[~np.isnan(ydata)]
            alpha = -11 / 3
            index = np.argmin(np.abs(xdata - 10))
            amp = ydata[index] * xdata[index] ** -alpha
            wn = np.min(ydata)
            arc_spectrum = amp * xdata ** alpha
            w = 10 * np.log10(arc_spectrum) if weighted else np.ones(np.shape(arc_spectrum))
            state["weights"] = w
            wdev = np.array(np.ma.filled(w, 0.0), dtype=np.float64)
            if powerspec_cut:       # np.ma.average over the rows with arc_spectrum > wn only
                keep = np.ma.filled(arc_spectrum > wn, False)
                if np.count_nonzero(keep) == 1:
                    # the reference squeezes the weights of a single row to a scalar, and
                    # np.ma.average rejects them (dynspec.py:2172-2175)
                    raise ValueError("Shape of weights must be consistent with shape of a "
                                     "along specified axis.")
                # np.ma.average(normSspec[indices, :]): the other rows are not read
                return wdev, keep
            return wdev

        norm, power, avg = _norm_rows(sspec, fdop, tdel, eta, maxnormfac, fdopnew, weights_fn)
        mask = np.isnan(norm)
        self.mask = mask
        self.powerspectrum = state["powerspectrum"]
        self.weights = state["weights"]
        # np.ma.average divides with numpy.ma's safe division, which masks a quotient whose
        # numerator is not small against its denominator: a zero weight sum (the device's
        # NaN; 0.0 is left under the mask) and the +-inf sum of a column holding a +-inf
        # sample (the infinity is left under the mask).  fit_arc's np.array(masked) then
        # sees that data, so keep it identical
        gone = np.isnan(avg)
        self.normsspecavg = np.ma.array(np.where(gone, 0.0, avg), mask=gone | np.isinf(avg))
        self.normsspec = np.ma.array(norm, mask=mask)
        self.normsspec_tdel = tdel
        self.normsspec_fdop = fdopnew
        return

    # ------------------------------------------------------------------
    def fit_arc(self, asymm=False, plot=False, delmax=None, numsteps=1e4,
                startbin=3, cutmid=3, lamsteps=False, etamax=None, etamin=None,
                low_power_diff=-1, high_power_diff=-0.5, ref_freq=1400,
                constraint=[0, np.inf], nsmooth=5, efac=1, filename=None,
                noise_error=True, display=True, figN=None, log_parabola=False,
                logsteps=False, plot_spec=False, fit_spectrum=False,
                subtract_artefacts=False, figsize=(9, 9), dpi=200,
                velocity=False, weighted=False):
        """Arc curvature with maximum power along it (reference dynspec.py:970-1346):
        sets eta / etaerr / etaerr2 (or betaeta... with lamsteps, ..._left / _right with
        asymm), eta_array, norm_sspec_avg, prob_eta_peak, noise, norm_delmax."""
        if plot or plot_spec:
            raise NotImplementedError("plotting is outside the GPU hot path")
        if velocity:
            raise NotImplementedError("velocity rescaling is outside the GPU hot path")
        if not hasattr(self, 'tdel'):
            self.calc_sspec()
        delmax = np.max(self.tdel) if delmax is None else delmax
        if lamsteps:
            if not hasattr(self, 'lamsspec'):
                self.calc_sspec(lamsteps=lamsteps)
            sspec = np.array(cp(self.lamsspec))
            yaxis = cp(self.beta)
        else:
            if not hasattr(self, 'sspec'):
                self.calc_sspec()
            sspec = np.array(cp(self.sspec))
            yaxis = cp(self.tdel)
        ind = np.argmin(abs(self.tdel - delmax))
        ymax = self.beta[ind]       # the reference reads self.beta in both modes (:1089)

        nr, nc = np.shape(sspec)
        # noise estimate from the outer quadrants (dynspec.py:1093-1097)
        a = np.array(sspec[int(nr / 2):, int(nc / 2 + np.ceil(cutmid / 2)):].ravel())
        b = np.array(sspec[int(nr / 2):, 0:int(nc / 2 - np.floor(cutmid / 2))].ravel())
        noise = np.std(np.concatenate((a, b)))
        ind = np.argmin(abs(self.tdel - delmax))
        yaxis = yaxis[0:ind]
        noise = np.sqrt(np.sum(np.power(noise, 2))) / np.sqrt(len(yaxis) * 2)
        self.noise = noise

        if etamax is None:
            etamax = ymax / ((self.fdop[1] - self.fdop[0]) * cutmid) ** 2
        if etamin is None:
            etamin = (yaxis[1] - yaxis[0]) * startbin / (max(self.fdop)) ** 2
        try:
            len(etamin)
            etamin_array = np.array(etamin).squeeze()
            etamax_array = np.array(etamax).squeeze()
        except TypeError:
            etamin_array = np.array([etamin])
            etamax_array = np.array([etamax])
        max_sqrt_eta = np.sqrt(np.max(etamax_array))
        min_sqrt_eta = np.sqrt(np.min(etamin_array))
        sqrt_eta_all = np.linspace(min_sqrt_eta, max_sqrt_eta, int(numsteps))

        for iarc in range(0, len(etamin_array)):
            if len(etamin_array) != 1:
                etamin = etamin_array.squeeze()[iarc]
                etamax = etamax_array.squeeze()[iarc]
            if not lamsteps:
                c = 299792458.0
                beta_to_eta = c * 1e6 / ((ref_freq * 10 ** 6) ** 2)
                etamax = etamax / (self.freq / ref_freq) ** 2
                etamax = etamax * beta_to_eta
                etamin = etamin / (self.freq / ref_freq) ** 2
                etamin = etamin * beta_to_eta
                constraint = constraint / (self.freq / ref_freq) ** 2
                constraint = constraint * beta_to_eta
            sqrt_eta = sqrt_eta_all[(sqrt_eta_all <= np.sqrt(etamax)) *
                                    (sqrt_eta_all >= np.sqrt(etamin))]
            numsteps_new = len(sqrt_eta)

            # delay-scrunched profile on the normalised Doppler axis (device)
            self.norm_sspec(eta=etamin, delmax=delmax, plot=False, startbin=startbin,
                            maxnormfac=1, cutmid=cutmid, lamsteps=lamsteps, scrunched=True,
                            logsteps=logsteps, plot_fit=False, numsteps=numsteps_new,
                            fit_spectrum=fit_spectrum, subtract_artefacts=subtract_artefacts,
                            velocity=velocity, weighted=weighted)
            norm_sspec = self.normsspecavg.squeeze()
            etafrac_array = self.normsspec_fdop
            ind1 = np.argwhere(etafrac_array >= 0)
            ind2 = np.argwhere(etafrac_array < 0)
            if asymm:
                norm_sspec_avg1 = np.array(norm_sspec[ind1])
                norm_sspec_avg2 = np.flip(norm_sspec[ind2], axis=0)
                nspec = 2
            else:
                norm_sspec_avg = np.add(norm_sspec[ind1], np.flip(norm_sspec[ind2], axis=0)) / 2
                nspec = 1
            etafrac_array_avg_orig = 1 / etafrac_array[ind1].squeeze()

            for dummy in range(0, nspec):
                etafrac_array_avg = etafrac_array_avg_orig
                if asymm and dummy == 0:
                    spec = np.array(norm_sspec_avg1)
                elif asymm and dummy == 1:
                    spec = np.array(norm_sspec_avg2)
                else:
                    spec = np.array(norm_sspec_avg)
                spec = spec.squeeze()
                filt_ind = is_valid(spec)
                spec = np.flip(spec[filt_ind], axis=0)
                etafrac_array_avg = np.flip(etafrac_array_avg[filt_ind], axis=0)

                etaArray = etamin * etafrac_array_avg ** 2
                ind = np.argwhere(etaArray < etamax)
                etaArray = etaArray[ind].squeeze()
                spec = spec[ind].squeeze()
                norm_sspec_avg_filt = savgol_filter(spec, nsmooth, 1)

                indrange = np.argwhere((etaArray > constraint[0]) * (etaArray < constraint[1]))
                sumpow_inrange = norm_sspec_avg_filt[indrange]
                ind = np.argmin(np.abs(norm_sspec_avg_filt - np.max(sumpow_inrange)))

                # window from low_power_diff (low-curvature side) to high_power_diff
                max_power = norm_sspec_avg_filt[ind]
                power = max_power
                ind1 = 1
                while (power > max_power + low_power_diff and
                       ind + ind1 < len(norm_sspec_avg_filt) - 1):
                    ind1 += 1
                    power = norm_sspec_avg_filt[ind - ind1]
                power = max_power
                ind2 = 1
                while (power > max_power + high_power_diff and
                       ind + ind2 < len(norm_sspec_avg_filt) - 1):
                    ind2 += 1
                    power = norm_sspec_avg_filt[ind + ind2]
                xdata = etaArray[int(ind - ind1):int(ind + ind2)]
                ydata = spec[int(ind - ind1):int(ind + ind2)]
                if log_parabola:
                    yfit, eta, etaerr = fit_log_parabola(xdata, ydata)
                else:
                    yfit, eta, etaerr = fit_parabola(xdata, ydata)
                if np.mean(np.gradient(np.diff(yfit))) > 0:
                    raise ValueError('Fit returned a forward parabola.')

                if noise_error:
                    etaerr2 = etaerr    # error from the parabola fit
                    power = max_power
                    ind1 = 1
                    while (power > (max_power - noise) and (ind - ind1 > 1)):
                        power = norm_sspec_avg_filt[ind - ind1]
                        ind1 += 1
                    power = max_power
                    ind2 = 1
                    while (power > (max_power - noise) and
                           (ind + ind2 < len(norm_sspec_avg_filt) - 1)):
                        ind2 += 1
                        power = norm_sspec_avg_filt[ind + ind2]
                    etaerr = np.abs(etaArray[int(ind - ind1)] - etaArray[int(ind + ind2)]) / 2

                self.eta_array = etaArray
                sigma = self.noise * efac
                prob = 1 / (sigma * np.sqrt(2 * np.pi)) * \
                    np.exp(-0.5 * ((spec - np.max(spec)) / sigma) ** 2)
                if asymm:
                    if dummy == 0:
                        self.norm_sspec_avg1 = spec
                        self.prob_eta_peak1 = prob
                    else:
                        self.norm_sspec_avg2 = spec
                        self.prob_eta_peak2 = prob
                else:
                    self.norm_sspec_avg = spec
                    self.prob_eta_peak = prob

                if iarc == 0:   # save primary
                    pre = "betaeta" if lamsteps else "eta"
                    if asymm and dummy == 0:
                        suf = "_left"
                    elif dummy == 1:
                        suf = "_right"
                    else:
                        suf = ""
                    setattr(self, pre + suf, eta)
                    setattr(self, pre + "err" + suf, etaerr / np.sqrt(2))
                    setattr(self, pre + "err2" + suf, etaerr2 / np.sqrt(2))
            self.norm_delmax = delmax
