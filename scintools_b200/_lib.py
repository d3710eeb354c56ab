"""ctypes binding of libscint_b200.so (C ABI in include/scint_b200.h).

There is NO fallback: if the shared library is missing this module raises at
import time; if no sm_90 device is present the first device call raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libscint_b200.so")


class SbError(RuntimeError):
    """A libscint_b200 call returned a non-zero status."""


if not os.path.exists(LIB_PATH):
    raise ImportError(
        "scintools_b200: %s not found. Build it with "
        "`python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
        "There is no CPU fallback." % LIB_PATH)

lib = ctypes.CDLL(LIB_PATH)

c_int = ctypes.c_int32
c_i64 = ctypes.c_int64
c_dbl = ctypes.c_double
c_flt = ctypes.c_float
vp = ctypes.c_void_p


class ThthGeom(ctypes.Structure):
    """struct sb_thth_geom"""
    _fields_ = [
        ("cs", vp), ("ntau", c_i64), ("nfd", c_i64),
        ("tau0", c_dbl), ("dtau", c_dbl), ("tau_absmax", c_dbl),
        ("fd0", c_dbl), ("dfd", c_dbl), ("fd_half", c_dbl),
        ("th_cents", vp), ("th_cents_host", vp),
        ("n_th", c_int), ("coherent", c_int),
        ("cs_pitch", c_i64), ("cs_half", c_int), ("cs_valid_cols", c_int),
        ("cs_bound", vp),
    ]


class SimParams(ctypes.Structure):
    """struct sb_sim_params"""
    _fields_ = [("nx", c_int), ("ny", c_int), ("dx", c_dbl), ("dy", c_dbl),
                ("alpha", c_dbl), ("ar", c_dbl), ("psi", c_dbl),
                ("inner", c_dbl), ("consp", c_dbl)]


class ScintFit(ctypes.Structure):
    """struct sb_scint_fit"""
    _fields_ = [("acf", vp), ("aux", vp), ("pitch", c_i64), ("s0", c_dbl), ("s1", c_dbl),
                ("c", c_dbl), ("p0", c_dbl * 5),
                ("r0", c_int), ("c0", c_int), ("r1", c_int), ("c1", c_int), ("n0", c_int),
                ("n1", c_int), ("shf", c_int), ("sht", c_int), ("pf", c_int), ("pt", c_int),
                ("zf", c_int), ("zt", c_int), ("vary", c_int), ("bounded", c_int),
                ("weighted", c_int), ("max_nfev", c_int)]



class AcfModel(ctypes.Structure):
    """struct sb_acf_model"""
    _fields_ = [("snp", vp), ("snp2", vp), ("dnun", vp), ("snx", vp), ("sny", vp),
                ("n1", c_int), ("n2", c_int), ("ndnun", c_int), ("nsn", c_int),
                ("quadrant", c_int), ("sigxn", c_dbl), ("sigyn", c_dbl), ("sqrtar", c_dbl),
                ("alph2", c_dbl), ("step1", c_dbl), ("step2", c_dbl), ("wn_amp", c_dbl),
                ("amp", c_dbl)]


_SIGS = {
    "sb_abi_version": (c_int, []),
    "sb_last_error": (ctypes.c_char_p, []),
    "sb_init": (c_int, [c_int]),
    "sb_release": (c_int, []),
    "sb_launch_count": (c_i64, []),
    "sb_profile_enable": (c_int, [c_int]),
    "sb_profile_collect": (c_int, [vp, vp, c_int]),
    "sb_eta_sweep": (c_int, [ctypes.POINTER(ThthGeom), vp, c_int, c_dbl, c_int,
                             vp, vp, vp, vp, vp]),
    "sb_thth_map": (c_int, [ctypes.POINTER(ThthGeom), c_dbl, c_int, vp, vp, vp,
                            vp, vp, vp, vp]),
    "sb_thin_sweep": (c_int, [ctypes.POINTER(ThthGeom), vp, c_int, c_dbl, c_int, vp, vp,
                              c_int, c_dbl, c_int, vp, vp, vp, vp, vp, vp]),
    "sb_thin_map": (c_int, [ctypes.POINTER(ThthGeom), vp, c_int, c_int, c_dbl, c_dbl, vp,
                            vp, vp]),
    "sb_sspec_f32": (c_int, [vp, c_int, c_int, vp, vp, c_dbl, c_dbl, c_int,
                             c_int, c_int, vp, vp, vp, vp]),
    "sb_rev_map": (c_int, [vp, c_int, vp, c_dbl, c_dbl, c_dbl, c_int, c_dbl, c_dbl, c_int,
                           c_int, vp, vp]),
    "sb_herm_eigvec": (c_int, [vp, c_int, c_int, c_dbl, c_int, vp, vp, vp, vp]),
    "sb_chisq_sweep": (c_int, [ctypes.POINTER(ThthGeom), vp, c_int, vp, c_dbl, c_dbl, vp,
                               c_int, c_int, vp, c_dbl, c_int, vp, vp, vp, vp, vp, vp]),
    "sb_gerchberg_saxton_f32": (c_int, [vp, vp, vp, c_int, c_int, c_int, vp]),
    "sb_scale_dyn_lambda_f32": (c_int, [vp, c_int, c_int, c_int, vp, vp, vp, vp, c_flt, c_flt,
                                        vp, vp, c_int, vp, vp]),
    "sb_norm_sspec_f32": (c_int, [vp, c_int, c_int, vp, vp, c_dbl, c_dbl, vp, c_int, vp, vp, vp]),
    "sb_norm_sspec_avg_f32": (c_int, [vp, c_int, c_int, vp, vp, vp]),
    "sb_ifft2_c2c_f32": (c_int, [vp, c_int, c_int, c_int, c_int, c_int, c_dbl, c_int, vp, vp]),
    "sb_acf_f32": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp]),
    "sb_acf_sspec_f32": (c_int, [vp, c_int, c_int, vp, vp, c_dbl, c_dbl, c_int, vp, vp]),
    "sb_sspec_tiles_f32": (c_int, [vp, c_int, c_int, c_int, c_int, c_int, c_int, vp, vp, c_dbl,
                                   c_dbl, vp, vp]),
    "sb_acf_tiles_f32": (c_int, [vp, c_int, c_int, c_int, c_int, c_int, c_int, vp, vp]),
    "sb_cs_f32": (c_int, [vp, c_int, c_int, c_int, c_flt, vp, c_int, c_i64, c_int, vp, vp]),
    "sb_cs_bound_f32": (c_int, [vp, c_int, c_int, c_int, c_flt, vp, vp]),
    "sb_cs_c2c_f32": (c_int, [vp, c_int, c_int, c_int, c_flt, c_flt, vp, vp, vp]),
    "sb_vlbi_retrieval": (c_int, [ctypes.POINTER(ThthGeom), vp, c_int, c_dbl, vp, c_dbl, c_dbl,
                                  c_int, c_int, c_dbl, c_int, vp, vp, vp, vp, vp]),
    "sb_asymmetry_batch": (c_int, [ctypes.POINTER(ThthGeom), c_int, vp, c_dbl, c_int, vp, vp, vp,
                                   vp, vp, vp, vp]),
    "sb_mosaic_build": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp, vp, vp]),
    "sb_mosaic_rot": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp]),
    "sb_mosaic_overlap": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp]),
    "sb_mosaic_fit": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp]),
    "sb_mosaic_hess": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp, vp, vp,
                               vp]),
    "sb_svd_topk": (c_int, [vp, c_int, c_int, c_int, vp, vp, vp, vp, vp, vp]),
    "sb_svd_apply": (c_int, [vp, c_int, c_int, c_int, vp, vp, vp, vp]),
    "sb_bandpass_rows": (c_int, [vp, c_int, c_int, c_int, vp, vp]),
    "sb_bandpass_cols": (c_int, [vp, c_int, c_int, c_int, vp, vp, vp]),
    "sb_bandpass_divide": (c_int, [vp, c_int, c_int, c_int, vp, vp, vp, vp]),
    "sb_slow_ft_f32": (c_int, [vp, c_int, c_int, vp, vp, vp]),
    "sb_inpaint_biharmonic_f64": (c_int, [vp, c_int, c_int, vp, c_int, vp, vp, c_int, vp, c_int,
                                          c_dbl, c_dbl, c_dbl, c_int, vp, vp, vp, vp]),
    "sb_medfilt_masked_f64": (c_int, [vp, c_int, c_int, vp, c_int, c_int, c_int, c_dbl, vp, vp]),
    "sb_scint_fit_1d": (c_int, [ctypes.POINTER(ScintFit), c_int, vp, vp, vp]),
    "sb_scint_fit_2d": (c_int, [ctypes.POINTER(ScintFit), c_int, vp, vp, vp]),
    "sb_acf_model_f64": (c_int, [ctypes.POINTER(AcfModel), vp, vp, vp]),
    "sb_sim_weights": (c_int, [ctypes.POINTER(SimParams), vp, vp]),
    "sb_sim_screen": (c_int, [c_int, c_int, vp, vp, vp, ctypes.c_uint64, vp, vp]),
    "sb_sim_intensity": (c_int, [c_int, c_int, c_int, vp, vp, c_dbl, c_dbl, vp,
                                 vp, vp]),
    "sb_convert_f64_f32": (c_int, [vp, vp, c_i64, vp]),
    "sb_convert_f32_f64": (c_int, [vp, vp, c_i64, vp]),
}

EXPORTS = tuple(_SIGS)


class Brightness(ctypes.Structure):
    """struct sb_brightness (include/scint_b200_brightness.h)"""
    _fields_ = [("nset", c_int), ("n", c_int), ("ntd", c_int), ("nfd", c_int), ("stages", c_int),
                ("x", vp), ("diag", vp), ("td", vp), ("par", vp), ("colx", vp), ("colq", vp),
                ("half_df", c_dbl), ("jac_cap", c_dbl), ("jac_out", c_dbl),
                ("rho", vp), ("B", vp), ("thetax", vp), ("thetay", vp), ("jac", vp), ("ss", vp),
                ("lss", vp), ("acf", vp)]


# entry points declared in include/scint_b200_brightness.h, outside scint_b200.h's set
BRIGHTNESS_SIGS = {
    "sb_brightness_f64": (c_int, [ctypes.POINTER(Brightness), vp]),
}


class ScatIm(ctypes.Structure):
    """struct sb_scatim (include/scint_b200_scatim.h)"""
    _fields_ = [("nitem", c_int), ("mx", c_int), ("my", c_int), ("nx", c_int), ("ny", c_int),
                ("shift", c_int), ("pitch", c_i64), ("sspec", vp), ("offset", vp), ("eta", vp),
                ("tx", vp), ("fx", vp), ("ty", vp), ("fy", vp), ("ax", vp), ("ay", vp),
                ("image", vp)]


# entry points declared in include/scint_b200_scatim.h, outside scint_b200.h's set
SCATIM_SIGS = {
    "sb_scattered_image_f64": (c_int, [ctypes.POINTER(ScatIm), vp]),
}

# entry points declared in include/scint_b200_clean.h, outside scint_b200.h's set
CLEAN_SIGS = {
    "sb_dyn_zero_counts_f64": (c_int, [vp, c_int, c_int, c_int, c_int, vp, vp, vp]),
    "sb_zap_f64": (c_int, [vp, c_i64, c_dbl, vp, vp]),
}

for _name, (_res, _args) in (list(_SIGS.items()) + list(BRIGHTNESS_SIGS.items()) +
                             list(SCATIM_SIGS.items()) + list(CLEAN_SIGS.items())):
    _fn = getattr(lib, _name)   # AttributeError here = ABI mismatch, fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


def check(rc):
    if rc != 0:
        msg = lib.sb_last_error()
        raise SbError("libscint_b200 error %d: %s" %
                      (rc, msg.decode() if msg else "?"))
