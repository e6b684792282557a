"""ctypes loader for libtaudem_b200.so (the C ABI declared in include/taudem_b200.h)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtaudem_b200.so")


class TaudemError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"taudem_b200 error {code}: {msg}")
        self.code = code


class Strip(C.Structure):
    _fields_ = [("nx", C.c_int), ("ny", C.c_int), ("pitch", C.c_int), ("has_top", C.c_int), ("has_bot", C.c_int)]


_lib = None

# name -> (restype, argtypes).  Every symbol include/taudem_b200.h declares is listed;
# tests/test_abi.py checks the shared library exports all of them.
_P = C.c_void_p
_S = C.c_char_p
_I = C.c_int
_F = C.c_float
_D = C.c_double
SIGNATURES = {
    "td_version": (_S, []),
    "td_last_error": (_S, []),
    "td_device_count": (_I, []),
    "td_warmup": (_I, []),
    "td_set_device": (_I, [_I]),
    "td_launch_count": (C.c_ulonglong, []),
    "td_reset_launch_count": (None, []),
    "td_last_compute_seconds": (_D, []),
    "td_flood": (_I, [_S, _S, _S, _I, _I, _I, _I, _S]),
    "td_setdird8": (_I, [_S, _S, _S, _S, _I]),
    "td_setdir": (_I, [_S, _S, _S, _S, _I]),
    "td_aread8": (_I, [_S, _S, _S, _S, _I, _I, _S, _I, _I, _I]),
    "td_area": (_I, [_S, _S, _S, _S, _I, _I, _S, _I, _I, _I]),
    "td_d8flowpathextremeup": (_I, [_S, _S, _S, _I, _S, _S, _I, _I, _I, _I]),
    "td_d8flowpathextremeup_host": (_I, [_P, _P, _P, _I, _I, C.c_int16, _I, _I, _P, _P, _I]),
    "td_gridnet": (_I, [_S, _S, _S, _S, _S, _S, _S, _I, _I, _I, _I, _I]),
    "td_gridnet_host": (_I, [_P, _P, _I, _P, _P, _P, _I, _I, C.c_int16, _P, _P, _P, _P, _I]),
    "td_dmarea": (_I, [_S, _S, _S, _S, _S, _I, _I, _S, _I, _I, _I]),
    "td_dinfdecayaccum_host": (_I, [_P, _P, _P, _P, _I, _I, C.c_float, C.c_float, _P, _P, _I, _P, _P, _I]),
    "td_dsllarea": (_I, [_S, _S, _S, _S, _S, _I, _I, _S, _S, _I, _I, _F]),
    "td_tlaccum": (_I, [_S, _S, _S, _S, _S, _S, _S, _S, _S, _I, _I, _I, _I, _I]),
    "td_dinfconclimaccum_host": (_I, [_P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _P, _P, _I, _P, _P, _I]),
    "td_dinftranslimaccum_host": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _P, _P, _I, _P, _P, _I]),
    "td_threshold": (_I, [_S, _S, _S, _F, _I]),
    "td_twigrid": (_I, [_S, _S, _S]),
    "td_threshold_host": (_I, [_P, _P, _P, _I, _I, _F, _F]),
    "td_twi_host": (_I, [_P, _P, _P, _I, _I, _F, _F]),
    "td_slopearea": (_I, [_S, _S, _S, _P]),
    "td_atanbgrid": (_I, [_S, _S, _S]),
    "td_slopearea_host": (_I, [_P, _P, _P, _I, _I, _F, _F]),
    "td_slopearearatio_host": (_I, [_P, _P, _P, _I, _I, _F]),
    "td_slopearea_dev": (_I, [_P, _P, _P, _P, Strip, _F, _F, _P]),
    "td_slopearearatio_dev": (_I, [_P, _P, _P, _P, Strip, _F, _P]),
    "td_threshold_dev": (_I, [_P, _P, _P, _P, Strip, _F, _F, _P]),
    "td_twi_dev": (_I, [_P, _P, _P, _P, Strip, _F, _F, _P]),
    "td_peukerdouglas": (_I, [_S, _S, _P]),
    "td_lengtharea": (_I, [_S, _S, _S, _P]),
    "td_peukerdouglas_host": (_I, [_P, _P, _I, _I, _F, _P]),
    "td_lengtharea_host": (_I, [_P, _P, _P, _I, _I, _F, _F]),
    "td_peukerdouglas_smooth_dev": (_I, [_P, _P, _P, Strip, _F, _P, _P]),
    "td_peukerdouglas_mark_dev": (_I, [_P, _P, _P, Strip, _F, _P]),
    "td_lengtharea_dev": (_I, [_P, _P, _P, _P, Strip, _F, _F, _P]),
    "td_sloped": (_I, [_S, _S, _S, _D]),
    "td_slopeavedown_host": (_I, [_P, _P, _P, _I, _I, _F, C.c_int16, _P, _P, _D, _D, _D]),
    "td_slopeavedown_init_dev": (_I, [_P, _P, _P, _P, _P, _P, _P, Strip, C.c_int16, _F, _P]),
    "td_slopeavedown_pass_dev": (_I, [_P, _P, _P, _P, _P, _P, Strip, _P, _D, _P, _P]),
    "td_slopeavedown_niter": (_I, [_D, _D, _D, _P]),
    "td_distgrid": (_I, [_S, _S, _S, _I]),
    "td_d8vdistdown": (_I, [_S, _S, _S, _S, _I]),
    "td_d8hdisttostrm_host": (_I, [_P, _P, _P, _I, _I, C.c_int16, C.c_int32, _I, _P, _P]),
    "td_d8vdisttostrm_host": (_I, [_P, _P, _P, _P, _I, _I, C.c_int16, C.c_int32, _I]),
    "td_disttostrm_last_levels": (C.c_longlong, []),
    "td_disttostrm_seed_dev": (_I, [_P, _P, _P, _P, _P, Strip, _I, C.c_int16, C.c_int32, _P]),
    "td_disttostrm_levels_dev": (_I, [_P, _I, _P, _P, _P, _P, Strip, _P, _P, _P]),
    "td_dinfdistdown": (_I, [_S, _S, _S, _S, _S, _S, _I, _I, _I, _I]),
    "td_dinfdistdown_host": (_I, [_P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _P, _P, _I, _I, _I]),
    "td_dinfdistdown_last_levels": (C.c_longlong, []),
    "td_dinfdistdown_seed_dev": (_I, [_P, _P, _P, _P, _P, _P, Strip, _F, _P, _P, _P]),
    "td_dinfdistdown_levels_dev": (_I, [_P, _I, _I, _P, _P, _P, _P, _P, _P, _P, Strip, _F, _F, _I, _P, _P, _P, _P]),
    "td_dinfdistdown_edge_dev": (_I, [_P, _P, _P, _P, Strip, _P]),
    "td_dinfdistdown_pythagoras_dev": (_I, [_P, _P, _P, Strip, _P]),
    "td_flowdircond": (_I, [_S, _S, _S]),
    "td_flowdircond_host": (_I, [_P, _P, _P, _I, _I, C.c_int16, _F]),
    "td_flowdircond_deps_dev": (_I, [_P, _P, _P, _P, Strip, C.c_int16, _P]),
    "td_flowdircond_sweep_run_dev": (_I, [_P, _P, _P, Strip, _F, _P, _P]),
    "td_retlimro": (_I, [_S, _S, _S, _S]),
    "td_retlimflow_host": (_I, [_P, _P, _P, _P, _I, _I, _F, _F, _F, _P, _P]),
    "td_retlimflow_deps_dev": (_I, [_P, _P, _P, _P, _P, Strip, _F, _F, _F, _P, _P, _P]),
    "td_retlimflow_sweep_run_dev": (_I, [_P, _P, _P, _P, _P, Strip, _F, _F, _P, _P, _P]),
    "td_nameadd": (_I, [_S, _S, _S]),
    "td_raster_info": (_I, [_S] + [_P] * 9),
    "td_raster_read": (_I, [_S, _I, _P, _I, _I]),
    "td_raster_cell_sizes": (_I, [_S, _P, _P, _I]),
    "td_raster_write": (_I, [_S, _I, _P, _I, _I, _D, _S, _D, _D, _I]),
    "td_flood_host": (_I, [_P, _P, _P, _I, _I, _F, _I]),
    "td_setdird8_host": (_I, [_P, _P, _P, _I, _I, _F, _P, _P]),
    "td_setdir_host": (_I, [_P, _P, _P, _I, _I, _F, _P, _P]),
    "td_aread8_host": (_I, [_P, _P, _P, _I, _I, C.c_int16, _F, _I]),
    "td_area_host": (_I, [_P, _P, _P, _I, _I, _F, _F, _P, _P, _I]),
    "td_contributing_areas_host": (_I, [_P, _P, _P, _P, _I, _I, C.c_int16, _F, _P, _P, _I]),
    "td_aread8_outlets_host": (_I, [_P, _P, _P, _I, _I, C.c_int16, _F, _I, _P, _P, _I]),
    "td_area_outlets_host": (_I, [_P, _P, _P, _I, _I, _F, _F, _P, _P, _I, _P, _P, _I]),
    "td_sweep_restrict_dev": (_I, [_P, Strip, _P, _P, _I, _P]),
    "td_sweep_restrict_round_dev": (_I, [_P, Strip, _P, _P, _I, _P, _P, _P, _I, _P]),
    "td_outlets_read": (_I, [C.c_char_p, C.c_char_p, _I, _I, _P, _P, _I, _P]),
    "td_ctx_create": (_P, []),
    "td_ctx_destroy": (None, [_P]),
    "td_pitch_for": (_I, [_I]),
    "td_ctx_counter": (C.c_ulonglong, [_P, _I]),
    "td_gen_dem_dev": (_I, [_P, Strip, _I, _I, C.c_uint, _F, _F, _P]),
    "td_gen_weights_dev": (_I, [_P, Strip, _I, C.c_uint, _P]),
    "td_flood_init_dev": (_I, [_P, _P, _P, _P, Strip, _F, _I, _P]),
    "td_flood_relax_dev": (_I, [_P, _P, _P, Strip, _I, _P, _P]),
    "td_flood_relax_edges_dev": (_I, [_P, _P, _P, Strip, _I, _P, _P]),
    "td_d8_slopes_dev": (_I, [_P, _P, _P, _P, Strip, _F, _P, _P, _P, _P]),
    "td_d8_flats_dev": (_I, [_P, _P, _P, Strip, _P, _P, _P, _P]),
    "td_d8_flats_strip_dev": (_I, [_P, _P, _P, Strip, _P, _P, _P, _P, _P]),
    "td_dinf_flats_strip_dev": (_I, [_P, _P, _P, Strip, _P, _P, _P, _P, _P]),
    "td_dinf_slopes_dev": (_I, [_P, _P, _P, _P, Strip, _F, _P, _P, _P, _P]),
    "td_dinf_flats_dev": (_I, [_P, _P, _P, Strip, _P, _P, _P, _P]),
    "td_aread8_deps_dev": (_I, [_P, _P, _P, Strip, C.c_int16, _P]),
    "td_aread8_sweep_dev": (_I, [_P, _P, _P, Strip, _F, _I, _I, _P]),
    "td_area_deps_dev": (_I, [_P, _P, _P, Strip, _F, _P, _P, _P]),
    "td_area_sweep_dev": (_I, [_P, _P, _P, _P, Strip, _I, _I, _P, _P]),
    "td_sweep_begin_dev": (_I, [_P, Strip, _P]),
    "td_sweep_apply_halo_dev": (_I, [_P, Strip, _P, _P, _P]),
    "td_aread8_sweep_run_dev": (_I, [_P, _P, _P, Strip, _F, _I, _I, _P, _P]),
    "td_sweep_peer_export_dev": (_I, [_P, Strip, _I, _P, _P, _P]),
    "td_sweep_peer_connect_dev": (_I, [_P, _I, _P, _P]),
    "td_sweep_peer_begin_dev": (_I, [_P, Strip, _P]),
    "td_sweep_peer_off_dev": (None, [_P]),
    "td_set_halo_cell_sizes_dev": (None, [_P, _D, _D, _D, _D]),
    "td_area_sweep_run_dev": (_I, [_P, _P, _P, _P, Strip, _I, _I, _P, _P, _P]),
    "td_d8flowpathextremeup_deps_dev": (_I, [_P, _P, _P, Strip, C.c_int16, _P]),
    "td_d8flowpathextremeup_sweep_run_dev": (_I, [_P, _P, _P, Strip, _I, _I, _P, _P]),
    "td_dinfdecayaccum_deps_dev": (_I, [_P, _P, _P, Strip, _F, _P, _P, _P]),
    "td_dinfdecayaccum_sweep_run_dev": (_I, [_P, _P, _P, _P, _P, Strip, _F, _I, _P, _P, _P]),
    "td_dinfconclimaccum_deps_dev": (_I, [_P, _P, _P, Strip, _F, _P, _P, _P]),
    "td_dinfconclimaccum_sweep_run_dev": (_I, [_P, _P, _P, _P, _P, _P, Strip, _F, _F, _F, _I, _P, _P, _P]),
    "td_dinftranslimaccum_deps_dev": (_I, [_P, _P, _P, _P, _P, Strip, _F, _P, _P, _P]),
    "td_dinftranslimaccum_sweep_run_dev": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, Strip, _F, _F, _F, _I, _P, _P, _P]),
    "td_gridnet_mask_dev": (_I, [_P, _P, _P, Strip, _I, _P]),
    "td_gridnet_deps_dev": (_I, [_P, _P, _P, Strip, C.c_int16, _P]),
    "td_gridnet_sweep_run_dev": (_I, [_P, _I, _P, _P, _P, Strip, _I, _P, _P]),
    "td_gridnet_order_dev": (_I, [_P, _P, _P, _P, _P, Strip, C.c_int16, _I, _P]),
}


def lib():
    """Returns the loaded C-ABI library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TaudemError(-1, f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                  "(make -C taudem_b200/csrc); there is no CPU fallback")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc):
    if rc != 0:
        raise TaudemError(rc, lib().td_last_error().decode(errors="replace"))


def version():
    return lib().td_version().decode()


def device_count():
    return lib().td_device_count()


def launch_count():
    return int(lib().td_launch_count())


def reset_launch_count():
    lib().td_reset_launch_count()


def last_compute_seconds():
    return float(lib().td_last_compute_seconds())
