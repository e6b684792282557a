"""taudem_b200 — H100-native TauDEM flow-direction / contributing-area path.

Python is only a thin ctypes binding over the C ABI in ``include/taudem_b200.h``
(``taudem_b200/lib/libtaudem_b200.so``).  The functions mirror the reference's
library entry points (``flood``, ``setdird8``, ``setdir``, ``aread8``, ``area``;
reference src/flood.h, src/d8.h:7, src/tardemlib.h:70, src/aread8.h:3,
src/areadinf.h:2) at file level, and offer the same computations on numpy
arrays (host-grid level).  There is no CPU fallback: without the shared
library or without a CUDA device every compute call raises.
"""
from ._lib import (TaudemError, lib, version, device_count, launch_count, reset_launch_count,
                   last_compute_seconds)
from .api import (flood, setdird8, setdir, aread8, area,
                  pitremove_grid, d8flowdir_grid, dinfflowdir_grid, aread8_grid, areadinf_grid, contributing_areas_grid, threshold_grid, twi_grid, slopearea_grid, slopearearatio_grid, d8flowpathextremeup_grid, dinfdecayaccum_grid, dinfconclimaccum_grid, dinftranslimaccum_grid, gridnet_grid,
                  peukerdouglas_grid, lengtharea_grid, slopeavedown_grid, flowdircond_grid, retlimflow_grid,
                  d8hdisttostrm_grid, d8vdisttostrm_grid, dinfdistdown_grid, read_raster, write_raster, raster_info, nameadd, read_outlets)

__all__ = [
    "TaudemError", "lib", "version", "device_count", "launch_count", "reset_launch_count",
    "last_compute_seconds", "flood", "setdird8", "setdir", "aread8", "area", "pitremove_grid",
    "d8flowdir_grid", "dinfflowdir_grid", "aread8_grid", "areadinf_grid", "contributing_areas_grid", "threshold_grid", "twi_grid", "slopearea_grid", "slopearearatio_grid", "d8flowpathextremeup_grid", "dinfdecayaccum_grid", "dinfconclimaccum_grid", "dinftranslimaccum_grid", "gridnet_grid", "peukerdouglas_grid",
    "lengtharea_grid", "slopeavedown_grid", "flowdircond_grid", "retlimflow_grid", "d8hdisttostrm_grid", "d8vdisttostrm_grid", "dinfdistdown_grid",
    "read_raster", "write_raster", "raster_info", "nameadd", "read_outlets",
]
