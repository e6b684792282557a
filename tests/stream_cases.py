"""Inputs of the stream-definition tests (peukerdouglas, lengtharea): the DEMs, the reference calls whose outputs are recorded in
tests/golden/stream_reference.json, and the two documented workflows

    peukerdouglas -> aread8 -wg ss -> threshold         (Peuker-Douglas curvature)
    gridnet (plen) + aread8 -> lengtharea               (length-area)

shared by tests/test_stream_definition.py (CPU: replay, emulated kernels) and tests/test_gpu_stream_definition.py (GPU)."""
import numpy as np

from taudem_b200 import synth

ND = np.float32(-3.0e38)
PD_WEIGHTS = (None, (0.5, 0.0, 0.2), (1.0, 0.3, 0.0))       # None = the tool's defaults 0.4 0.1 0.05
PD_RANKS = (1, 3)
LA_PAR = ((None, None), (0.01, 1.5), (0.03, 1.0))            # (M, y); None = the defaults 0.03 1.3
PD_THRESH = 5.0


def rough():
    """a rough DEM quantised to half units: plateaus and exact ties inside groups of four"""
    d = synth.gen_dem(61, 47, hurst=0.5, tilt=1.0, seed=11)
    return (np.round(d * 2.0) / 2.0).astype(np.float32)


def holes():
    """an odd shape with nodata holes: blobs, single cells, cells on every edge and in the corners"""
    d = synth.punch_holes(synth.gen_dem(53, 131, hurst=0.8, tilt=2.0, seed=12), nodata=float(ND), seed=3).astype(np.float32)
    d[0, 5:9] = ND; d[-1, 17] = ND; d[20:23, 0] = ND; d[31, -1] = ND; d[0, 0] = ND; d[-1, -1] = ND
    d[10, 40] = ND; d[11, 42] = ND; d[40, 100] = ND; d[1, 60] = ND; d[-2, 61] = ND
    return d


DEMS = {"rough": rough, "holes": holes}


def pd_calls():
    """(name, dem, weights, ranks) of every recorded peukerdouglas call"""
    out = []
    for name, make in DEMS.items():
        for w in PD_WEIGHTS:
            for ranks in PD_RANKS:
                out.append((name, make(), w, ranks))
    return out


def la_inputs():
    """(plen, ad8 unweighted, ad8 weighted) of a filled DEM by the C restatement: gridnet's longest path and aread8 (the weighted
    contributing area has fractions, which lengtharea rounds half away from zero)"""
    import port
    dem = synth.gen_dem(67, 89, hurst=0.7, tilt=2.0, seed=21)
    p, _ = port.d8flowdir(port.pitremove(dem))
    plen = port.gridnet(p)[0]
    ad8 = port.aread8(p)
    w = (synth.gen_weights(*dem.shape) * np.float32(2.5)).astype(np.float32)
    ad8w = port.aread8(p, weights=w)
    return plen, ad8, ad8w


def pd_workflow(R, dem):
    """the Peuker-Douglas chain on a RefPipeline: (fel, p, ss, ad8 weighted by ss, src)"""
    fel = R.pitremove(dem)
    p, _ = R.d8flowdir(fel)
    ss = R.peukerdouglas(fel)
    ssa = R.aread8(p, weights=np.asarray(ss, np.float32))
    src = R.threshold(ssa, PD_THRESH)
    return fel, p, ss, ssa, src


def la_workflow(R, dem):
    """the length-area chain on a RefPipeline: (fel, p, plen, ad8, ss)"""
    fel = R.pitremove(dem)
    p, _ = R.d8flowdir(fel)
    plen = R.gridnet(p)[0]
    ad8 = R.aread8(p)
    ss = R.lengtharea(plen, ad8)
    return fel, p, plen, ad8, ss


def workflow_dem():
    return synth.gen_dem(72, 96, hurst=0.75, tilt=2.0, seed=31)
