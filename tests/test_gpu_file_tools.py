"""Every executable once on a small DEM chain (pitremove -> flow directions -> areas -> threshold -> ...), with the -wg, -mask, -cs and
-o paths and two size mismatches, at one GPU and at TAUDEM_B200_GPUS=2 (rounds mode).  Stdout, with the timing numbers masked, is
compared to transcripts of the same runs, and every output file bit for bit to the host-grid call on the same arrays."""
import os
import re
import subprocess

import numpy as np
import pytest

from util import assert_bits, write_point_shapefile

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")

# (label, executable, arguments: "<x>" names the file x.tif of the work directory, "<shp>" the outlets)
RUNS = [
    ("pitremove", "pitremove", "-z <dem> -fel <fel>"),
    ("d8flowdir", "d8flowdir", "-fel <fel> -p <p> -sd8 <sd8>"),
    ("dinfflowdir", "dinfflowdir", "-fel <fel> -ang <ang> -slp <slp>"),
    ("aread8", "aread8", "-p <p> -ad8 <ad8> -wg <w>"),
    ("areadinf", "areadinf", "-ang <ang> -sca <sca>"),
    ("areadinf -o", "areadinf", "-ang <ang> -sca <scao> -o <shp>"),
    ("threshold", "threshold", "-ssa <ad8> -src <src> -thresh 50 -mask <fel>"),
    ("d8flowpathextremeup", "d8flowpathextremeup", "-p <p> -sa <sd8> -ssa <ssa>"),
    ("gridnet", "gridnet", "-p <p> -plen <plen> -tlen <tlen> -gord <gord> -mask <src> -thresh 1"),
    ("dinfdecayaccum", "dinfdecayaccum", "-ang <ang> -dm <dm> -dsca <dsca> -wg <w>"),
    ("dinfconclimaccum", "dinfconclimaccum", "-ang <ang> -dg <dg> -dm <dm> -q <w> -ctpt <ctpt> -csol 0.5"),
    ("dinftranslimaccum", "dinftranslimaccum", "-ang <ang> -tsup <w> -tc <tc> -cs <dm> -ctpt <tctpt> -tla <tla> -tdep <tdep>"),
    ("twi", "twi", "-slp <slp> -sca <sca> -twi <twi>"),
    ("slopearea", "slopearea", "-slp <slp> -sca <sca> -sa <sa>"),
    ("slopearearatio", "slopearearatio", "-slp <slp> -sca <sca> -sar <sar>"),
    ("peukerdouglas", "peukerdouglas", "-fel <fel> -ss <ss>"),
    ("lengtharea", "lengtharea", "-plen <plen> -ad8 <ad8> -ss <lass>"),
    ("slopeavedown", "slopeavedown", "-p <p> -fel <fel> -slpd <slpd>"),
    ("flowdircond", "flowdircond", "-p <p> -z <dem> -zfdc <zfdc>"),
    ("retlimflow", "retlimflow", "-ang <ang> -wg <w> -rc <dm> -qrl <qrl>"),
    ("d8hdisttostrm", "d8hdisttostrm", "-p <p> -src <src> -dist <hdist>"),
    ("d8vdisttostrm", "d8vdisttostrm", "-p <p> -fel <fel> -src <src> -dist <vdist>"),
    ("aread8 size", "aread8", "-p <p> -ad8 <bad> -wg <w9>"),
    ("slopeavedown size", "slopeavedown", "-p <p9> -fel <fel> -slpd <bad>"),
]


def inputs(work, ny=160, nx=200):
    """The chain's first inputs and the outlet shapefile; returns the outlet cells (cols, rows)"""
    import taudem_b200 as td
    from taudem_b200 import synth
    td.write_raster(os.path.join(work, "dem.tif"), synth.gen_dem(ny, nx, hurst=0.8, tilt=1.0, seed=5), -9999.0)
    td.write_raster(os.path.join(work, "w.tif"), np.full((ny, nx), 1.5, np.float32), -1.0)
    td.write_raster(os.path.join(work, "dm.tif"), np.full((ny, nx), 0.75, np.float32), -1.0)
    td.write_raster(os.path.join(work, "tc.tif"), np.full((ny, nx), 20.0, np.float32), -1.0)
    td.write_raster(os.path.join(work, "dg.tif"), (np.arange(ny * nx).reshape(ny, nx) % 3 == 0).astype(np.int16), -1)
    td.write_raster(os.path.join(work, "w9.tif"), np.ones((ny, nx + 1), np.float32), -1.0)
    td.write_raster(os.path.join(work, "p9.tif"), np.ones((ny + 1, nx), np.int16), -32768)
    cols, rows = [nx // 2, nx // 3, 5], [ny // 2, ny - 4, ny // 4]
    write_point_shapefile(os.path.join(work, "outlets.shp"), [(c + 0.5) * 30.0 for c in cols], [30.0 * ny - (r + 0.5) * 30.0 for r in rows])
    return cols, rows


def run_chain(bindir, work, gpus):
    """Runs RUNS in order; returns {label: (exit status, stdout with <tmp> for the work directory and <t> for each time)}"""
    env = dict(os.environ)
    env["TAUDEM_B200_GPUS"] = str(gpus)
    env["TAUDEM_B200_PEER"] = "0"
    out = {}
    for label, exe, args in RUNS:
        argv = [os.path.join(work, a[1:-1] + ".tif") if a.startswith("<") else a for a in args.split()]
        argv = [os.path.join(work, "outlets.shp") if a.endswith("shp.tif") else a for a in argv]
        r = subprocess.run([os.path.join(bindir, exe), *argv], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
        out[label] = (r.returncode, re.sub(r"(time: )[0-9.e+-]+", r"\1<t>", r.stdout.replace(work, "<tmp>")))
    return out


@pytest.fixture(scope="module")
def chain(tmp_path_factory):
    runs = {}
    for gpus in (1, 2):
        work = str(tmp_path_factory.mktemp(f"gpus{gpus}"))
        cells = inputs(work)
        runs[gpus] = (work, run_chain(BIN, work, gpus), cells)
    return runs


@pytest.mark.parametrize("gpus", [1, 2])
def test_transcripts(chain, gpus):
    _, got, _ = chain[gpus]
    for label, _, _ in RUNS:
        assert got[label] == EXPECTED[gpus][label], f"{label}: {got[label][1]}"


@pytest.mark.parametrize("gpus", [1, 2])
def test_outputs_match_the_grid_calls(chain, gpus):
    import taudem_b200 as td
    work, _, (cols, rows) = chain[gpus]
    f = lambda name: os.path.join(work, name + ".tif")
    rd = lambda name, dt=np.float32: td.read_raster(f(name), dt)
    nd = lambda name: td.raster_info(f(name))["nodata"]
    dem, w, dm, tc, dg = rd("dem"), rd("w"), rd("dm"), rd("tc"), rd("dg", np.int16)
    fel, p, ang, sd8, slp = rd("fel"), rd("p", np.int16), rd("ang"), rd("sd8"), rd("slp")
    ad8, sca, src, plen = rd("ad8"), rd("sca"), rd("src", np.int16), rd("plen")
    fnd, pnd, and_ = nd("fel"), int(nd("p")), nd("ang")
    want = {"fel": td.pitremove_grid(dem, -9999.0)}
    want["p"], want["sd8"] = td.d8flowdir_grid(fel, fnd)
    want["ang"], want["slp"] = td.dinfflowdir_grid(fel, fnd)
    want["ad8"] = td.aread8_grid(p, pnd, weights=w, w_nodata=-1.0)
    want["sca"] = td.areadinf_grid(ang, and_)
    want["scao"] = td.areadinf_grid(ang, and_, outlets=(cols, rows))
    want["src"] = td.threshold_grid(ad8, 50.0, mask=fel, nodata=nd("ad8"))
    want["ssa"] = td.d8flowpathextremeup_grid(p, sd8, nodata=pnd)
    want["plen"], want["tlen"], want["gord"] = td.gridnet_grid(p, mask=src.astype(np.int32), thresh=1, nodata=pnd)
    want["dsca"] = td.dinfdecayaccum_grid(ang, dm, weights=w, nodata=and_, dm_nodata=-1.0)
    want["ctpt"] = td.dinfconclimaccum_grid(ang, dm, w, dg, csol=0.5, nodata=and_, dm_nodata=-1.0, q_nodata=-1.0)
    want["tla"], want["tdep"], want["tctpt"] = td.dinftranslimaccum_grid(ang, w, tc, cs=dm, nodata=and_, tsup_nodata=-1.0, tc_nodata=-1.0, cs_nodata=-1.0)
    want["twi"] = td.twi_grid(slp, sca, nd("slp"), nd("sca"))
    want["sa"] = td.slopearea_grid(slp, sca)
    want["sar"] = td.slopearearatio_grid(slp, sca, nd("sca"))
    want["ss"] = td.peukerdouglas_grid(fel, nodata=fnd)
    want["lass"] = td.lengtharea_grid(plen, rd("ad8", np.int32))
    want["slpd"] = td.slopeavedown_grid(fel, p, nodata=fnd, p_nodata=pnd)
    want["zfdc"] = td.flowdircond_grid(p, dem, p_nodata=pnd, nodata=-9999.0)
    want["qrl"] = td.retlimflow_grid(ang, w, dm, ang_nodata=and_, wg_nodata=-1.0, rc_nodata=-1.0)
    want["hdist"] = td.d8hdisttostrm_grid(p, src.astype(np.int32), 1, p_nodata=pnd, src_nodata=int(nd("src")))
    want["vdist"] = td.d8vdisttostrm_grid(p, fel, src.astype(np.int32), 1, p_nodata=pnd, src_nodata=int(nd("src")))
    for name, a in want.items():
        assert_bits(rd(name, a.dtype), a, f"{name} at {gpus} GPU(s)")
    assert not os.path.exists(f("bad"))


EXPECTED = {
    1: {
        'pitremove': (0, 'PitRemove version 5.4.0-b200\nInput file <tmp>/dem.tif has projected coordinate system.\nNodata value input to create partition from file: -9999.000000\nNodata value recast to float used in partition raster: -9999.000000\nProcesses: 1\nHeader read time: <t>\nData read time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'd8flowdir': (0, 'D8FlowDir version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 1\nHeader read time: <t>\nData read time: <t>\nCompute Slope time: <t>\nWrite Slope time: <t>\nResolve Flat time: <t>\nWrite Flat time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'dinfflowdir': (0, 'DinfFlowDir version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 1\nHeader read time: <t>\nData read time: <t>\nCompute Slope time: <t>\nWrite Slope time: <t>\nResolve Flat time: <t>\nWrite Flat time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'aread8': (0, 'AreaD8 version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nNumber of Processes: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'areadinf': (0, 'AreaDinf version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'areadinf -o': (0, 'AreaDinf version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'threshold': (0, 'Threshold version 5.4.0-b200\nInput file <tmp>/ad8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'd8flowpathextremeup': (0, 'D8FlowPathExtremeUp version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/sd8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'gridnet': (0, 'GridNet version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'dinfdecayaccum': (0, 'DinfDecayAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'dinfconclimaccum': (0, 'DinfConcLimAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dg.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to int16_t used in partition raster: -1.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'dinftranslimaccum': (0, 'DinfTransLimAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/tc.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'twi': (0, 'Topographic Wetness Index version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopearea': (0, 'SlopeArea version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopearearatio': (0, 'SlopeAreaRatio version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'peukerdouglas': (0, 'PeukerDouglas version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'lengtharea': (0, 'LengthArea version 5.4.0-b200\nInput file <tmp>/plen.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/ad8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to int32_t used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopeavedown': (0, 'SlopeAveDown version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'flowdircond': (0, 'FlowDirCond version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/dem.tif has projected coordinate system.\nNodata value input to create partition from file: -9999.000000\nNodata value recast to float used in partition raster: -9999.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'retlimflow': (0, 'Retention limited flow accumulation version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'd8hdisttostrm': (0, 'D8HDistToStrm version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'd8vdisttostrm': (0, 'D8VDistToStrm version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'aread8 size': (0, 'AreaD8 version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/w9.tif has projected coordinate system.\nColumns do not match: 200 201\nFile sizes do not match\n<tmp>/w9.tif\narea error 5\n'),
        'slopeavedown size': (0, 'SlopeAveDown version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/p9.tif has projected coordinate system.\nRows do not match: 160 161\nFile sizes do not match\n<tmp>/p9.tif\nsloped error 5\n'),
    },
    2: {
        'pitremove': (0, 'PitRemove version 5.4.0-b200\nInput file <tmp>/dem.tif has projected coordinate system.\nNodata value input to create partition from file: -9999.000000\nNodata value recast to float used in partition raster: -9999.000000\nProcesses: 2\nHeader read time: <t>\nData read time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 4\nFlat cells left: 0\n'),
        'd8flowdir': (0, 'D8FlowDir version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 2\nHeader read time: <t>\nData read time: <t>\nCompute Slope time: <t>\nWrite Slope time: <t>\nResolve Flat time: <t>\nWrite Flat time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 0\nFlat cells left: 0\n'),
        'dinfflowdir': (0, 'DinfFlowDir version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 2\nHeader read time: <t>\nData read time: <t>\nCompute Slope time: <t>\nWrite Slope time: <t>\nResolve Flat time: <t>\nWrite Flat time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 0\nFlat cells left: 0\n'),
        'aread8': (0, 'AreaD8 version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nNumber of Processes: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'areadinf': (0, 'AreaDinf version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'areadinf -o': (0, 'AreaDinf version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nProcessors: 1\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'threshold': (0, 'Threshold version 5.4.0-b200\nInput file <tmp>/ad8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'd8flowpathextremeup': (0, 'D8FlowPathExtremeUp version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/sd8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'gridnet': (0, 'GridNet version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 9\n'),
        'dinfdecayaccum': (0, 'DinfDecayAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'dinfconclimaccum': (0, 'DinfConcLimAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dg.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to int16_t used in partition raster: -1.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'dinftranslimaccum': (0, 'DinfTransLimAccum version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/tc.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'twi': (0, 'Topographic Wetness Index version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopearea': (0, 'SlopeArea version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopearearatio': (0, 'SlopeAreaRatio version 5.4.0-b200\nInput file <tmp>/slp.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/sca.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'peukerdouglas': (0, 'PeukerDouglas version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 1\n'),
        'lengtharea': (0, 'LengthArea version 5.4.0-b200\nInput file <tmp>/plen.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/ad8.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to int32_t used in partition raster: -1.000000\nCompute time: <t>\nRead time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\n'),
        'slopeavedown': (0, 'SlopeAveDown version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 5\n'),
        'flowdircond': (0, 'FlowDirCond version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/dem.tif has projected coordinate system.\nNodata value input to create partition from file: -9999.000000\nNodata value recast to float used in partition raster: -9999.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'retlimflow': (0, 'Retention limited flow accumulation version 5.4.0-b200\nInput file <tmp>/ang.tif has projected coordinate system.\nNodata value input to create partition from file: -340282346638528859811704183484516925440.000000\nNodata value recast to float used in partition raster: -340282346638528859811704183484516925440.000000\nInput file <tmp>/w.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nInput file <tmp>/dm.tif has projected coordinate system.\nNodata value input to create partition from file: -1.000000\nNodata value recast to float used in partition raster: -1.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 3\n'),
        'd8hdisttostrm': (0, 'D8HDistToStrm version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 4\n'),
        'd8vdisttostrm': (0, 'D8VDistToStrm version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/src.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int32_t used in partition raster: -32768.000000\nProcessors: 2\nRead time: <t>\nCompute time: <t>\nWrite time: <t>\nTotal time: <t>\nDevice compute time: <t>\nExchange rounds: 4\n'),
        'aread8 size': (0, 'AreaD8 version 5.4.0-b200\nInput file <tmp>/p.tif has projected coordinate system.\nNodata value input to create partition from file: -32768.000000\nNodata value recast to int16_t used in partition raster: -32768.000000\nInput file <tmp>/w9.tif has projected coordinate system.\nColumns do not match: 200 201\nFile sizes do not match\n<tmp>/w9.tif\narea error 5\n'),
        'slopeavedown size': (0, 'SlopeAveDown version 5.4.0-b200\nInput file <tmp>/fel.tif has projected coordinate system.\nNodata value input to create partition from file: -300000000549775575777803994281145270272.000000\nNodata value recast to float used in partition raster: -300000000549775575777803994281145270272.000000\nInput file <tmp>/p9.tif has projected coordinate system.\nRows do not match: 160 161\nFile sizes do not match\n<tmp>/p9.tif\nsloped error 5\n'),
    },
}
