"""The reference outputs of the stream-definition tests (peukerdouglas, lengtharea and the workflows around them), the way
tests/reference.py provides the other tools' outputs: tests/golden/stream_reference.json stores a digest of each output keyed by a
digest of the call; `RefPipeline` writes the input files and replays — peukerdouglas and lengtharea are recomputed by the numpy
restatements (tests/stream_restate.py), every other tool by reference.RefPipeline's restatements — and each result must match its
stored digest bit for bit.  TD_RECORD_REFERENCE=<file> with oracle/_ref built (make -C oracle ref && make -C oracle -f stream.mk)
runs the tools instead, requires the restatements to reproduce them, and writes the digests to <file> at exit (with
tests/reference.py's)."""
import json
import os

import numpy as np

import reference
import refrun
import stream_restate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_reference.json")
_stored = None


def stored():
    global _stored
    if _stored is None:
        with open(GOLDEN) as f:
            _stored = json.load(f)
    return _stored


def available():
    """the two reference executables are built (oracle/stream.mk)"""
    return all(os.access(os.path.join(refrun.REF, t), os.X_OK) for t in ("peukerdouglas", "lengtharea"))


class Files(refrun.RefPipeline):
    """refrun.RefPipeline with the two stream-definition tools: arrays in, arrays out, through a scratch directory"""

    def peukerdouglas(self, fel, weights=None, nodata=-3.0e38):
        """weights: (middle, side, diagonal) for -par, None = the tool's defaults"""
        self.put("felin.tif", fel, nodata)
        args = ["-fel", self.path("felin.tif"), "-ss", self.path("ss.tif")]
        if weights is not None:
            args += ["-par"] + [repr(float(w)) for w in weights]
        _, self.times["peukerdouglas"] = refrun.run_tool("peukerdouglas", args, self.np_ranks)
        return self.get("ss.tif", np.int16)

    def lengtharea(self, plen, ad8, m=None, y=None, nodata=-1.0):
        """plen and ad8 as gridnet and aread8 write them (float32, nodata -1); the tool reads ad8 as 32-bit integers"""
        self.put("plenin.tif", plen, nodata)
        self.put("ad8in.tif", np.asarray(ad8, np.float32), nodata)
        args = ["-plen", self.path("plenin.tif"), "-ad8", self.path("ad8in.tif"), "-ss", self.path("lass.tif")]
        if m is not None:
            args += ["-par", repr(float(m)), repr(float(y))]
        _, self.times["lengtharea"] = refrun.run_tool("lengtharea", args, self.np_ranks)
        return self.get("lass.tif", np.int16)


class RefPipeline(reference.RefPipeline):
    """reference.RefPipeline's calls plus peukerdouglas and lengtharea, replayed from tests/golden/stream_reference.json"""

    TOOLS = reference.RefPipeline.TOOLS + ("peukerdouglas", "lengtharea")

    def __init__(self, workdir=None, dx=30.0, dy=30.0, np_ranks=1):
        if reference.RECORD and not available():
            raise RuntimeError("TD_RECORD_REFERENCE needs oracle/_ref/peukerdouglas and lengtharea (make -C oracle -f stream.mk)")
        super().__init__(workdir=workdir, dx=dx, dy=dy, np_ranks=np_ranks)
        self.files = Files(workdir=self.dir, dx=dx, dy=dy, np_ranks=np_ranks)

    def _restate(self, tool, args, kw):
        kw = dict(kw)
        if tool == "peukerdouglas":
            if kw.get("weights") is None:
                kw.pop("weights", None)
            return stream_restate.peukerdouglas(*args, **kw)
        if tool == "lengtharea":
            kw.pop("nodata", None)                          # (plen < 0 decides, not plen's nodata)
            return stream_restate.lengtharea(*args, **kw)
        return super()._restate(tool, args, kw)

    def _call(self, tool, args, kw):
        key = reference.call_key(tool, self.dx, self.dy, self.np_ranks, args, kw)
        out = getattr(self.files, tool)(*args, **kw)          # writes the input files (and runs the tool when recording)
        many = isinstance(out, tuple)
        if reference.RECORD:
            reference._recorded[key] = [None if o is None else reference.digest(o) for o in (out if many else (out,))]
            mine = self._restate(tool, args, kw)
            if [None if m is None else reference.digest(m) for m in (mine if many else (mine,))] != reference._recorded[key]:
                raise AssertionError(f"{tool}: the restatement does not reproduce the reference's output")
            return out
        want = stored().get(key)
        if want is None:
            raise AssertionError(f"{tool}: no stored reference output for these inputs in {GOLDEN} "
                                 "(record it with TD_RECORD_REFERENCE=<file> where oracle/_ref is built)")
        mine = self._restate(tool, args, kw)
        res = mine if isinstance(mine, tuple) else (mine,)
        assert len(res) == len(want), f"{tool}: {len(res)} outputs, {len(want)} stored"
        for i, (r, h) in enumerate(zip(res, want)):
            assert (None if r is None else reference.digest(r)) == h, f"{tool}[{i}]: the restatement no longer reproduces the reference's output"
        reference.replayed[key] = tool
        return res if many else res[0]
