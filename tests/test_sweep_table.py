"""Which algebra / grid combinations the contributing-area sweep (taudem_b200/csrc/sweep_warp.cu, td::wsweep_run) accepts: every
(D8 / D-infinity, weights, algebra) with every grid present, then every accepted combination with each of its grids missing in
turn.  A rejected call returns TD_ERR_ARG before it touches anything; an accepted one runs a whole sweep on the CPU emulator."""
import itertools

import pytest

import test_emu

TD_OK, TD_ERR_ARG = 0, 1
W, DM, DIST, EXTRA, DG, OUT2, CIN, OUT3 = 1, 2, 4, 8, 16, 32, 64, 128
GRIDS = {"w": W, "dm": DM, "dist": DIST, "extra": EXTRA, "extra.dg": DG, "extra.out2": OUT2, "extra.cin": CIN, "extra.out3": OUT3}

# (dinf, usew, alg) -> the grids the sweep rejects a call without.  Every combination not listed is rejected.
ACCEPTED = {
    (0, 0, 0): 0, (0, 1, 0): 0, (1, 0, 0): 0, (1, 1, 0): 0,                 # aread8 / areadinf, with and without weights
    (0, 1, 1): 0, (0, 1, 2): 0,                                             # d8flowpathextremeup: largest / smallest value upstream
    (1, 0, 3): DM, (1, 1, 3): DM,                                           # dinfdecayaccum
    (0, 0, 4): DIST, (0, 0, 5): DIST, (0, 0, 6): DIST,                      # gridnet (the mask `dm` is optional)
    (1, 1, 7): W | DM | EXTRA | DG,                                         # dinfconclimaccum
    (1, 1, 8): W | DM | EXTRA | OUT2,                                       # dinftranslimaccum
    (1, 1, 9): W | DM | EXTRA | OUT2 | CIN | OUT3,                          # dinftranslimaccum with a concentration
}


@pytest.fixture(scope="module")
def emu():
    import ctypes as C
    lib = test_emu._build()
    lib.emu_wsweep_call.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint]
    return lib


@pytest.mark.parametrize("dinf,usew", list(itertools.product((0, 1), (0, 1))))
def test_every_algebra_with_every_grid(emu, dinf, usew):
    for alg in range(-1, 11):
        want = TD_OK if (dinf, usew, alg) in ACCEPTED else TD_ERR_ARG
        assert emu.emu_wsweep_call(dinf, usew, alg, 0) == want, (dinf, usew, alg)


@pytest.mark.parametrize("combo", sorted(ACCEPTED), ids=lambda c: "dinf%d-usew%d-alg%d" % c)
def test_each_grid_missing(emu, combo):
    dinf, usew, alg = combo
    required = ACCEPTED[combo]
    for name, bit in GRIDS.items():
        if bit == W and usew and not required & W:
            continue                     # the weights of algebras 0-3 are the caller's promise: read, not checked
        want = TD_ERR_ARG if required & bit else TD_OK
        assert emu.emu_wsweep_call(dinf, usew, alg, bit) == want, (combo, name)
