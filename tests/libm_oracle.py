"""The host libm and a correctly rounded float log / power over whole arrays (tests/libm_oracle.c, built here with the system C
compiler into the emulator's build directory and loaded with ctypes).  The oracle of the point-wise tests: the reference calls
glibc's logf / powf, the kernels compute the correctly rounded value, and the two differ exactly where libm is not correctly
rounded — which is counted on the machine the tests run on, never assumed."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
BUILD = os.path.join(HERE, "emu", "_build")
SRC = os.path.join(HERE, "libm_oracle.c")
FLT_POS_FINITE = 0x7F800000                       # bit patterns 0 .. 0x7f7fffff: +0 and every positive finite float

_lib = None


def lib():
    global _lib
    if _lib is None:
        os.makedirs(BUILD, exist_ok=True)
        so = os.path.join(BUILD, "liblibm_oracle.so")
        if not os.path.exists(so) or os.path.getmtime(SRC) > os.path.getmtime(so):
            tmp = f"{so}.{os.getpid()}"
            subprocess.check_call(["cc", "-O2", "-std=c11", "-D_GNU_SOURCE", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-fno-builtin",
                                   "-o", tmp, SRC, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        P, F, N, U = C.c_void_p, C.c_float, C.c_long, C.c_uint32
        for name, args in (("lo_logf", [P, P, N]), ("lo_powf", [P, F, P, N]), ("lo_log_cr", [P, P, N]), ("lo_pow_cr", [P, F, P, N]),
                           ("lo_slopearea", [P, P, F, F, P, N]), ("lo_lengtharea", [P, P, F, F, P, N])):
            getattr(L, name).argtypes = args
            getattr(L, name).restype = None
        L.lo_sweep.argtypes = [C.c_int, F, U, P, N, P, P, N]
        L.lo_sweep.restype = N
        L.lo_powf_unfaithful.argtypes = [F, U, N, P, N]
        L.lo_powf_unfaithful.restype = N
        L.lo_lengtharea_flips.argtypes = [F, F, U, N, P, P, N]
        L.lo_lengtharea_flips.restype = N
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def logf(x):
    x = _f32(x); out = np.empty_like(x); lib().lo_logf(x.ctypes.data, out.ctypes.data, x.size); return out


def powf(x, e):
    x = _f32(x); out = np.empty_like(x); lib().lo_powf(x.ctypes.data, np.float32(e), out.ctypes.data, x.size); return out


def log_cr(x):
    x = _f32(x); out = np.empty_like(x); lib().lo_log_cr(x.ctypes.data, out.ctypes.data, x.size); return out


def pow_cr(x, e):
    x = _f32(x); out = np.empty_like(x); lib().lo_pow_cr(x.ctypes.data, np.float32(e), out.ctypes.data, x.size); return out


def slopearea_product(slp, sca, m, n):
    """the reference's powf(slp, m) * powf(sca, n) in float, every cell"""
    slp, sca = _f32(slp), _f32(sca)
    out = np.empty_like(slp)
    lib().lo_slopearea(slp.ctypes.data, sca.ctypes.data, np.float32(m), np.float32(n), out.ctypes.data, slp.size)
    return out


def lengtharea(plen, ad8, m, y):
    """the reference's lengtharea cell by cell (ad8 already int32): 1 / 0 by (float)ad8 >= M * powf(plen, y), -32768 where plen < 0"""
    plen, ad8 = _f32(plen), np.ascontiguousarray(ad8, np.int32)
    out = np.empty(plen.shape, np.int16)
    lib().lo_lengtharea(plen.ctypes.data, ad8.ctypes.data, np.float32(m), np.float32(y), out.ctypes.data, plen.size)
    return out


def sweep(which, e, u0, gpu, cap=64):
    """x = the floats with bit patterns u0 .. u0 + len(gpu) - 1; which 0: gpu = log x, 1: gpu = x^e.  Returns (counts, bad):
    counts = (cells where gpu differs from libm, inputs where libm is not correctly rounded, cells where gpu is not correctly
    rounded, cells in exactly one of the first two sets); bad = the first cells of the last two kinds (bit patterns)."""
    gpu = _f32(gpu)
    cnt = np.zeros(4, np.int64)
    bad = np.zeros(cap, np.uint32)
    nbad = lib().lo_sweep(which, np.float32(e), u0, gpu.ctypes.data, gpu.size, cnt.ctypes.data, bad.ctypes.data, cap)
    return tuple(int(c) for c in cnt), bad[:min(nbad, cap)]


def powf_unfaithful(e, u0=0, n=FLT_POS_FINITE, cap=64):
    """inputs of [u0, u0 + n) where libm's powf(x, e) is neither the correctly rounded power nor the float on the exact power's
    other side (as bit patterns, at most cap), and how many there are"""
    bad = np.zeros(cap, np.uint32)
    k = lib().lo_powf_unfaithful(np.float32(e), u0, n, bad.ctypes.data, cap)
    return k, bad[:min(k, cap)]


def lengtharea_flips(m, y, u0, n, cap):
    """(plen, ad8) pairs, plen = the floats with bit patterns u0 .. u0 + n - 1, whose decision (float)ad8 >= M * p differs between
    p = libm's powf and p = the correctly rounded power; sorted by plen, at most cap, and the number that exist"""
    plen = np.zeros(cap, np.float32)
    ad8 = np.zeros(cap, np.int32)
    k = lib().lo_lengtharea_flips(np.float32(m), np.float32(y), u0, n, plen.ctypes.data, ad8.ctypes.data, cap)
    plen, ad8 = plen[:min(k, cap)], ad8[:min(k, cap)]
    o = np.lexsort((ad8, plen))
    return plen[o], ad8[o], k
