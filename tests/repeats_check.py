"""ctypes binding of tests/repeats_check.c, the serial CPU statement of the repeats for large inputs.
Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "repeats_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_repeats_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "librepeats_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        L.repeats_check_runs.argtypes = [u64, vp, vp, u32, vp, vp, vp, vp, u64]
        L.repeats_check_runs.restype = u64
        L.repeats_check_spans.argtypes = [u64, vp, vp, vp, u32, u32, ctypes.c_int, vp, vp, u64, ctypes.POINTER(u64)]
        L.repeats_check_spans.restype = ctypes.c_int64
        _lib = L
    return _lib


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def runs(sa, lcp, min_len):
    """(start, end, first, last) on one host core."""
    sa, lcp = _u32(sa), _u32(lcp)
    k = lib().repeats_check_runs(len(sa), sa.ctypes.data, lcp.ctypes.data, min_len, None, None, None, None, 0)
    out = [np.zeros(k, dtype=np.uint32) for _ in range(4)]
    lib().repeats_check_runs(len(sa), sa.ctypes.data, lcp.ctypes.data, min_len, *(o.ctypes.data for o in out), k)
    return tuple(out)


def spans(sa, lcp, starts, min_len, mode):
    """(begin, end, covered) on one host core.  starts = None: a single text."""
    sa, lcp = _u32(sa), _u32(lcp)
    s = None if starts is None else _u32(starts)
    sp, nd = (None, 0) if s is None else (s.ctypes.data, len(s))
    cov = ctypes.c_uint64(0)
    k = lib().repeats_check_spans(len(sa), sa.ctypes.data, lcp.ctypes.data, sp, nd, min_len, mode, None, None, 0,
                                  ctypes.byref(cov))
    assert k >= 0
    b, e = np.zeros(k, dtype=np.uint32), np.zeros(k, dtype=np.uint32)
    lib().repeats_check_spans(len(sa), sa.ctypes.data, lcp.ctypes.data, sp, nd, min_len, mode, b.ctypes.data,
                              e.ctypes.data, k, ctypes.byref(cov))
    return b, e, int(cov.value)
