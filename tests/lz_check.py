"""ctypes binding of tests/lz_check.c, the serial CPU statement of the LPF and the LZ77 factorization for
large inputs, and its decoder.  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lz_check.c")
_lib = None
LITERAL = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_lz_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "liblz_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        L.lz_check.argtypes = [u64, vp, vp, vp, vp, vp, vp, vp, u64]
        L.lz_check.restype = ctypes.c_int64
        L.lz_decode.argtypes = [u64, u64, vp, vp, vp, vp, vp]
        L.lz_decode.restype = ctypes.c_int64
        _lib = L
    return _lib


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def lz(sa, lcp):
    """(lpf, src, start, length, source) on one host core."""
    sa, lcp = _u32(sa), _u32(lcp)
    n = len(sa)
    lpf, src = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    out = [np.zeros(n, np.uint32) for _ in range(3)]               # z <= n
    z = lib().lz_check(n, sa.ctypes.data, lcp.ctypes.data, lpf.ctypes.data, src.ctypes.data,
                       *(o.ctypes.data for o in out), n)
    assert z >= 0
    return (lpf, src) + tuple(o[:z].copy() for o in out)


def decode(text, start, length, source):
    """The text rebuilt from the factors, with the literals' bytes taken from `text`; raises on a malformed
    factor."""
    t = np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text
    start, length, source = _u32(start), _u32(length), _u32(source)
    lits = np.ascontiguousarray(t[start[source == LITERAL]], dtype=np.uint8)
    out = np.zeros(len(t), dtype=np.uint8)
    bad = lib().lz_decode(len(t), len(start), start.ctypes.data, length.ctypes.data, source.ctypes.data,
                          lits.ctypes.data if len(lits) else None, out.ctypes.data)
    if bad:
        raise ValueError("factor %d is malformed" % (bad - 1))
    return out
