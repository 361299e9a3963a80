"""ctypes binding of tests/match_check.c, the serial CPU statement of matching statistics for large
inputs.  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "match_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_match_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libmatch_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        L.match_check.argtypes = [vp, u64, vp, u64, vp, vp, vp, u64, u64, u64, vp, vp, vp]
        L.match_check.restype = None
        _lib = L
    return _lib


def stats(text, starts, sa, queries_blob, q_off, x0=0, x1=None, ranges=True):
    """(len, start, end) of pattern positions [x0, x1) on one host core (start and end None without
    `ranges`).  starts = None: a single text."""
    t = np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text
    t = np.ascontiguousarray(t, dtype=np.uint8)
    sa = np.ascontiguousarray(sa, dtype=np.uint32)
    s = np.zeros(0, np.uint32) if starts is None else np.ascontiguousarray(starts, dtype=np.uint32)
    q = np.ascontiguousarray(queries_blob, dtype=np.uint8)
    off = np.ascontiguousarray(q_off, dtype=np.uint64)
    assert len(sa) == len(t) and int(off[-1]) == len(q)
    x1 = len(q) if x1 is None else x1
    ln = np.zeros(x1 - x0, dtype=np.uint32)
    st = np.zeros(x1 - x0, dtype=np.uint32) if ranges else None
    en = np.zeros(x1 - x0, dtype=np.uint32) if ranges else None
    lib().match_check(t.ctypes.data, len(t), s.ctypes.data if len(s) else None, len(s), sa.ctypes.data,
                      q.ctypes.data, off.ctypes.data, len(off) - 1, x0, x1, ln.ctypes.data,
                      st.ctypes.data if ranges else None, en.ctypes.data if ranges else None)
    return ln, st, en
