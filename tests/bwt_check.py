"""ctypes binding of tests/bwt_check.c, the serial CPU statement of the Burrows-Wheeler transform of documents
for large inputs: the forward transform from SA / G and the inverse by the LF walk.  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bwt_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_bwt_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libbwt_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        L.bwt_forward.argtypes = [u64, vp, vp, vp, u32, vp, vp]
        L.bwt_forward.restype = ctypes.c_int64
        L.bwt_inverse.argtypes = [u64, u32, vp, vp, vp, vp]
        L.bwt_inverse.restype = ctypes.c_int
        _lib = L
    return _lib


def _u8(t):
    return np.frombuffer(bytes(t), dtype=np.uint8) if not isinstance(t, np.ndarray) else np.ascontiguousarray(t, np.uint8)


def forward(text, g, starts=None):
    """(bwt bytes, term_rows u32[k], r) on one host core; starts None is a single text."""
    t = _u8(text)
    g = np.ascontiguousarray(g, dtype=np.uint32)
    st = np.zeros(1, np.uint32) if starts is None else np.ascontiguousarray(starts, dtype=np.uint32)
    n, k = len(t), len(st)
    bwt = np.zeros(max(n, 1), np.uint8)
    term = np.zeros(max(k, 1), np.uint32)
    r = lib().bwt_forward(n, t.ctypes.data, g.ctypes.data, st.ctypes.data, k, bwt.ctypes.data, term.ctypes.data)
    return bwt[:n].tobytes(), term[:k].copy(), int(r)


def inverse(bwt, term_rows):
    """(text bytes, starts u32[k]), or None when no documents have that transform."""
    b = _u8(bwt)
    t = np.ascontiguousarray(term_rows, dtype=np.uint32)
    n, k = len(b), len(t)
    text = np.zeros(max(n, 1), np.uint8)
    starts = np.zeros(max(k, 1), np.uint32)
    if lib().bwt_inverse(n, k, b.ctypes.data, t.ctypes.data, text.ctypes.data, starts.ctypes.data):
        return None
    return text[:n].tobytes(), starts[:k].copy()
