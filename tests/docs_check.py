"""ctypes binding of tests/docs_check.c, the CPU checker of a separator-free generalized
suffix array for large inputs.  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by
the source's hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "docs_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_docs_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libdocs_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        L.docs_check.argtypes = [vp, u64, vp, u64, vp, vp]
        L.docs_check.restype = ctypes.c_int64
        _lib = L
    return _lib


def check(text, starts, g, glcp=None) -> int:
    """0 if g (and glcp) are the generalized suffix array (and its LCP) of the documents of
    `text` cut at `starts`; otherwise -1 - i for the first bad rank i, or a large negative
    number when g is not a permutation."""
    t = np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text
    t = np.ascontiguousarray(t, dtype=np.uint8)
    s = np.ascontiguousarray(starts, dtype=np.uint32)
    g = np.ascontiguousarray(g, dtype=np.uint32)
    assert len(g) == len(t)
    lp = None
    if glcp is not None:
        glcp = np.ascontiguousarray(glcp, dtype=np.uint32)
        assert len(glcp) == len(t)
        lp = glcp.ctypes.data
    return int(lib().docs_check(t.ctypes.data, len(t), s.ctypes.data, len(s), g.ctypes.data, lp))
