"""ctypes binding of tests/docs_tree_check.c, the serial construction of the generalized suffix tree
(b200sa_docs_tree) for large inputs.  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the
source's hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "docs_tree_check.c")
FIELDS = ("parent", "depth", "sa_lo", "sa_hi", "label_start", "subtree_end", "term_end", "doc_count")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_docs_tree_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libdocs_tree_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        L.docs_tree_check.argtypes = [u64, vp, vp, vp, u64, u64] + [vp] * 8
        L.docs_tree_check.restype = ctypes.c_int64
        _lib = L
    return _lib


def tree(g, glcp, starts) -> dict:
    """The eight arrays of the generalized suffix tree of (G, glcp, doc_starts), built serially."""
    g = np.ascontiguousarray(g, dtype=np.uint32)
    glcp = np.ascontiguousarray(glcp, dtype=np.uint32)
    s = np.ascontiguousarray(starts, dtype=np.uint32)
    n = len(g)
    cap = 2 * n + 1
    out = {f: np.empty(cap, dtype=np.uint32) for f in FIELDS}
    N = lib().docs_tree_check(n, g.ctypes.data, glcp.ctypes.data, s.ctypes.data, len(s), cap,
                              *[out[f].ctypes.data for f in FIELDS])
    assert N > 0, "docs_tree_check rejected its input (%d)" % N
    return {f: a[:N].copy() for f, a in out.items()}
