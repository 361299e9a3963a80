"""ctypes binding of tests/tree_oracle.c, the CPU restatement of the reference's
suffix tree construction (suffix_tree/src/lib.rs:392-505).  Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory
(keyed by the source's hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tree_oracle.c")
FIELDS = ("parent", "depth", "sa_lo", "sa_hi", "label_start", "subtree_end")
NONE = 0xFFFFFFFF
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_tree_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libtree_oracle_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared",
                                   "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64 = ctypes.c_void_p, ctypes.c_uint64
        L.oracle_suffix_tree.argtypes = [u64, vp, vp, u64] + [vp] * 9
        L.oracle_suffix_tree.restype = ctypes.c_int64
        L.oracle_tree_labels_differ.argtypes = [vp, u64, vp, vp, vp]
        L.oracle_tree_labels_differ.restype = ctypes.c_int64
        _lib = L
    return _lib


def suffix_tree(sa, lcp) -> dict:
    """The reference's tree of (table, lcp_lens) as the six canonical preorder arrays plus
    own_start / own_end (the reference's own label offsets) and terminal (NONE if none)."""
    sa = np.ascontiguousarray(sa, dtype=np.uint32)
    lcp = np.ascontiguousarray(lcp, dtype=np.uint32)
    n = len(sa)
    cap = 2 * n + 1
    names = FIELDS + ("own_start", "own_end", "terminal")
    out = {f: np.empty(cap, dtype=np.uint32) for f in names}
    N = lib().oracle_suffix_tree(n, sa.ctypes.data, lcp.ctypes.data, cap, *[out[f].ctypes.data for f in names])
    assert N > 0, "oracle_suffix_tree rejected its input (%d)" % N
    return {f: a[:N].copy() for f, a in out.items()}


def label_lengths(a: dict) -> np.ndarray:
    """len() of every node from the canonical arrays (0 at the root)."""
    p = a["parent"].astype(np.int64)
    d = a["depth"].astype(np.int64)
    out = np.zeros(len(p), dtype=np.uint32)
    out[1:] = d[1:] - d[p[1:]]
    return out


def labels_differ(text, starts_a, starts_b, lengths) -> int:
    """First node id >= 1 whose label bytes differ between two offset arrays, or -1."""
    t = np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text
    t = np.ascontiguousarray(t, dtype=np.uint8)
    a = np.ascontiguousarray(starts_a, dtype=np.uint32)
    b = np.ascontiguousarray(starts_b, dtype=np.uint32)
    ln = np.ascontiguousarray(lengths, dtype=np.uint32)
    return int(lib().oracle_tree_labels_differ(t.ctypes.data, len(ln), a.ctypes.data, b.ctypes.data, ln.ctypes.data))
