"""ctypes binding of tests/fixed_check.c, the serial CPU statement of fixed symbols in IUPAC queries
(B200SA_APPROX_FIXED) for large inputs, for both metrics.
Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fixed_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_fixed_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libfixed_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        L.fixed_check.argtypes = [vp, u64, vp, u64, vp, vp, u64, u64, u32, ctypes.c_int, vp, vp, vp]
        L.fixed_check.restype = u64
        _lib = L
    return _lib


def fixed_blob(text, starts, blob, q_off, k, metric="hamming", q0=0, q1=None):
    """(offsets u64[q1 - q0 + 1], pos u32[], d u32[]) of queries [q0, q1) of the blob cut at q_off, on one host
    core; d is mis(p) over the free symbols, or dist(p) with metric="edit".  starts = None: a single text."""
    t = np.ascontiguousarray(np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text,
                             dtype=np.uint8)
    s = np.zeros(0, np.uint32) if starts is None else np.ascontiguousarray(starts, dtype=np.uint32)
    q = np.ascontiguousarray(blob, dtype=np.uint8)
    off = np.ascontiguousarray(q_off, dtype=np.uint64)
    q1 = len(off) - 1 if q1 is None else q1
    cnt = np.zeros(max(q1 - q0, 1), dtype=np.uint64)
    args = (t.ctypes.data, len(t), s.ctypes.data if len(s) else None, len(s), q.ctypes.data if len(q) else None,
            off.ctypes.data, q0, q1, int(k), int(metric == "edit"), cnt.ctypes.data)
    total = lib().fixed_check(*args, None, None)
    if total == 2 ** 64 - 1:
        raise MemoryError("fixed_check: no memory for a column of %d entries" % (max(np.diff(off)) + 2))
    pos = np.zeros(max(total, 1), dtype=np.uint32)
    d = np.zeros(max(total, 1), dtype=np.uint32)
    if total:
        lib().fixed_check(*args, pos.ctypes.data, d.ctypes.data)
    o = np.zeros(q1 - q0 + 1, dtype=np.uint64)
    o[1:] = np.cumsum(cnt[:q1 - q0])
    return o, pos[:total], d[:total]


def fixed(text, starts, queries, k, metric="hamming"):
    """fixed_blob over a list of queries."""
    qs = [bytes(x) for x in queries]
    off = np.zeros(len(qs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in qs])
    return fixed_blob(text, starts, np.frombuffer(b"".join(qs), dtype=np.uint8), off, k, metric)
