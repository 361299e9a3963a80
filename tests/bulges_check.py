"""ctypes binding of tests/bulges_check.c, the serial CPU statement of separate budgets for substitutions, DNA
bulges and RNA bulges (B200SA_APPROX_BULGES) for large inputs, with or without IUPAC codes and fixed symbols.
Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bulges_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_bulges_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libbulges_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        i32 = ctypes.c_int
        L.bulges_check.argtypes = [vp, u64, vp, u64, vp, vp, u64, u64, u32, u32, u32, i32, i32, vp, vp, vp]
        L.bulges_check.restype = u64
        _lib = L
    return _lib


def bulges_blob(text, starts, blob, q_off, t, d, r, iupac=False, fixed=False, q0=0, q1=None):
    """(offsets u64[q1 - q0 + 1], pos u32[], dist u32[]) of queries [q0, q1) of the blob cut at q_off, on one host
    core.  starts = None: a single text."""
    tx = np.ascontiguousarray(np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text,
                              dtype=np.uint8)
    s = np.zeros(0, np.uint32) if starts is None else np.ascontiguousarray(starts, dtype=np.uint32)
    q = np.ascontiguousarray(blob, dtype=np.uint8)
    off = np.ascontiguousarray(q_off, dtype=np.uint64)
    q1 = len(off) - 1 if q1 is None else q1
    cnt = np.zeros(max(q1 - q0, 1), dtype=np.uint64)
    args = (tx.ctypes.data, len(tx), s.ctypes.data if len(s) else None, len(s), q.ctypes.data if len(q) else None,
            off.ctypes.data, q0, q1, int(t), int(d), int(r), int(iupac), int(fixed), cnt.ctypes.data)
    total = lib().bulges_check(*args, None, None)
    if total == 2 ** 64 - 1:
        raise MemoryError("bulges_check: no memory for the rows of %d bytes" % max(np.diff(off)))
    pos = np.zeros(max(total, 1), dtype=np.uint32)
    dd = np.zeros(max(total, 1), dtype=np.uint32)
    if total:
        lib().bulges_check(*args, pos.ctypes.data, dd.ctypes.data)
    o = np.zeros(q1 - q0 + 1, dtype=np.uint64)
    o[1:] = np.cumsum(cnt[:q1 - q0])
    return o, pos[:total], dd[:total]


def bulges(text, starts, queries, t, d, r, iupac=False, fixed=False):
    """bulges_blob over a list of queries."""
    qs = [bytes(x) for x in queries]
    off = np.zeros(len(qs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in qs])
    return bulges_blob(text, starts, np.frombuffer(b"".join(qs), dtype=np.uint8), off, t, d, r, iupac, fixed)
