"""ctypes binding of tests/align_check.c, the serial CPU statement of the alignments of approximate hits
(B200SA_APPROX_ALIGN) for large inputs.
Test infrastructure only.

The shared object is compiled on first use into a per-user temporary directory (keyed by the source's
hash), so the source tree stays read-only."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "align_check.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "suffix_align_check_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libalign_check_%s.so" % tag)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", tmp, _SRC])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, u64, ci = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int
        L.align_check.argtypes = [vp, u64, vp, u64, vp, vp, vp, vp, vp, u64, ci, ci, vp, vp]
        L.align_check.restype = u64
        _lib = L
    return _lib


def align_hits(text, starts, queries, hq, hp, hd, edit, iupac=False):
    """(counts u32[h], words u32[]) of hits (query index hq, position hp, distance | MINUS hd) on one host
    core.  starts = None: a single text."""
    t = np.ascontiguousarray(np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text,
                             dtype=np.uint8)
    s = np.zeros(0, np.uint32) if starts is None else np.ascontiguousarray(starts, dtype=np.uint32)
    qs = [bytes(x) for x in queries]
    blob = np.frombuffer(b"".join(qs) or b"\0", dtype=np.uint8)
    off = np.zeros(len(qs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in qs])
    hq, hp, hd = (np.ascontiguousarray(a, dtype=np.uint32) for a in (hq, hp, hd))
    cnt = np.zeros(max(len(hp), 1), dtype=np.uint32)
    args = (t.ctypes.data, len(t), s.ctypes.data if len(s) else None, len(s), blob.ctypes.data, off.ctypes.data,
            hq.ctypes.data, hp.ctypes.data, hd.ctypes.data, len(hp), int(edit), int(iupac), cnt.ctypes.data)
    total = lib().align_check(*args, None)
    if total == 2 ** 64 - 1:
        raise AssertionError("align_check: a walk's cost differs from its distance, or no memory")
    words = np.zeros(max(total, 1), dtype=np.uint32)
    lib().align_check(*args, words.ctypes.data)
    return cnt[:len(hp)], words[:total]
