"""Suffix array of a uint32 string by prefix doubling in numpy: the reference for the device's
reduced-string sort (b200sa_test_reduced_sa) at sizes where a brute-force sort is too slow.

Round h orders the suffixes by (rank[i], rank[i+h]), where rank is the order by the first h
symbols and 0 stands past the end (a proper prefix sorts first).  O(m log^2 m)."""
import numpy as np


def u32_sa(R) -> np.ndarray:
    R = np.asarray(R, dtype=np.uint32)
    m = len(R)
    if m == 0:
        return np.zeros(0, dtype=np.uint32)
    rank = R.astype(np.int64) + 1                   # 0 = past the end
    h = 1
    while True:
        nxt = np.zeros(m, dtype=np.int64)
        if h < m:
            nxt[: m - h] = rank[h:]
        sa = np.lexsort((nxt, rank))                # primary key last
        a, b = rank[sa], nxt[sa]
        head = np.ones(m, dtype=np.int64)
        head[1:] = (a[1:] != a[:-1]) | (b[1:] != b[:-1])
        rank = np.empty(m, dtype=np.int64)
        rank[sa] = np.cumsum(head)
        if rank[sa[-1]] == m:                       # every suffix has a rank of its own
            return sa.astype(np.uint32)
        h *= 2
