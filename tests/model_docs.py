"""Host statements of the separator-free generalized suffix array (include/b200sa.h,
b200sa_docs_build): the definition by brute force, and a numpy model of the device
formulation (suffix_b200/csrc/docs.cuh) on SA + LCP of the concatenation."""
import numpy as np


def concat(docs):
    docs = [bytes(d) for d in docs]
    starts = np.zeros(len(docs), dtype=np.uint32)
    pos = 0
    for k, d in enumerate(docs):
        starts[k] = pos
        pos += len(d)
    return b"".join(docs), starts


def doc_of(starts, p):
    """Last document starting at or before p (empty documents share their start with the next)."""
    return int(np.searchsorted(starts, p, side="right")) - 1


def brute(docs):
    """(G, glcp) by definition: positions sorted by (T_p, d), LCPs by direct compare."""
    text, starts = concat(docs)
    n = len(text)
    ends = list(starts[1:]) + [n]
    d = [doc_of(starts, p) for p in range(n)]
    suf = [text[p:int(ends[d[p]])] for p in range(n)]
    g = sorted(range(n), key=lambda p: (suf[p], d[p]))
    lcp = [0] * n
    for i in range(1, n):
        a, b = suf[g[i - 1]], suf[g[i]]
        k = 0
        while k < len(a) and k < len(b) and a[k] == b[k]:
            k += 1
        lcp[i] = k
    return np.asarray(g, dtype=np.uint32), np.asarray(lcp, dtype=np.uint32)


def model(docs, sa, lcp):
    """Steps 2-5 of the device formulation, given SA and LCP of the concatenation.
    Returns (G, glcp, |A|)."""
    text, starts = concat(docs)
    n = len(text)
    if n == 0:
        return np.zeros(0, np.uint32), np.zeros(0, np.uint32), 0
    sa = np.asarray(sa, dtype=np.int64)
    lcp = np.asarray(lcp, dtype=np.int64)
    ends = np.append(starts[1:], n).astype(np.int64)
    dsa = np.searchsorted(starts, sa, side="right") - 1          # document of each rank
    rem = ends[dsa] - sa                                          # r per rank
    in_a = lcp >= rem                                             # rank 0: lcp 0 < r
    pre = np.concatenate([[0], np.cumsum(in_a)[:-1]])             # #A before each rank
    ulist = np.nonzero(~in_a)[0]
    alist = np.nonzero(in_a)[0]
    # lo: largest j < i with lcp[j] < r (the per-rank-threshold ANSV)
    lo = np.empty(len(alist), dtype=np.int64)
    for k, i in enumerate(alist):
        j = i - 1
        while lcp[j] >= rem[i]:
            j -= 1
        lo[k] = j
    order = sorted(range(len(alist)), key=lambda k: (lo[k], rem[alist[k]], dsa[alist[k]]))
    gr = np.full(n, -1, dtype=np.int64)
    glo = np.full(n, -1, dtype=np.int64)
    for k, o in enumerate(order):
        i, l = alist[o], lo[o]
        u_first = lcp[l] < rem[l] and (rem[l], sa[l]) < (rem[i], sa[i])
        s = k + (l - pre[l]) + (1 if u_first else 0)
        assert gr[s] == -1
        gr[s], glo[s] = i, l
    free = np.nonzero(gr < 0)[0]
    assert len(free) == len(ulist)
    gr[free] = ulist
    glo[free] = ulist
    g = sa[gr]
    glcp = np.zeros(n, dtype=np.int64)
    for s in range(1, n):
        x, y = gr[s], gr[s - 1]
        v = min(rem[x], rem[y])
        if glo[s] != glo[s - 1]:
            assert glo[s - 1] < glo[s]
            v = min(v, int(lcp[glo[s - 1] + 1:glo[s] + 1].min()))
        glcp[s] = v
    return g.astype(np.uint32), glcp.astype(np.uint32), len(alist)


def random_docs(rng, alphabets=(b"a", b"ab", b"abc", b"ACGT", b"\x00\xff")):
    """A small random document set: empty, duplicated and prefix-of-each-other documents included."""
    alpha = alphabets[int(rng.integers(0, len(alphabets)))]
    k = int(rng.integers(1, 7))
    docs = []
    for _ in range(k):
        r = rng.random()
        if docs and r < 0.2:
            docs.append(docs[int(rng.integers(0, len(docs)))])                 # duplicate
        elif docs and r < 0.35:
            src = docs[int(rng.integers(0, len(docs)))]
            docs.append(src[:int(rng.integers(0, len(src) + 1))])              # prefix of another
        elif r < 0.45:
            docs.append(b"")
        else:
            m = int(rng.integers(1, 9))
            docs.append(bytes(alpha[int(c)] for c in rng.integers(0, len(alpha), m)))
    return docs
