"""Host statements of the repeats of a table (include/b200sa.h, b200sa_repeat_lens_dev,
b200sa_repeat_runs_dev, b200sa_duplicate_spans_dev): the definitions by brute force on the documents
themselves (no suffix array), and a numpy model of the device formulation
(suffix_b200/csrc/repeats.cuh) on the table and its LCP array."""
import numpy as np

from tests import model_docs

ANY, EARLIER, OTHER_DOC, EARLIER_DOC = 0, 1, 2, 3
MODES = (ANY, EARLIER, OTHER_DOC, EARLIER_DOC)


# ------------------------------------------------------------------ the definitions
def _layout(docs):
    text, starts = model_docs.concat(docs)
    n = len(text)
    doc = [model_docs.doc_of(starts, p) for p in range(n)]
    ends = [int(x) for x in starts[1:]] + [n]
    return text, starts, n, doc, ends


def brute_repeat_lens(docs):
    """rl[p]: the longest prefix of S_p that is a prefix of S_p' for some p' != p."""
    text, _, n, doc, ends = _layout(docs)
    suf = [text[p:ends[doc[p]]] for p in range(n)]
    rl = np.zeros(n, dtype=np.uint32)
    for p in range(n):
        for q in range(n):
            if q != p:
                k = 0
                while k < len(suf[p]) and k < len(suf[q]) and suf[p][k] == suf[q][k]:
                    k += 1
                rl[p] = max(rl[p], k)
    return rl


def brute_grams(docs, L):
    """{gram: ascending positions} of the grams of L bytes that lie inside one document."""
    text, _, n, doc, ends = _layout(docs)
    occ = {}
    for p in range(n):
        if p + L <= ends[doc[p]]:
            occ.setdefault(text[p:p + L], []).append(p)
    return occ


def brute_flags(docs, L):
    """{mode: bool[n]}: the flagged positions of every mode, from the grams' occurrence lists."""
    _, _, n, doc, _ = _layout(docs)
    flags = {m: np.zeros(n, dtype=bool) for m in MODES}
    for where in brute_grams(docs, L).values():
        for p in where:
            flags[ANY][p] = len(where) > 1
            flags[EARLIER][p] = any(q < p for q in where)
            flags[OTHER_DOC][p] = any(doc[q] != doc[p] for q in where)
            flags[EARLIER_DOC][p] = any(doc[q] < doc[p] for q in where)
    return flags


def spans_of_flags(docs, flagged, L):
    """(begin, end, covered) by a sweep over a byte mask."""
    _, starts, n, _, _ = _layout(docs)
    mask = [False] * n
    for p in np.nonzero(flagged)[0]:
        for x in range(int(p), min(int(p) + L, n)):
            mask[x] = True
    cut = {int(s) for s in starts}
    begin, end = [], []
    for x in range(n):
        if mask[x] and (x == 0 or not mask[x - 1] or x in cut):
            begin.append(x)
        if mask[x] and (x + 1 == n or not mask[x + 1] or x + 1 in cut):
            end.append(x + 1)
    return np.asarray(begin, dtype=np.uint32), np.asarray(end, dtype=np.uint32), sum(mask)


# ------------------------------------------------------------------ the device formulation
def _lam(lcp):
    return np.append(np.asarray(lcp, dtype=np.int64), 0)


def repeat_lens(g, lcp):
    lam = _lam(lcp)
    rl = np.zeros(len(g), dtype=np.uint32)
    rl[np.asarray(g, dtype=np.int64)] = np.maximum(lam[:-1], lam[1:])
    return rl


def _segments(g, lcp, L):
    """(seg, seg_first, seg_last): the head rank of every rank's segment and, at the head's slot, the
    smallest and largest position of the segment -- inclusive max scans of (seg << 32 | value) read at
    the segment's last rank."""
    n = len(g)
    lam = _lam(lcp)
    r = np.arange(n, dtype=np.int64)
    seg = np.maximum.accumulate(np.where(lam[:-1] < L, r + 1, 0)) - 1
    last_rank = lam[1:] < L
    out = []
    for value in ((~np.asarray(g, dtype=np.uint32)), np.asarray(g, dtype=np.uint32)):
        inc = np.maximum.accumulate((seg.astype(np.uint64) << np.uint64(32)) | value.astype(np.uint64))
        ext = np.zeros(n, dtype=np.uint32)
        ext[seg[last_rank]] = (inc[last_rank] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        out.append(ext)
    return seg, ~out[0], out[1]


def runs(g, lcp, L):
    """(start, end, first, last) of the runs at L."""
    lam = _lam(lcp)
    start = np.nonzero((lam[:-1] < L) & (lam[1:] >= L))[0]
    end = np.nonzero((lam[:-1] >= L) & (lam[1:] < L))[0] + 1
    _, sf, sl = _segments(g, lcp, L)
    return start.astype(np.uint32), end.astype(np.uint32), sf[start], sl[start]


def flags(g, lcp, starts, L, mode):
    """bool[n] in text order.  starts = None: a single text."""
    n = len(g)
    lam = _lam(lcp)
    g = np.asarray(g, dtype=np.int64)
    seg, sf, sl = _segments(g, lcp, L)
    f = (lam[:-1] >= L) | (lam[1:] >= L)
    if mode == EARLIER:
        f &= g != sf[seg]
    elif mode in (OTHER_DOC, EARLIER_DOC):
        st = np.asarray(starts, dtype=np.int64)
        d = np.searchsorted(st, g, side="right") - 1
        other = sf[seg] < st[d]
        if mode == OTHER_DOC:
            other |= sl[seg] >= np.append(st[1:], n)[d]
        f &= other
    out = np.zeros(n, dtype=bool)
    out[g[f]] = True
    return out


def spans(flagged, starts, L):
    """(begin, end, covered): a max scan of (flagged ? x + 1 : 0) gives the nearest flagged position at
    or before x; the cover, its begins and ends follow byte by byte."""
    n = len(flagged)
    x = np.arange(n, dtype=np.int64)
    near = np.maximum.accumulate(np.where(flagged, x + 1, 0)) if n else x
    cov = (near > 0) & (x - (near - 1) < L)
    cut = np.zeros(n + 1, dtype=bool)
    if starts is not None:
        cut[np.asarray(starts, dtype=np.int64)] = True
    cut[0] = cut[n] = True
    pad = np.concatenate([[False], cov, [False]])
    begin = np.nonzero(cov & (~pad[:-2] | cut[:-1]))[0]
    end = np.nonzero(cov & (~pad[2:] | cut[1:]))[0] + 1
    return begin.astype(np.uint32), end.astype(np.uint32), int(cov.sum())


def duplicate_spans(g, lcp, starts, L, mode):
    return spans(flags(g, lcp, starts, L, mode), starts, L)
