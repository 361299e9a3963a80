"""Host statements of IUPAC queries in approximate positions (include/b200sa.h, B200SA_APPROX_IUPAC): (a) the
definition by brute force, mis(p) and dist(p) with "T[p + x] != q[x]" read as "T[p + x] is not in the class of
q[x]", and (b) the device's rule in Python -- the stretch pieces, their table ranges, the candidates and the
reporters of f-14 and f-15 over the per-slot pieces -- over G from model_docs.brute.  A single text is one
document."""
import itertools

import numpy as np

from tests import model_approx, model_docs

_pack, _ends = model_approx._pack, model_approx._ends

CLASSES = {
    "A": b"A", "C": b"C", "G": b"G", "T": b"T", "U": b"T",
    "R": b"AG", "Y": b"CT", "S": b"CG", "W": b"AT", "K": b"GT", "M": b"AC",
    "B": b"CGT", "D": b"AGT", "H": b"ACT", "V": b"ACG", "N": b"ACGT",
}
CONCRETE = set(b"ACGTUacgtu")


def classes(q):
    """The class of each query byte (a frozenset of text bytes); ValueError for a byte that is no IUPAC code."""
    out = []
    for x, b in enumerate(q):
        c = CLASSES.get(chr(b).upper()) if b < 128 else None
        if c is None:
            raise ValueError("byte 0x%02x at offset %d is not an IUPAC code" % (b, x))
        out.append(frozenset(c))
    return out


def expansions(q):
    """Every concrete uppercase query the IUPAC query q stands for."""
    return [bytes(t) for t in itertools.product(*[sorted(c) for c in classes(q)])]


def mis(window, cls):
    return sum(t not in c for t, c in zip(window, cls))


def dists(doc, cls):
    """dist(p) of every p of one document (int64[len(doc)]), model_edit.dists with the class test."""
    L, m = len(doc), len(cls)
    t = np.frombuffer(doc, dtype=np.uint8).astype(np.int64)
    idx = np.arange(L + 1, dtype=np.int64)
    row = np.zeros(L + 1, dtype=np.int64)
    for x in range(m - 1, -1, -1):
        y = row + 1                                              # delete q[x]
        y[:L] = np.minimum(y[:L], row[1:] + ~np.isin(t, list(cls[x])))
        row = np.minimum.accumulate((y + idx)[::-1])[::-1] - idx
    return row[:L]


def brute(docs, queries, k, metric="hamming"):
    """(offsets, pos, d) of every p with d(p) <= k, by ascending p: mis(p) over windows inside one document, or
    dist(p) with metric="edit"."""
    text, starts = model_docs.concat(docs)
    out = []
    for q in queries:
        cls, hits = classes(q), []
        if q:
            for s, e in zip(starts.tolist(), _ends(starts, len(text))):
                if metric == "hamming":
                    for p in range(s, e - len(q) + 1):
                        d = mis(text[p:p + len(q)], cls)
                        if d <= k:
                            hits.append((p, d))
                elif e > s:
                    d = dists(text[s:e], cls)
                    hits += [(s + int(p), int(d[p])) for p in np.flatnonzero(d <= k)]
        out.append(hits)
    return _pack(out)


def stretches(q):
    """[(start, length)] of the maximal runs of concrete symbols (A C G T U, either case)."""
    out, x = [], 0
    while x < len(q):
        if q[x] in CONCRETE:
            y = x
            while y < len(q) and q[y] in CONCRETE:
                y += 1
            out.append((x, y - x))
            x = y
        else:
            x += 1
    return out


def piece_length(q, k):
    """t, the largest length with sum floor(L_i / t) >= k + 1, or None when sum L_i < k + 1 (whole table)."""
    P, ls = k + 1, [L for _, L in stretches(q)]
    if sum(ls) < P:
        return None
    return max(t for t in range(1, sum(ls) // P + 1) if sum(L // t for L in ls) >= P)


def pieces(q, k):
    """The k + 1 pieces [(offset, length)] of q, or None for the whole-table slot."""
    t = piece_length(q, k)
    if t is None:
        return None
    P, out = k + 1, []
    for x, L in stretches(q):
        c = min(L // t, P - len(out))
        out += [(x + j * L // c, (j + 1) * L // c - j * L // c) for j in range(c)]
    assert len(out) == P
    return out


def canon(q):
    """The canonical copy: the uppercase base of a concrete symbol, else the class (a different byte per class)."""
    return bytes(b"T"[0] if chr(b).upper() == "U" else ord(chr(b).upper()) for b in q)


def rule(docs, queries, k, metric="hamming"):
    """The device's rule: candidates from the table range of each piece (every rank for the whole-table slot),
    and per metric the reporter of f-14 (the first exactly matching piece) or f-15 (the least (piece, position)
    within k of its place).  Lists every report, so a repeat shows as a duplicate."""
    text, starts = model_docs.concat(docs)
    g, _ = model_docs.brute(docs)
    ends = _ends(starts, len(text))
    out = []
    for q in queries:
        m, cls, cq, hits = len(q), classes(q), canon(q), []
        pcs = pieces(q, k) if m else []
        dcache = {}

        def doc(p):
            d = model_docs.doc_of(starts, p)
            return int(starts[d]), ends[d], d

        def dist(p):
            s, e, d = doc(p)
            if d not in dcache:
                dcache[d] = dists(text[s:e], cls)
            return int(dcache[d][p - s])

        def exact(o, L, x, ds, de):                            # piece (o, L) at x, inside [ds, de)
            return ds <= x and x + L <= de and text[x:x + L] == cq[o:o + L]

        if m and pcs is None:                                   # the whole-table slot
            for s in (int(r) for r in g):
                if metric == "hamming":
                    ds, de, _ = doc(s)
                    if s + m <= de and mis(text[s:s + m], cls) <= k:
                        hits.append((s, mis(text[s:s + m], cls)))
                elif dist(s) <= k:
                    hits.append((s, dist(s)))
        elif m:
            for j, (o, L) in enumerate(pcs):
                lo, hi = model_approx.table_range(text, starts, g, cq[o:o + L])
                for s in (int(r) for r in g[lo:hi]):
                    ds, de, _ = doc(s)
                    if metric == "hamming":
                        p = s - o
                        if p < ds or p + m > de or mis(text[p:p + m], cls) > k:
                            continue
                        if any(exact(oi, Li, p + oi, ds, de) for oi, Li in pcs[:j]):
                            continue
                        hits.append((p, mis(text[p:p + m], cls)))
                    else:
                        for p in range(max(ds, s - o - k), min(de - 1, s - o + k) + 1):
                            if dist(p) > k:
                                continue
                            if any(exact(oi, Li, p + oi + d, ds, de) for oi, Li in pcs[:j]
                                   for d in range(-k, k + 1)):
                                continue
                            if any(exact(o, L, x, ds, de) for x in range(p + o - k, s)):
                                continue
                            hits.append((p, dist(p)))
        out.append(sorted(hits))
    return _pack(out)
