"""Host statements of approximate positions on both DNA strands (include/b200sa.h, B200SA_APPROX_BOTH_STRANDS):
the reverse complement of a query, plain or in IUPAC codes, and (a) the definition -- the plus hits of q and the
minus hits of rc(q) under the call's metric and IUPAC setting, with best(q) over both strands -- composed from
tests/model_approx.py, tests/model_edit.py, tests/model_iupac.py and tests/model_best.py, and (b) the device's
merge rule, which places each hit by its index in its own sublist plus its co-rank in the other.  A single text
is one document."""
import numpy as np

from tests import model_approx, model_best, model_edit, model_iupac

MINUS = 0x80000000                      # B200SA_APPROX_MINUS

PLAIN = {b"A"[0]: b"T"[0], b"T"[0]: b"A"[0], b"C"[0]: b"G"[0], b"G"[0]: b"C"[0]}
PLAIN.update({a | 0x20: b | 0x20 for a, b in list(PLAIN.items())})
IUPAC = dict(PLAIN)
for a, b in ("UA", "RY", "YR", "KM", "MK", "BV", "VB", "DH", "HD", "SS", "WW", "NN"):
    IUPAC[ord(a)], IUPAC[ord(a) | 0x20] = ord(b), ord(b) | 0x20


def comp(b, iupac=False):
    """The complement of one byte: A <-> T, C <-> G in either case and every other byte itself; with iupac the
    code whose class is the complemented class (U -> A, R <-> Y, K <-> M, B <-> V, D <-> H; S, W, N themselves)."""
    return (IUPAC if iupac else PLAIN).get(b, b)


def revcomp(q, iupac=False):
    """rc(q)[x] = comp(q[m - 1 - x])."""
    return bytes(comp(b, iupac) for b in reversed(bytes(q)))


def one_strand(docs, queries, k, metric="hamming", iupac=False):
    """The call without the flag: (offsets, pos, d)."""
    if iupac:
        return model_iupac.brute(docs, queries, k, metric)
    return model_approx.brute(docs, queries, k) if metric == "hamming" else model_edit.brute(docs, queries, k)


def merge(plus, minus):
    """The device's rule for one query: plus and minus are its two sublists [(p, d)] by ascending p.  A plus hit
    at index a goes to a + #{minus p' < p}, a minus hit at index b to b + #{plus p' <= p}; d of a minus hit gets
    MINUS."""
    pp = np.asarray([p for p, _ in plus], dtype=np.int64)
    mp = np.asarray([p for p, _ in minus], dtype=np.int64)
    out = [None] * (len(plus) + len(minus))
    for x, h in zip((np.arange(len(pp)) + np.searchsorted(mp, pp, side="left")).tolist(), plus):
        out[x] = h
    for x, (p, d) in zip((np.arange(len(mp)) + np.searchsorted(pp, mp, side="right")).tolist(), minus):
        out[x] = (p, d | MINUS)
    assert None not in out
    return out


def brute(docs, queries, k, metric="hamming", iupac=False, best=None):
    """(offsets, pos, d | MINUS on a minus hit) of both strands: q's list is its occurrences (p, +) and rc(q)'s
    (p, -) ordered by (p, strand) with + first.  best=s: best(q) the least d over both strands, both lists cut to
    d <= t(q) = min(k, best(q) + s)."""
    plus = model_best.lists(one_strand(docs, queries, k, metric, iupac))
    minus = model_best.lists(one_strand(docs, [revcomp(q, iupac) for q in queries], k, metric, iupac))
    out = []
    for hp, hm in zip(plus, minus):
        if best is not None:
            ds = [d for _, d in hp + hm]
            t = model_best.threshold(min(ds), k, best) if ds else -1
            hp, hm = [h for h in hp if h[1] <= t], [h for h in hm if h[1] <= t]
        out.append(sorted([(p, d) for p, d in hp] + [(p, d | MINUS) for p, d in hm],
                          key=lambda h: (h[0], h[1] >= MINUS)))
    return model_approx._pack(out)


def split(packed):
    """(offsets, pos, d, minus) of a packed both-strand result, as approximate_positions_batch returns it."""
    off, pos, d = packed
    d = np.asarray(d, dtype=np.uint32)
    return off, pos, d & np.uint32(MINUS - 1), (d & np.uint32(MINUS)) != 0


def strand_lists(packed):
    """Per-query (plus [(p, d)], minus [(p, d)]) of a packed both-strand result."""
    out = []
    for h in model_best.lists(packed):
        out.append(([(p, d) for p, d in h if d < MINUS], [(p, d - MINUS) for p, d in h if d >= MINUS]))
    return out
