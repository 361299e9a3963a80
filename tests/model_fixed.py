"""Host statements of fixed symbols in IUPAC queries (include/b200sa.h, B200SA_APPROX_FIXED), by brute force on
top of tests/model_iupac.py and tests/model_align.py: the Hamming window, the constrained edit DP giving dist(p),
the constrained canonical walk giving the BAM words, and the listing of a whole call for any mix of metric, best,
strands, documents and align.  A fixed symbol is a lowercase letter; rc(q) keeps the case of each symbol, so its
marks are q's reversed.  A single text is one document."""
import numpy as np

from tests import model_align, model_approx, model_approx_docs, model_best, model_docs, model_iupac, model_strand

I, D, EQ, X = model_align.I, model_align.D, model_align.EQ, model_align.X
MINUS = model_strand.MINUS
BIG = 1 << 40                                 # an infinite distance


def marks(q):
    """bool[m]: the fixed symbols, the lowercase bytes."""
    return np.array([0x61 <= b <= 0x7A for b in bytes(q)], dtype=bool)


def window(win, cls, fx):
    """mis(p) over the free symbols of one window, or None when a fixed symbol misses."""
    miss = [t not in c for t, c in zip(win, cls)]
    if any(a and f for a, f in zip(miss, fx)):
        return None
    return sum(miss)


def full_dp(mis, fx):
    """D[x, t - p] for 0 <= x <= m, p <= t <= E under the three rules (BIG where no alignment keeps them), from
    mis = model_align.mismatch(T[p, E), Q) and fx = marks(Q)."""
    m, L = mis.shape
    idx = np.arange(L + 1, dtype=np.int64)
    Dm = np.zeros((m + 1, L + 1), dtype=np.int64)
    for x in range(m - 1, -1, -1):
        y = np.full(L + 1, BIG, dtype=np.int64)
        if not fx[x]:
            y = np.minimum(y, Dm[x + 1] + 1)                             # I
        diag = Dm[x + 1, 1:] + mis[x]
        if fx[x]:
            diag = np.where(mis[x], BIG, diag)                           # no X on a fixed symbol
        y[:L] = np.minimum(y[:L], diag)
        if fx[x] or (x > 0 and fx[x - 1]):
            Dm[x] = np.minimum(y, BIG)                                   # no D next to a fixed symbol
        else:
            Dm[x] = np.minimum(np.minimum.accumulate((y + idx)[::-1])[::-1] - idx, BIG)
    return Dm


def dists(doc, q):
    """dist(p) of every p of one document (int64[len(doc)], BIG when infinite): row 0 of the DP from the
    document's start holds D(0, t) for every t."""
    return full_dp(model_align.mismatch(doc, q, True), marks(q))[0, :len(doc)]


def one_strand(docs, queries, k, metric="hamming"):
    """The call on one strand without best: (offsets, pos, d) of every p with d(p) <= k, by ascending p."""
    text, starts = model_docs.concat(docs)
    out = []
    for q in queries:
        cls, fx, hits = model_iupac.classes(q), marks(q), []
        if q:
            for s, e in zip(starts.tolist(), model_approx._ends(starts, len(text))):
                if metric == "hamming":
                    for p in range(s, e - len(q) + 1):
                        d = window(text[p:p + len(q)], cls, fx)
                        if d is not None and d <= k:
                            hits.append((p, d))
                elif e > s:
                    d = dists(text[s:e], q)
                    hits += [(s + int(p), int(d[p])) for p in np.flatnonzero(d <= k)]
        out.append(hits)
    return model_approx._pack(out)


def flagless(docs, queries, k, metric="hamming", best=None, strands="forward"):
    """L(q) of every query: the hit list of the call without B200SA_APPROX_DOCUMENTS and B200SA_APPROX_ALIGN,
    packed (offsets, pos, d | MINUS on a minus hit)."""
    plus = model_best.lists(one_strand(docs, queries, k, metric))
    if strands == "both":
        minus = model_best.lists(one_strand(docs, [model_strand.revcomp(q, True) for q in queries], k, metric))
    else:
        minus = [[] for _ in queries]
    out = []
    for hp, hm in zip(plus, minus):
        if best is not None:
            ds = [d for _, d in hp + hm]
            t = model_best.threshold(min(ds), k, best) if ds else -1
            hp, hm = [h for h in hp if h[1] <= t], [h for h in hm if h[1] <= t]
        out.append(sorted([(p, d) for p, d in hp] + [(p, d | MINUS) for p, d in hm],
                          key=lambda h: (h[0], h[1] >= MINUS)))
    return model_approx._pack(out)


def walk(mis, fx, Dm):
    """The constrained canonical walk from (0, p): the first allowed move that holds.  (moves, u, cells) with
    cells the (x, u) it visits."""
    m, L = mis.shape
    x = u = 0
    moves, cells = [], [(0, 0)]
    while x < m:
        v = int(Dm[x, u])
        if u < L and not (fx[x] and mis[x, u]) and v == Dm[x + 1, u + 1] + int(mis[x, u]):
            moves.append(X if mis[x, u] else EQ)
            x, u = x + 1, u + 1
        elif not fx[x] and v == Dm[x + 1, u] + 1:
            moves.append(I)
            x += 1
        else:
            assert not fx[x] and not (x > 0 and fx[x - 1]) and v == Dm[x, u + 1] + 1
            moves.append(D)
            u += 1
        cells.append((x, u))
    return moves, u, cells


def align(text, E, p, q, d, metric="hamming", minus=False):
    """(ops [(code, len)], end) of the hit (p, d) of q (rc(q) on a minus hit) in text whose document ends at E."""
    Q = model_align.symbols(q, True, minus)
    m, fx = len(Q), marks(Q)
    if metric == "hamming":
        mis = model_align.mismatch(text[p:p + m], Q, True)
        assert not any(mis[x, x] and fx[x] for x in range(m))
        return model_align.merge([X if mis[x, x] else EQ for x in range(m)]), p + m
    mis = model_align.mismatch(text[p:E], Q, True)
    Dm = full_dp(mis, fx)
    assert Dm[0, 0] == d, (Dm[0, 0], d)
    moves, u, _ = walk(mis, fx, Dm)
    return model_align.merge(moves), p + u


def listing(docs, queries, k, metric="hamming", best=None, strands="forward", documents=False, align_ops=False):
    """(offsets, pos, d) of the call with B200SA_APPROX_FIXED | B200SA_APPROX_IUPAC and the given mix: the hits,
    the document listing (documents=True) or the alignment operations (align_ops=True)."""
    packed = flagless(docs, queries, k, metric, best, strands)
    starts = model_approx_docs.starts_of(docs)
    if documents:
        return model_approx._pack(model_approx_docs.reduce_lists(packed, starts))
    if not align_ops:
        return packed
    off, pos, dist = packed
    text = b"".join(bytes(x) for x in docs)
    ends = model_approx._ends(starts, len(text)) if len(starts) else []
    out = []
    for qi, q in enumerate(queries):
        ent = []
        for i in range(int(off[qi]), int(off[qi + 1])):
            p, dd = int(pos[i]), int(dist[i])
            minus, dd = dd >= MINUS, dd & (MINUS - 1)
            E = ends[model_approx_docs.doc_of(starts, p)]
            ops, _ = align(text, E, p, q, dd, metric, minus)
            ent += [(p, w) for w in model_align.words(ops, minus)]
        out.append(ent)
    return model_approx._pack(out)
