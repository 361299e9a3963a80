"""Host statements of separate budgets for substitutions, DNA bulges and RNA bulges (include/b200sa.h,
B200SA_APPROX_BULGES), by brute force: for every start p, the layered DP over every end e <= E of p's document
(no band), the constrained canonical walk, and the listing of a whole call for any mix of IUPAC, FIXED, strands,
documents and align.  X is a substitution, I a query byte with no text byte (an RNA bulge), D a text byte with no
query byte (a DNA bulge).  A single text is one document."""
import numpy as np

from tests import model_align, model_approx, model_approx_docs, model_fixed, model_strand

I, D, EQ, X = model_align.I, model_align.D, model_align.EQ, model_align.X
MINUS = model_strand.MINUS
BIG = 1 << 20                                 # no alignment


def layered(mis, fx, d, r):
    """S[x, u, i, e] for 0 <= x <= m, 0 <= u <= L (int64): the least #X of an alignment of Q[x, m) to T[p + u,
    p + u') for some u' <= L, with at most i I and at most e D moves, BIG when there is none; mis =
    model_align.mismatch(T[p, p + L), Q), fx the fixed symbols (f-21: never X or I, no D at (x, u) when Q[x] or
    Q[x - 1] is fixed)."""
    m, L = mis.shape
    S = np.full((m + 1, L + 1, r + 1, d + 1), BIG, dtype=np.int64)
    S[m] = 0
    for x in range(m - 1, -1, -1):
        nodel = fx[x] or (x > 0 and fx[x - 1])
        for u in range(L, -1, -1):
            for i in range(r + 1):
                for e in range(d + 1):
                    y = BIG
                    if u < L and not (fx[x] and mis[x, u]):
                        y = min(y, S[x + 1, u + 1, i, e] + int(mis[x, u]))
                    if i > 0 and not fx[x]:
                        y = min(y, S[x + 1, u, i - 1, e])
                    if e > 0 and u < L and not nodel:
                        y = min(y, S[x, u + 1, i, e - 1])
                    S[x, u, i, e] = y
    return S


def feasible(S, x, u, iu, du, xu, C):
    """Some alignment of Q[x, m) from T[p + u] has <= iu I, <= du D, <= xu X and costs at most C."""
    if C < 0 or u >= S.shape[1]:
        return False
    return any(S[x, u, i, e] <= xu and S[x, u, i, e] + i + e <= C for i in range(iu + 1) for e in range(du + 1))


def dist_of(S, t, d, r):
    """dist(p) from S of p's window, or None when p is no occurrence."""
    c = [int(S[0, 0, i, e]) + i + e for i in range(r + 1) for e in range(d + 1) if S[0, 0, i, e] <= t]
    return min(c) if c else None


def _setup(text, E, p, Q, iupac, fixed, d):
    m = len(Q)
    L = min(E - p, m + d)                     # no alignment with at most d D moves spans more text
    mis = model_align.mismatch(text[p:p + L], Q, iupac)
    fx = model_fixed.marks(Q) if fixed else np.zeros(m, dtype=bool)
    return mis, fx


def dist(text, E, p, Q, t, d, r, iupac=False, fixed=False):
    """dist(p) of Q at p in text whose document ends at E, or None."""
    if not Q:
        return None
    mis, fx = _setup(text, E, p, Q, iupac, fixed, d)
    return dist_of(layered(mis, fx, d, r), t, d, r)


def align(text, E, p, Q, dd, t, d, r, iupac=False, fixed=False):
    """(ops [(code, len)], end) of the hit (p, dd): the walk from (0, 0) with budgets (r, d, t) and cost dd taking
    the first move, diagonal, I, D, that keeps some alignment within the budgets at the remaining cost."""
    mis, fx = _setup(text, E, p, Q, iupac, fixed, d)
    S = layered(mis, fx, d, r)
    m, L = mis.shape
    assert dist_of(S, t, d, r) == dd
    x = u = 0
    iu, du, xu, C = r, d, t, dd
    moves = []
    while x < m:
        nodel = fx[x] or (x > 0 and fx[x - 1])
        mi = int(mis[x, u]) if u < L else 1
        if u < L and not (fx[x] and mi) and mi <= xu and feasible(S, x + 1, u + 1, iu, du, xu - mi, C - mi):
            moves.append(X if mi else EQ)
            x, u, xu, C = x + 1, u + 1, xu - mi, C - mi
        elif not fx[x] and iu > 0 and feasible(S, x + 1, u, iu - 1, du, xu, C - 1):
            moves.append(I)
            x, iu, C = x + 1, iu - 1, C - 1
        else:
            assert not nodel and u < L and du > 0 and feasible(S, x, u + 1, iu, du - 1, xu, C - 1)
            moves.append(D)
            u, du, C = u + 1, du - 1, C - 1
    assert C == 0
    return model_align.merge(moves), p + u


def one_strand(docs, queries, t, d, r, iupac=False, fixed=False):
    """(offsets, pos, dist) of every occurrence by ascending p."""
    text = b"".join(bytes(x) for x in docs)
    starts = model_approx_docs.starts_of(docs)
    ends = model_approx._ends(starts, len(text)) if len(starts) else []
    out = []
    for Q in queries:
        hits = []
        for s, E in zip(starts.tolist(), ends):
            for p in range(s, E):
                dd = dist(text, E, p, Q, t, d, r, iupac, fixed)
                if dd is not None:
                    hits.append((p, dd))
        out.append(hits)
    return model_approx._pack(out)


def flagless(docs, queries, t, d, r, iupac=False, fixed=False, strands="forward"):
    """L(q) of every query: the hits, packed (offsets, pos, dist | MINUS on a minus hit), by (p, strand)."""
    from tests import model_best
    plus = model_best.lists(one_strand(docs, queries, t, d, r, iupac, fixed))
    if strands == "both":
        rcs = [model_strand.revcomp(q, iupac) for q in queries]
        minus = model_best.lists(one_strand(docs, rcs, t, d, r, iupac, fixed))
    else:
        minus = [[] for _ in queries]
    out = [sorted([(p, x) for p, x in hp] + [(p, x | MINUS) for p, x in hm], key=lambda h: (h[0], h[1] >= MINUS))
           for hp, hm in zip(plus, minus)]
    return model_approx._pack(out)


def listing(docs, queries, t, d, r, iupac=False, fixed=False, strands="forward", documents=False, align_ops=False):
    """(offsets, pos, d) of the call with B200SA_APPROX_BULGES | B200SA_APPROX_EDIT and the given mix: the hits,
    the document listing (documents=True) or the alignment operations (align_ops=True)."""
    packed = flagless(docs, queries, t, d, r, iupac, fixed, strands)
    starts = model_approx_docs.starts_of(docs)
    if documents:
        return model_approx._pack(model_approx_docs.reduce_lists(packed, starts))
    if not align_ops:
        return packed
    off, pos, dist_ = packed
    text = b"".join(bytes(x) for x in docs)
    ends = model_approx._ends(starts, len(text)) if len(starts) else []
    out = []
    for qi, q in enumerate(queries):
        ent = []
        for i in range(int(off[qi]), int(off[qi + 1])):
            p, dd = int(pos[i]), int(dist_[i])
            minus, dd = dd >= MINUS, dd & (MINUS - 1)
            E = ends[model_approx_docs.doc_of(starts, p)]
            ops, _ = align(text, E, p, model_align.symbols(q, iupac, minus), dd, t, d, r, iupac, fixed)
            ent += [(p, w) for w in model_align.words(ops, minus)]
        out.append(ent)
    return model_approx._pack(out)
