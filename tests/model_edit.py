"""Host statements of the edit metric of approximate positions (include/b200sa.h, B200SA_APPROX_EDIT): (a) the
definition, dist(p) = min over e <= end(p) of ED(q, T[p, e)), literally per (p, e) and by the classical reversed
Sellers recurrence over a whole document, and (b) the device's rule in numpy -- pieces, their table ranges,
windows of starts around every candidate, the band of 4k + 1 diagonals, and the least (piece, position) pair
as the one reporter -- over G from model_docs.brute.  A single text is one document."""
import numpy as np

from tests import model_approx, model_docs

_pack, _ends, pieces, table_range = model_approx._pack, model_approx._ends, model_approx.pieces, model_approx.table_range


def levenshtein(a, b):
    """ED(a, b) with unit costs."""
    prev = list(range(len(b) + 1))
    for x, ca in enumerate(a, 1):
        cur = [x] + [0] * len(b)
        for y, cb in enumerate(b, 1):
            cur[y] = min(prev[y] + 1, cur[y - 1] + 1, prev[y - 1] + (ca != cb))
        prev = cur
    return prev[-1]


def literal(docs, queries, k):
    """The definition word for word: every (p, e) of every document.  Small inputs only."""
    text, starts = model_docs.concat(docs)
    out = []
    for q in queries:
        hits = []
        if q:
            for s, e in zip(starts.tolist(), _ends(starts, len(text))):
                for p in range(s, e):
                    d = min(levenshtein(q, text[p:x]) for x in range(p, e + 1))
                    if d <= k:
                        hits.append((p, d))
        out.append(hits)
    return _pack(out)


def dists(doc, q):
    """dist(p) of every p of one document (int64[len(doc)]): D(x, t) = min over e of ED(q[x:], doc[t:e]),
    row x = m all zeros, column t = len(doc) the deletions m - x; D(x, t) = min(D(x, t + 1) + 1,
    D(x + 1, t) + 1, D(x + 1, t + 1) + [q[x] != doc[t]]).  The row's left-to-right dependency is a suffix
    minimum of D + t."""
    L, m = len(doc), len(q)
    t = np.frombuffer(doc, dtype=np.uint8).astype(np.int64)
    idx = np.arange(L + 1, dtype=np.int64)
    row = np.zeros(L + 1, dtype=np.int64)
    for x in range(m - 1, -1, -1):
        y = row + 1                                              # delete q[x]
        y[:L] = np.minimum(y[:L], row[1:] + (t != q[x]))
        row = np.minimum.accumulate((y + idx)[::-1])[::-1] - idx
    return row[:L]


def brute(docs, queries, k):
    """(offsets, pos, dist) of every p with dist(p) <= k, by ascending p, from dists() per document."""
    text, starts = model_docs.concat(docs)
    out = []
    for q in queries:
        hits = []
        if q:
            for s, e in zip(starts.tolist(), _ends(starts, len(text))):
                if e > s:
                    d = dists(text[s:e], q)
                    hits += [(s + int(p), int(d[p])) for p in np.flatnonzero(d <= k)]
        out.append(hits)
    return _pack(out)


def band(text, q, k, c, ds, de):
    """Row 0 of the band DP of candidates (int64[C] centres c, document bounds ds, de): int64[C, 4k + 1],
    column d the value at t = c - 2k + d, exact where <= k, cells outside [ds, de] at a large INF."""
    INF = 1 << 20
    W, m = 4 * k + 1, len(q)
    tx = np.frombuffer(text, dtype=np.uint8).astype(np.int64) if text else np.zeros(0, np.int64)
    d = np.arange(W, dtype=np.int64)[None, :]
    base = (c - 2 * k)[:, None]
    lo, hi = ds[:, None], de[:, None]
    t = base + m + d
    row = np.where((t >= lo) & (t <= hi), 0, INF)
    for x in range(m - 1, -1, -1):
        t = base + x + d
        inside = (t >= lo) & (t < hi)
        ch = tx[np.clip(t, 0, max(len(tx) - 1, 0))] if len(tx) else np.zeros_like(t)
        up = np.concatenate([np.full((len(c), 1), INF), row[:, :-1]], axis=1) + 1
        y = np.where(inside, np.minimum(up, row + (ch != q[x])), np.where(t == hi, up, INF))
        y = np.minimum.accumulate((y + d)[:, ::-1], axis=1)[:, ::-1] - d  # the move from t + 1
        row = np.where(inside | (t == hi), np.minimum(y, INF), INF)
    return row


def piece_at(text, x, piece, ds, de):
    return ds <= x and x + len(piece) <= de and text[x:x + len(piece)] == piece


def reporter(text, q, k, p, ds, de):
    """R(p): the least (i, s'') with piece i exactly at s'' inside [ds, de) and |s'' - o_i - p| <= k."""
    for i, (a, b) in enumerate(pieces(len(q), k)):
        for x in range(p + a - k, p + a + k + 1):
            if piece_at(text, x, q[a:b], ds, de):
                return i, x
    return None


def model(docs, g, queries, k):
    """The device's rule: slot (q, j) holds the table range of piece j; a rank s = G[i] of it considers the
    starts p of s's document with |p - (s - o_j)| <= k, their dist from the band, and emits those with
    dist <= k whose reporter is (j, s).  A query of 0 < m <= k has one slot with the whole table, each rank
    reporting its own position."""
    text, starts = model_docs.concat(docs)
    n = len(text)
    ends = _ends(starts, n)
    out = []
    for q in queries:
        m, hits = len(q), []
        if m == 0:
            slots = []
        elif m <= k:
            slots = [(0, 0, (0, n))]
        else:
            ps = pieces(m, k)
            slots = [(j, ps[j][0], table_range(text, starts, g, q[ps[j][0]:ps[j][1]])) for j in range(k + 1)]
        cand = [(j, oj, int(g[i])) for j, oj, (s0, e0) in slots for i in range(s0, e0)]
        if cand:
            js, oj, ss = (np.asarray(x, dtype=np.int64) for x in zip(*cand))
            docs_of = [model_docs.doc_of(starts, int(s)) for s in ss]
            ds = np.asarray([int(starts[x]) for x in docs_of], dtype=np.int64)
            de = np.asarray([ends[x] for x in docs_of], dtype=np.int64)
            c = ss - oj
            row = band(text, q, k, c, ds, de)
            for r in range(len(cand)):
                j, s = int(js[r]), int(ss[r])
                if m <= k:
                    assert row[r, 2 * k] <= m
                    hits.append((s, int(row[r, 2 * k])))
                    continue
                for p in range(max(int(ds[r]), int(c[r]) - k), min(int(de[r]) - 1, int(c[r]) + k) + 1):
                    dist = int(row[r, p - int(c[r]) + 2 * k])
                    if dist <= k and reporter(text, q, k, p, int(ds[r]), int(de[r])) == (j, s):
                        hits.append((p, dist))
        assert len({p for p, _ in hits}) == len(hits), "an occurrence reported twice"
        out.append(sorted(hits))
    return _pack(out)
