"""Host statements of approximate positions (include/b200sa.h, b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev): (a) the definition by brute force over every window, and (b) the
device's rule in pure Python -- pieces, table ranges of the pieces, candidates, and the first exactly
matching piece as the one reporter -- over G from model_docs.brute.  A single text is one document."""
import numpy as np

from tests import model_docs


def _pack(lists):
    """(offsets u64[nq + 1], pos u32[], mis u32[]) of per-query lists of (p, mis)."""
    off = np.zeros(len(lists) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(h) for h in lists])
    flat = [x for h in lists for x in h]
    pos = np.asarray([p for p, _ in flat], dtype=np.uint32)
    mis = np.asarray([e for _, e in flat], dtype=np.uint32)
    return off, pos, mis


def _ends(starts, n):
    return [int(x) for x in starts[1:]] + [n]


def hamming(a, b):
    return sum(x != y for x, y in zip(a, b))


def brute(docs, queries, k):
    """Every window [p, p + m) inside one document with at most k mismatches, by ascending p."""
    text, starts = model_docs.concat(docs)
    ends = _ends(starts, len(text))
    out = []
    for q in queries:
        m, hits = len(q), []
        if m:
            for s, e in zip(starts.tolist(), ends):
                for p in range(s, e - m + 1):
                    d = hamming(text[p:p + m], q)
                    if d <= k:
                        hits.append((p, d))
        out.append(hits)
    return _pack(out)


def pieces(m, k):
    """The k + 1 pieces [j*m/P, (j+1)*m/P) of a query of m > k bytes."""
    P = k + 1
    return [(j * m // P, (j + 1) * m // P) for j in range(P)]


def table_range(text, starts, g, piece):
    """[s, e) of the ranks of G whose suffix, cut at its document's end, starts with piece (contiguous)."""
    n = len(text)
    ends = _ends(starts, n)
    hit = [text[int(p):ends[model_docs.doc_of(starts, int(p))]].startswith(piece) for p in g]
    idx = [i for i, h in enumerate(hit) if h]
    if not idx:
        return 0, 0
    assert idx == list(range(idx[0], idx[-1] + 1))
    return idx[0], idx[-1] + 1


def model(docs, g, queries, k):
    """The device's rule: slot (q, j) holds the table range of piece j; a rank s = G[i] of it gives
    p = s - o_j, kept when the window lies in s's document, no piece i < j matches exactly and the other
    pieces add at most k mismatches.  A query of 0 < m <= k has one slot with the whole table."""
    text, starts = model_docs.concat(docs)
    n = len(text)
    ends = _ends(starts, n)
    out = []
    for q in queries:
        m, hits = len(q), []
        if m == 0:
            slots = []
        elif m <= k:
            slots = [(0, (0, 0), (0, n))]
        else:
            ps = pieces(m, k)
            slots = [(j, ps[j], table_range(text, starts, g, q[ps[j][0]:ps[j][1]])) for j in range(k + 1)]
        for j, (oj, _), (s0, e0) in slots:
            for i in range(s0, e0):
                s = int(g[i])
                if s < oj:
                    continue
                p = s - oj
                d = model_docs.doc_of(starts, s)
                if p < int(starts[d]) or p + m > ends[d]:
                    continue
                w = text[p:p + m]
                if m <= k:
                    hits.append((p, hamming(w, q)))
                    continue
                ps = pieces(m, k)
                assert w[ps[j][0]:ps[j][1]] == q[ps[j][0]:ps[j][1]]
                if any(w[a:b] == q[a:b] for a, b in ps[:j]):
                    continue                                  # an earlier slot reports it
                mis = sum(hamming(w[a:b], q[a:b]) for a, b in ps)
                if mis <= k:
                    hits.append((p, mis))
        assert len({p for p, _ in hits}) == len(hits), "an occurrence reported twice"
        out.append(sorted(hits))
    return _pack(out)
