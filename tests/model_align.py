"""Host statements of the alignments of approximate hits (include/b200sa.h, B200SA_APPROX_ALIGN): (a) the
definition -- the Hamming window, and for the edit metric the full DP D(x, t) over p <= t <= E with the canonical
walk -- (b) the banded variant the device runs, over the 2d + 1 diagonals t - p - x in [-d, d] with values
saturated at d + 1, and (c) the BAM encoding of the operations and the listing of a whole call, composed from
tests/model_approx_docs.py.  A single text is one document."""
import numpy as np

from tests import model_approx, model_approx_docs, model_iupac, model_strand

MINUS = model_strand.MINUS
I, D, EQ, X = 1, 2, 7, 8                  # BAM operation codes
OPS = "MIDNSHP=X"


def symbols(q, iupac=False, minus=False):
    """Q: q, or rc(q) for a minus hit."""
    return model_strand.revcomp(q, iupac) if minus else bytes(q)


def mismatch(seg, Q, iupac=False):
    """bool[m, len(seg)]: [not match(x, t)] for query symbol x against text byte seg[t]."""
    t = np.frombuffer(bytes(seg), dtype=np.uint8)
    if iupac:
        cls = model_iupac.classes(Q)
        return np.array([~np.isin(t, sorted(c)) for c in cls], dtype=bool).reshape(len(Q), len(t))
    q = np.frombuffer(bytes(Q), dtype=np.uint8)
    return q[:, None] != t[None, :]


def full_dp(mis):
    """D[x, t - p] for 0 <= x <= m and p <= t <= E (int64[m + 1, E - p + 1]) from mis = mismatch(T[p, E), Q)."""
    m, L = mis.shape
    idx = np.arange(L + 1, dtype=np.int64)
    D = np.zeros((m + 1, L + 1), dtype=np.int64)
    for x in range(m - 1, -1, -1):
        y = D[x + 1] + 1                                       # insertion: D(x + 1, t) + 1
        y[:L] = np.minimum(y[:L], D[x + 1, 1:] + mis[x])       # diagonal
        D[x] = np.minimum.accumulate((y + idx)[::-1])[::-1] - idx   # deletion: D(x, t + 1) + 1
    return D


def walk(value, mis):
    """The canonical walk from (0, p) over value(x, u), u = t - p, with E - p = mis.shape[1]: moves as
    (code, x, u) in walk order."""
    m, L = mis.shape
    x = u = 0
    moves = []
    while x < m:
        v = value(x, u)
        if u < L and v == value(x + 1, u + 1) + int(mis[x, u]):
            moves.append(X if mis[x, u] else EQ)
            x, u = x + 1, u + 1
        elif v == value(x + 1, u) + 1:
            moves.append(I)
            x += 1
        else:
            moves.append(D)
            u += 1
    return moves, u


def band_dp(mis, d):
    """The device's banded DP: B[x, j] for cell t - p = x + j - d, j in [0, 2d + 1), saturated at d + 1; cells
    outside p <= t <= E hold d + 1."""
    m, L = mis.shape
    W, INF = 2 * d + 1, d + 1
    j = np.arange(W, dtype=np.int64)
    B = np.full((m + 1, W), INF, dtype=np.int64)
    u = m + j - d
    B[m] = np.where((u >= 0) & (u <= L), 0, INF)
    for x in range(m - 1, -1, -1):
        u = x + j - d
        valid = (u >= 0) & (u <= L)
        up = np.concatenate([[INF], B[x + 1, :-1]]) + 1         # D(x + 1, t) + 1: one diagonal down
        diag = np.full(W, 2 * INF, dtype=np.int64)
        inner = valid & (u < L)
        diag[inner] = B[x + 1, inner] + mis[x, u[inner]]
        a = np.where(valid, np.minimum(np.minimum(diag, up), INF), INF)
        s = np.minimum.accumulate((a + j)[::-1])[::-1] - j      # the deletion, a suffix minimum
        B[x] = np.where(valid, np.minimum(s, INF), INF)
    return B


def merge(moves):
    """[(code, len)] of adjacent equal moves."""
    out = []
    for c in moves:
        if out and out[-1][0] == c:
            out[-1][1] += 1
        else:
            out.append([c, 1])
    return [(c, n) for c, n in out]


def words(ops, minus=False):
    """BAM words len << 4 | code, with MINUS on a minus hit."""
    return [(n << 4 | c) | (MINUS if minus else 0) for c, n in ops]


def cigar(ops):
    return "".join("%d%s" % (n, OPS[c]) for c, n in ops)


def align(text, E, p, q, d, metric="hamming", iupac=False, minus=False, banded=False):
    """(ops [(code, len)], end) of the hit (p, d) of q in text whose document ends at E."""
    Q = symbols(q, iupac, minus)
    m = len(Q)
    if metric == "hamming":
        mis = mismatch(text[p:p + m], Q, iupac)
        return merge([X if mis[x, x] else EQ for x in range(m)]), p + m
    mis = mismatch(text[p:E], Q, iupac)
    if banded:
        B = band_dp(mis, d)
        value = lambda x, u: int(B[x, u - x + d]) if 0 <= u - x + d <= 2 * d else d + 1
    else:
        Dm = full_dp(mis)
        value = lambda x, u: int(Dm[x, u])
    assert value(0, 0) == d, (value(0, 0), d)
    moves, u = walk(value, mis)
    return merge(moves), p + u


def listing(docs, queries, k, metric="hamming", iupac=False, best=None, strands="forward", banded=True):
    """(offsets, pos, words) of the call with B200SA_APPROX_ALIGN: every hit of L(q) (the call without the flag),
    in its order, expanded into its operations."""
    off, pos, dist = model_approx_docs.flagless(docs, queries, k, metric, iupac, best, strands)
    text = b"".join(bytes(x) for x in docs)
    starts = model_approx_docs.starts_of(docs)
    ends = model_approx._ends(starts, len(text)) if len(starts) else []
    out = []
    for qi, q in enumerate(queries):
        ent = []
        for i in range(int(off[qi]), int(off[qi + 1])):
            p, dd = int(pos[i]), int(dist[i])
            minus, dd = dd >= MINUS, dd & (MINUS - 1)
            E = ends[model_approx_docs.doc_of(starts, p)]
            ops, _ = align(text, E, p, q, dd, metric, iupac, minus, banded)
            ent += [(p, w) for w in words(ops, minus)]
        out.append(ent)
    return model_approx._pack(out)
