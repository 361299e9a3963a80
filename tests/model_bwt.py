"""Host statements of the Burrows-Wheeler transform of documents and its inverse (include/b200sa.h,
b200sa_bwt_dev / b200sa_unbwt_dev): the definition by brute force -- rotations sorted with the terminators
as ordered symbols, no suffix array -- and a numpy model of the device steps (suffix_b200/csrc/bwt.cuh):
the row layout over G, psi by a stable argsort, rulers by hash, their walks, pointer doubling and the
emit."""
import numpy as np

from tests import model_docs

TERM = -1                 # F of a terminator row in the model's psi / F arrays
RULER_DEFAULT = 64        # BWT_RULER_DEFAULT


# ---- the definition
def brute(docs):
    """(bwt bytes, term_rows list, full L as symbols, r): the rotations of every D_d $_d sorted, with $_d the
    symbol (0, d) and byte b the symbol (1, b), so $_0 < $_1 < ... < every byte."""
    rots = []
    for d, doc in enumerate(docs):
        s = [(1, b) for b in bytes(doc)] + [(0, d)]
        rots += [tuple(s[i:] + s[:i]) for i in range(len(s))]
    rots.sort()
    L = [r[-1] for r in rots]
    term_rows = [0] * len(docs)
    for row, (kind, v) in enumerate(L):
        if kind == 0:
            term_rows[v] = row
    bwt = bytes(v for kind, v in L if kind == 1)
    runs = sum(1 for i in range(len(L)) if i == 0 or L[i] != L[i - 1])
    return bwt, term_rows, L, runs


def psi_by_definition(bwt, term_rows):
    """psi and F (TERM on a terminator row) of step 5, or None when the term rows are out of range or
    repeated."""
    n, k = len(bwt), len(term_rows)
    if k == 0 or len(set(term_rows)) != k or any(not 0 <= t < n + k for t in term_rows):
        return None
    is_term = [False] * (n + k)
    for t in term_rows:
        is_term[t] = True
    rows = [row for row in range(n + k) if not is_term[row]]        # the non-terminator rows, in row order
    order = sorted(range(n), key=lambda u: bwt[u])                 # stable: by byte, then by row
    psi = list(term_rows) + [rows[u] for u in order]
    F = [TERM] * k + [bwt[u] for u in order]
    return psi, F


def inverse_by_definition(bwt, term_rows):
    """The documents of step 5, or None when (bwt, term_rows) breaks the validity rule of step 6."""
    pf = psi_by_definition(bytes(bwt), list(term_rows))
    if pf is None:
        return None
    psi, F = pf
    k, seen, docs = len(term_rows), 0, []
    for d in range(k):
        x, out = psi[d], []
        seen += 1
        while x >= k:
            out.append(F[x])
            seen += 1
            if len(out) > len(psi):
                return None
            x = psi[x]
        if x != d:
            return None
        docs.append(bytes(out))
    return docs if seen == len(psi) else None


# ---- the device steps
def forward(docs, g):
    """(bwt, term_rows u32[k], r) from G as the device gathers them: row d < k from the document's last
    byte, row k + r from the byte before G[r], docs_find owning a position shared by empty documents."""
    text, starts = model_docs.concat(docs)
    n, k = len(text), len(docs)
    t = np.frombuffer(text, dtype=np.uint8).astype(np.int64)
    st = starts.astype(np.int64)
    ends = np.append(st[1:], n)
    sym = np.empty(n + k, dtype=np.int64)
    nonempty = ends > st
    sym[:k] = np.where(nonempty, t[np.maximum(ends - 1, 0)] if n else 0, 256 + np.arange(k))
    g = np.asarray(g, dtype=np.int64)
    d = np.searchsorted(st, g, side="right") - 1
    sym[k:] = np.where(g == st[d], 256 + d, t[g - 1] if n else 0)
    term = sym >= 256
    term_rows = np.zeros(k, dtype=np.uint32)
    term_rows[sym[term] - 256] = np.nonzero(term)[0]
    runs = int(np.count_nonzero(np.diff(sym))) + 1 if n + k else 0
    return sym[~term].astype(np.uint8).tobytes(), term_rows, runs


def _mix(x):
    x = np.asarray(x, dtype=np.uint32).copy()
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x7feb352d)
    x ^= x >> np.uint32(15)
    x *= np.uint32(0x846ca68b)
    x ^= x >> np.uint32(16)
    return x


def is_ruler(rows, k, s, n):
    """Rows below k, and (s <= n) the rows whose hash h has h * s < 2^32."""
    rows = np.asarray(rows, dtype=np.int64)
    hashed = (_mix(rows).astype(np.uint64) * np.uint64(s)) >> np.uint64(32) == 0 if s <= n else False
    return (rows < k) | hashed


def inverse(bwt, term_rows, s=RULER_DEFAULT):
    """(documents or None, record): the device's inverse step by step.  record: rulers, longest walk, rank
    rounds (None where the call stops before them), and why an input is rejected ('terms' or 'cycles')."""
    b = np.frombuffer(bytes(bwt), dtype=np.uint8)
    t = np.asarray(term_rows, dtype=np.int64)
    n, k = len(b), len(t)
    nrows = n + k
    rec = {"rulers": None, "longest": None, "rounds": None, "reject": None}
    ts = np.sort(t)
    if k == 0 or ts[-1] >= nrows or ts[0] < 0 or np.any(ts[1:] == ts[:-1]):
        rec["reject"] = "terms"
        return None, rec
    # 1. psi and F
    order = np.argsort(b, kind="stable")                       # index u of the j-th non-terminator row
    fk = b[order].astype(np.int64)
    psi = np.empty(nrows, dtype=np.int64)
    psi[:k] = t
    psi[k:] = order + np.searchsorted(ts - np.arange(k), order, side="right")
    F = np.full(nrows, TERM, dtype=np.int64)
    F[k:] = fk
    # 2. rulers and their walks
    ruler = is_ruler(np.arange(nrows), k, s, n)
    rrow = np.nonzero(ruler)[0]
    m = len(rrow)
    rank = np.full(nrows, -1, dtype=np.int64)
    rank[rrow] = np.arange(m)
    cur, steps = rrow.copy(), np.zeros(m, dtype=np.int64)
    act = np.arange(m)
    while len(act):
        cur[act] = psi[cur[act]]
        steps[act] += 1
        act = act[~ruler[cur[act]]]
    tail = cur < k
    nxt = np.where(tail, cur, rank[np.maximum(cur, 0)])
    val = np.where(tail, steps - 1, steps)
    rec["rulers"], rec["longest"] = m, int(steps.max()) if m else 0
    # 3. pointer doubling, bit_length(m) rounds at most, each one synchronous
    rounds = 0
    for _ in range(int(m).bit_length()):
        move = nxt >= k
        if not move.any():
            break
        j = np.nonzero(move)[0]
        nn, vv = nxt.copy(), val.copy()
        nn[j], vv[j] = nxt[nxt[j]], val[j] + val[nxt[j]]
        nxt, val = nn, vv
        rounds += 1
    rec["rounds"] = rounds
    if not (np.array_equal(nxt[:k], np.arange(k)) and int(steps[nxt < k].sum()) == nrows):
        rec["reject"] = "cycles"
        return None, rec
    # 4. document starts, then every ruler writes its segment
    lens = val[:k]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    pos = starts[nxt] + lens[nxt] - val
    out = np.zeros(n, dtype=np.uint8)
    cur = rrow.copy()
    for i in range(int(steps.max()) if m else 0):
        a = np.nonzero(steps > i)[0]
        cur[a] = psi[cur[a]]
        w = a[cur[a] >= k]
        out[pos[w]] = F[cur[w]]
        pos[w] += 1
    text = out.tobytes()
    return [text[int(starts[d]):int(starts[d] + lens[d])] for d in range(k)], rec
