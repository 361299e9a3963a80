"""Pure-Python statement of the generalized suffix tree of include/b200sa.h (b200sa_docs_tree):
rules 1-8 of the single-text tree with rule 3' and per-rank document suffix lengths, the
terminal prefix term_end and the distinct-document counts by Hui's method, over (G, glcp) of
b200sa_docs_build.  Stack-based ANSV as in tests/model_tree.py.  It is the specification the
CUDA kernels (suffix_b200/csrc/tree.cuh, docs_tree.cuh) implement; `brute` is the definition."""
import numpy as np

from tests import model_docs
from tests.model_tree import NONE, _ansv

FIELDS = ("parent", "depth", "sa_lo", "sa_hi", "label_start", "subtree_end", "term_end", "doc_count")


def _ends(starts, n):
    return [int(x) for x in starts[1:]] + [n]


def tree_arrays(g, glcp, starts, n) -> dict:
    """The eight arrays by preorder id from G, glcp and doc_starts (n = total bytes)."""
    g = [int(x) for x in g]
    if n == 0:
        return {f: np.array([v], dtype=np.uint32) for f, v in zip(FIELDS, (NONE, 0, 0, 0, 0, 1, 0, 0))}
    ends = _ends(starts, n)
    doc = [model_docs.doc_of(starts, p) for p in g]
    ln = [ends[d] - p for d, p in zip(doc, g)]
    L = [int(x) for x in glcp] + [0]                      # glcp[n] := 0
    psv, pse, nsv = _ansv(L, n)
    by_lo = [[] for _ in range(n)]
    by_lo[0].append((0, n))                               # rule 1
    for i in range(1, n):                                 # rule 2
        if L[i] > 0 and pse[i] == psv[i]:
            by_lo[psv[i]].append((L[i], nsv[i]))
    for r in range(n):                                    # rule 3'
        merged = (r + 1 < n and L[r + 1] == ln[r]) or (r > 0 and L[r] == ln[r])
        if not merged:
            by_lo[r].append((ln[r], r + 1))
    lo_of, dep, hi_of, ident = [], [], [], {}
    for lo in range(n):                                   # rule 4
        for d, hi in sorted(by_lo[lo]):
            ident[(lo, d)] = len(lo_of)
            lo_of.append(lo)
            dep.append(d)
            hi_of.append(hi)
    N = len(lo_of)
    first, nxt = [0] * (n + 1), N                         # first id with sa_lo >= lo
    for lo in range(n, -1, -1):
        if lo < n and by_lo[lo]:
            nxt = ident[(lo, min(by_lo[lo])[0])]
        first[lo] = nxt if lo < n else N
    parent, label_start, subtree_end = [NONE] * N, [0] * N, [N] * N
    for v in range(1, N):
        lo, hi, d = lo_of[v], hi_of[v], dep[v]
        pd = max(L[lo], L[hi])                            # rule 5
        parent[v] = 0 if pd == 0 else ident[(lo if L[hi] > L[lo] else psv[lo], pd)]
        label_start[v] = g[lo] + pd                       # rule 6
        subtree_end[v] = first[hi] if hi < n else N       # rule 7
    # term_end: the last rank of each run of equal strings closes the terminals of node (a, len)
    term_end = list(lo_of)
    for r in range(n):
        if r + 1 < n and L[r + 1] == ln[r] and ln[r + 1] == ln[r]:
            continue
        a = r
        if L[r] >= ln[r]:
            a = r - 1
            while L[a] >= ln[r]:
                a -= 1
        term_end[ident[(a, ln[r])]] = r + 1
    # Hui: ranks stably by document; each pair (prev, i) adds 1 at the node of its common prefix
    order = sorted(range(n), key=lambda r: doc[r])
    pairs_at = [0] * (N + 1)
    for k in range(1, n):
        p, i = order[k - 1], order[k]
        if doc[p] != doc[i]:
            continue
        D = min(L[p + 1:i + 1])
        if D == 0:
            pairs_at[0] += 1
        else:
            lo = p
            while L[lo] >= D:
                lo -= 1
            pairs_at[ident[(lo, D)]] += 1
    P = [0] * (N + 1)
    for v in range(N):
        P[v + 1] = P[v] + pairs_at[v]
    doc_count = [(hi_of[v] - lo_of[v]) - (P[subtree_end[v]] - P[v]) for v in range(N)]
    return {f: np.array(a, dtype=np.uint32) for f, a in zip(
        FIELDS, (parent, dep, lo_of, hi_of, label_start, subtree_end, term_end, doc_count))}


def brute(docs) -> dict:
    """The definition: the compressed trie of the document suffixes T_p, nodes in lexicographic
    order, with the eight arrays derived from the node strings directly.  Also returns, under
    "strings" and "doc_sets", every node's string and its set of documents."""
    text, starts = model_docs.concat(docs)
    n = len(text)
    g, _ = model_docs.brute(docs)
    g = [int(x) for x in g]
    ends = _ends(starts, n)
    doc = {p: model_docs.doc_of(starts, p) for p in range(n)}
    suf = {p: text[p:ends[doc[p]]] for p in range(n)}
    ts = [suf[p] for p in g]                               # T in G order
    nodes = {b""} | set(ts)
    for s in {t[:k] for t in ts for k in range(len(t))}:
        if len({t[len(s)] for t in ts if len(t) > len(s) and t.startswith(s)}) >= 2:
            nodes.add(s)
    strs = sorted(nodes)
    N = len(strs)
    ident = {s: v for v, s in enumerate(strs)}
    out = {f: [] for f in FIELDS}
    doc_sets = []
    for v, s in enumerate(strs):
        rows = [i for i, t in enumerate(ts) if t.startswith(s)]
        lo, hi = (rows[0], rows[-1] + 1) if rows else (0, 0)
        assert rows == list(range(lo, hi))
        par = NONE
        for k in range(len(s) - 1, -1, -1):
            if s[:k] in ident:
                par = ident[s[:k]]
                break
        end = v + 1
        while end < N and strs[end].startswith(s):
            end += 1
        nterm = sum(1 for i in rows if ts[i] == s)
        assert all(ts[i] == s for i in rows[:nterm])       # terminals are a prefix of the range
        ds = {doc[g[i]] for i in rows}
        doc_sets.append(ds)
        pd = 0 if par == NONE else len(strs[par])
        for f, x in zip(FIELDS, (par, len(s), lo, hi, (g[lo] + pd) if v else 0, end, lo + nterm, len(ds))):
            out[f].append(x)
    res = {f: np.array(a, dtype=np.uint32) for f, a in out.items()}
    res["strings"] = strs
    res["doc_sets"] = doc_sets
    return res
