"""Host statement of document listing (include/b200sa.h, b200sa_docs_list_index_dev / b200sa_docs_list_dev):
byd, prev, the listing predicate prev[i] <= s and tf, on G from model_docs.brute."""
import numpy as np

from tests import model_docs


def index(docs):
    """(G, doc of every rank, byd, prev) of a document set."""
    g, _ = model_docs.brute(docs)
    _, starts = model_docs.concat(docs)
    n = len(g)
    doc = (np.searchsorted(starts, g, side="right") - 1).astype(np.int64)
    byd = np.lexsort((np.arange(n), doc)).astype(np.uint32)        # stable by document, then rank
    prev = np.zeros(n, dtype=np.uint32)
    for k in range(1, n):
        if doc[byd[k - 1]] == doc[byd[k]]:
            prev[byd[k]] = byd[k - 1] + 1
    return g, doc, byd, prev


def query_range(docs, g, q):
    """[s, e) of the ranks whose document suffix starts with q (b200sa_docs_positions_dev)."""
    text, starts = model_docs.concat(docs)
    n = len(text)
    if not q or n == 0:
        return 0, 0
    ends = np.append(starts[1:], n)
    hits = []
    for i, p in enumerate(g.tolist()):
        d = int(np.searchsorted(starts, p, side="right")) - 1
        if text[p:int(ends[d])].startswith(q):
            hits.append(i)
    if not hits:
        return 0, 0
    assert hits == list(range(hits[0], hits[-1] + 1))              # a contiguous range of G
    return hits[0], hits[-1] + 1


def listing(starts, n, doc, byd, prev, s, e):
    """(i, d, tf) for every listed rank i of [s, e), ascending i."""
    ends = np.append(starts[1:], n).astype(np.int64)
    out = []
    for i in range(s, e):
        if prev[i] <= s:
            d = int(doc[i])
            run = byd[int(starts[d]):int(ends[d])]
            tf = int(np.searchsorted(run, e)) - int(np.searchsorted(run, i))
            out.append((i, d, tf))
    return out
