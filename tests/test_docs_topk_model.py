"""The top-k model (tests/model_docs_topk.py) against brute force: for every query, the documents that contain
it ranked by overlapping occurrence count (then by document), from np.unique over the documents of G[s:e], on
the random document sets of model_docs.random_docs, every substring of each set up to length 4 and absent
queries, for k in {1, 2, 3, 1024}."""
import numpy as np

from tests import model_docs, model_docs_list, model_docs_topk

KS = (1, 2, 3, 1024)


def _brute(doc, s, e, k):
    d, cnt = np.unique(doc[s:e], return_counts=True)
    o = np.lexsort((d, -cnt))                                       # count descending, then document
    return [(int(d[i]), int(cnt[i])) for i in o[:k]]


def _check(docs, queries):
    g, doc, byd, prev = model_docs_list.index(docs)
    text, starts = model_docs.concat(docs)
    n = len(text)
    for q in queries:
        s, e = model_docs_list.query_range(docs, g, q)
        df = len({d for d, x in enumerate(docs) if q and q in x})
        for k in KS:
            got = model_docs_topk.top_k(starts, n, doc, byd, prev, s, e, k)
            assert got == _brute(doc, s, e, k), (docs, q, k)
            assert len(got) == min(k, df)
            assert all((-a[1], a[0]) < (-b[1], b[0]) for a, b in zip(got, got[1:]))   # strict: keys are unique


def test_random_sets_every_short_substring():
    rng = np.random.default_rng(7)
    for _ in range(2400):
        docs = model_docs.random_docs(rng)
        qs = {x[a:a + m] for x in docs for m in range(1, 5) for a in range(len(x) - m + 1)}
        qs |= {b"", b"z", b"\x01", b"aaaaaaaaaaz", (docs[0] + b"\x02") if docs else b"\x02"}   # absent
        _check(docs, sorted(qs))


def test_small_cases():
    _check([], [b"a", b""])
    _check([b""], [b"a"])
    docs = [b"ab", b"abab", b"b", b"ababab", b"", b"ab"]
    _check(docs, [b"a", b"ab", b"b", b"ba", b"c"])
    g, doc, byd, prev = model_docs_list.index(docs)
    text, starts = model_docs.concat(docs)
    s, e = model_docs_list.query_range(docs, g, b"ab")
    # tf 3 (D3), 2 (D1), then the tie at 1 by document: D0, D5
    assert model_docs_topk.top_k(starts, len(text), doc, byd, prev, s, e, 3) == [(3, 3), (1, 2), (0, 1)]
    assert model_docs_topk.top_k(starts, len(text), doc, byd, prev, s, e, 9) == [(3, 3), (1, 2), (0, 1), (5, 1)]
