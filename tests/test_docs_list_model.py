"""The document-listing model (tests/model_docs_list.py) against brute force: for every query, the set of
documents that contain it and the overlapping occurrence count in each, on the random document sets of
model_docs.random_docs, every substring of each set up to length 4 and absent queries."""
import numpy as np

from tests import model_docs, model_docs_list


def _count(doc: bytes, q: bytes) -> int:
    k, i = 0, doc.find(q)
    while i >= 0:
        k += 1
        i = doc.find(q, i + 1)
    return k


def _check(docs, queries):
    g, doc, byd, prev = model_docs_list.index(docs)
    text, starts = model_docs.concat(docs)
    n = len(text)
    ends = np.append(starts[1:], n)
    # byd: every document's ranks, in increasing order, at [starts[d], ends[d])
    for d in range(len(docs)):
        run = byd[int(starts[d]):int(ends[d])].tolist()
        assert run == sorted(r for r in range(n) if doc[r] == d), (docs, d)
    for q in queries:
        s, e = model_docs_list.query_range(docs, g, q)
        got = model_docs_list.listing(starts, n, doc, byd, prev, s, e)
        assert [i for i, _, _ in got] == sorted(i for i, _, _ in got)
        want = {d: _count(x, q) for d, x in enumerate(docs) if q and q in x}
        assert {d: tf for _, d, tf in got} == want, (docs, q)
        assert len(got) == len(want)                               # one entry per document


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
    _check([b"aaaa", b"", b"aa", b"aaaa"], [b"a", b"aa", b"aaa", b"aaaaa"])
    g, doc, byd, prev = model_docs_list.index([b"ab", b"b", b"", b"ab"])
    # G by (suffix, document): ab in D0, ab in D3, b in D0, D1, D3 -> byd 0 2 | 3 | | 1 4, prev 0 0 1 0 2
    assert g.tolist() == [0, 3, 1, 2, 4]
    assert byd.tolist() == [0, 2, 3, 1, 4] and prev.tolist() == [0, 0, 1, 0, 2]
