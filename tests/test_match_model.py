"""The matching-statistics model (tests/model_match.py) against the definition by brute force: len by
bytes.find on every document, [start, end) as the positions range of the matched string, SMEMs as the
matches contained in no other match of their query."""
import itertools

import numpy as np

from tests import families, model_docs, model_match


def _check(docs, queries, min_lens=(1, 2, 3)):
    docs = [bytes(d) for d in docs]
    g, glcp = model_docs.brute(docs)
    off, ln, st, en = model_match.model(docs, g, glcp, queries)
    for k, q in enumerate(queries):
        a = int(off[k])
        want = model_match.brute_len(docs, q)
        assert ln[a:a + len(q)].tolist() == want, (docs, q)
        for j, l in enumerate(want):
            assert (int(st[a + j]), int(en[a + j])) == model_match.brute_range(docs, g, q[j:j + l]), (docs, q, j)
            assert j + 1 >= len(q) or want[j + 1] >= l - 1          # x + len[x] never decreases
    for m in min_lens:
        so, qpos = model_match.smems(off, ln, m)
        for k, q in enumerate(queries):
            a = int(off[k])
            got = qpos[int(so[k]):int(so[k + 1])].tolist()
            assert got == model_match.brute_smems(ln[a:a + len(q)].tolist(), m), (docs, q, m)
    return off, ln, st, en


def test_every_text_over_ab_up_to_7_every_query_up_to_5():
    queries = [bytes(q) for m in range(0, 6) for q in itertools.product(b"ab", repeat=m)]
    for n in range(0, 8):
        for t in itertools.product(b"ab", repeat=n):
            _check([bytes(t)], queries, min_lens=(1, 2))


def _queries(rng, docs):
    text = b"".join(docs)
    qs = [b"", b"z", text, text + b"a", b"zz" + text[:3]]
    for _ in range(6):
        if text:
            a = int(rng.integers(0, len(text)))
            q = bytearray(text[a:a + int(rng.integers(1, 9))] + text[:int(rng.integers(0, 4))])
            if rng.random() < 0.5:
                q[int(rng.integers(0, len(q)))] = text[int(rng.integers(0, len(text)))]   # a substitution
            qs.append(bytes(q))
    return qs


def test_random_document_sets():
    rng = np.random.default_rng(11)
    for _ in range(2000):
        docs = model_docs.random_docs(rng)
        _check(docs, _queries(rng, docs))


def test_family_heads_and_one_document_is_the_single_text():
    rng = np.random.default_rng(12)
    for name, text in families.adversarial():
        t = text[:48]
        qs = _queries(rng, [t])
        one = _check([t], qs)
        # cut into documents: empty ones, a duplicate and all-equal bytes among them
        cut = [t[:7], b"", t[7:20], t[7:20], t[20:], b"", b"aaaa"]
        _check(cut, qs)
        whole = _check([b"", t, b""], qs)                 # empty documents around one text change nothing
        for a, b in zip(one, whole):
            assert np.array_equal(a, b), name


def test_small_cases():
    _check([], [b"a", b""])
    _check([b""], [b"a"])
    _check([b"aaaa"], [b"aaa", b"aaaa", b"aaaaaa"])
    _check([b"ab", b"b", b"", b"ab"], [b"abab", b"bb", b"ba"])
    # a match stops at a document end: "abcd" occurs in no single document
    off, ln, st, en = _check([b"ab", b"cd"], [b"abcd"])
    assert ln.tolist() == [2, 1, 2, 1]
    # SMEMs of "abcd" at min_len 2: "ab" and "cd"
    so, qpos = model_match.smems(off, ln, 2)
    assert so.tolist() == [0, 2] and qpos.tolist() == [0, 2]


def test_c_checker_equals_the_model():
    from tests import match_check
    rng = np.random.default_rng(13)
    for k in range(300):
        docs = model_docs.random_docs(rng)
        qs = _queries(rng, docs)
        g, glcp = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        off, ln, st, en = model_match.model(docs, g, glcp, qs)
        blob = np.frombuffer(b"".join(qs), dtype=np.uint8)
        got = match_check.stats(text, starts, g, blob, off)
        assert all(np.array_equal(a, b) for a, b in zip(got, (ln, st, en))), (docs, qs)
        if len(docs) == 1:                                      # the single-text route of the checker
            got = match_check.stats(text, None, g, blob, off, 1, len(blob) - 1)
            assert all(np.array_equal(a, b[1:len(blob) - 1]) for a, b in zip(got, (ln, st, en)))
