"""The numpy model of the LPF / LZ77 device steps (tests/model_lz.py) against the definitions by brute force,
known answers, and the properties the device parse relies on."""
import math

import numpy as np
import pytest

from tests import model_docs, model_lz as mz

L = mz.LITERAL

# text: (lpf, factors (start, len, src or None for a literal))
KNOWN = {
    b"aaaaaaaa": ([0, 7, 6, 5, 4, 3, 2, 1], [(0, 1, None), (1, 7, 0)]),
    b"abababab": ([0, 0, 6, 5, 4, 3, 2, 1], [(0, 1, None), (1, 1, None), (2, 6, 0)]),
    b"banana": ([0, 0, 0, 3, 2, 1], [(0, 1, None), (1, 1, None), (2, 1, None), (3, 3, 1)]),
    b"mississippi": ([0, 0, 0, 1, 4, 3, 2, 1, 0, 1, 1],
                     [(0, 1, None), (1, 1, None), (2, 1, None), (3, 1, 2), (4, 4, 1), (8, 1, None), (9, 1, 8),
                      (10, 1, 7)]),
    b"abaababaabaab": ([0, 0, 1, 3, 2, 6, 5, 4, 5, 4, 3, 2, 1],
                       [(0, 1, None), (1, 1, None), (2, 1, 0), (3, 3, 0), (6, 5, 1), (11, 2, 8)]),
}


def _table(docs):
    return model_docs.brute(mz._docs(docs))


@pytest.mark.parametrize("text", list(KNOWN))
def test_known_answers(text):
    want_lpf, want_f = KNOWN[text]
    g, lcp = _table(text)
    lpf, src = mz.lpf_src(g, lcp)
    assert lpf.tolist() == want_lpf and mz.brute_lpf(text).tolist() == want_lpf
    start, length, source, rounds = mz.factors(g, lcp)
    got = [(int(s), int(l), None if q == L else int(q)) for s, l, q in zip(start, length, source)]
    assert got == want_f
    assert rounds == math.ceil(math.log2(len(got)))
    if text == b"mississippi":
        assert [None if q == L else int(q) for q in src] == [None, None, None, 2, 1, 2, 3, 4, None, 8, 7]


def _fib(k):
    a, b = b"a", b"ab"
    for _ in range(k):
        a, b = b, b + a
    return b


def check(docs):
    """Model against brute force, and every stated property, on one text or document set."""
    docs = mz._docs(docs)
    text, starts = model_docs.concat(docs)
    n = len(text)
    g, lcp = model_docs.brute(docs)
    lpf, src = mz.lpf_src(g, lcp)
    assert np.array_equal(lpf, mz.brute_lpf(docs)), docs
    ends = np.append(starts[1:], n).astype(np.int64)
    de = ends[np.searchsorted(starts, np.arange(n), side="right") - 1]
    assert np.all(lpf.astype(np.int64) <= de - np.arange(n))                     # no factor crosses a document end
    assert np.all(lpf[1:].astype(np.int64) >= lpf[:-1].astype(np.int64) - 1)     # next never decreases
    for p in range(n):                                                            # src is an earlier occurrence
        if lpf[p]:
            assert src[p] < p and text[src[p]:src[p] + lpf[p]] == text[p:p + lpf[p]]
        else:
            assert src[p] == L
    start, length, source, rounds = mz.factors(g, lcp)
    s0, l0 = mz.serial_parse(lpf)
    assert np.array_equal(start, s0) and np.array_equal(length, l0), docs
    z = len(start)
    assert int(length.astype(np.int64).sum()) == n
    assert rounds == (math.ceil(math.log2(z)) if z else 0)
    nonempty = [int(starts[d]) for d in range(len(docs)) if len(docs[d])]
    assert set(nonempty) <= set(start.tolist())
    lit = bytes(text[s] for s, q in zip(start.tolist(), source.tolist()) if q == L)
    assert mz.decode(n, start, length, source, lit) == text
    return z, rounds


@pytest.mark.parametrize("alpha", [b"a", b"ab", b"ACGT", bytes(range(256))])
def test_random_texts(alpha):
    rng = np.random.default_rng(len(alpha))
    for _ in range(120):
        n = int(rng.integers(1, 60))
        check(bytes(rng.choice(list(alpha), n)))


def test_families():
    for k in range(1, 8):
        check(_fib(k))                                                  # Fibonacci words
    for period in (b"ab", b"abc", b"aab", b"ACGTA"):
        for reps in (1, 2, 5, 11):
            check(period * reps + period[:2])                           # periodic strings
    for n in (1, 2, 3, 4, 5, 8, 9, 16, 17, 33, 64, 65):                 # all distinct: z = n, the most rounds
        z, rounds = check(bytes(range(n)))
        assert z == n and rounds == math.ceil(math.log2(n))


def test_document_sets():
    rng = np.random.default_rng(7)
    sets = [[b""], [b"", b"x"], [b"x", b"x"], [b"a", b"", b"a", b"b"], [b"ab", b"ab", b"b", b""],
            [b"", b"", b"abc", b"", b"c"]]
    sets += [model_docs.random_docs(rng) for _ in range(300)]
    sets += [[bytes([int(x)]) if rng.random() < 0.5 else b"" for x in rng.integers(0, 3, 8)] for _ in range(50)]
    for docs in sets:
        if sum(map(len, docs)):
            check(docs)


def test_one_document_is_the_single_text():
    rng = np.random.default_rng(11)
    for _ in range(50):
        t = bytes(rng.choice(list(b"ab"), int(rng.integers(1, 40))))
        g1, l1 = _table(t)
        g2, l2 = model_docs.brute([t])
        assert [x.tolist() for x in mz.factors(g1, l1)[:3]] == [x.tolist() for x in mz.factors(g2, l2)[:3]]


def test_rounds_at_powers_of_two():
    # z at 2^k - 1, 2^k and 2^k + 1: distinct bytes then one long copy
    for k in range(1, 7):
        for z in (2 ** k - 1, 2 ** k, 2 ** k + 1):
            if z < 2:
                continue
            t = bytes(range(z - 1)) + bytes(range(z - 1))[:3] if z >= 4 else bytes(range(z))
            g, lcp = _table(t)
            start, _, _, rounds = mz.factors(g, lcp)
            assert rounds == math.ceil(math.log2(len(start)))


def test_serial_checker_equals_the_model():
    from tests import lz_check
    rng = np.random.default_rng(13)
    cases = [bytes(rng.choice(list(a), int(rng.integers(1, 200)))) for a in (b"a", b"ab", b"ACGT") for _ in range(40)]
    cases += [bytes(range(256)), _fib(9), b"abc" * 50]
    cases += [model_docs.random_docs(rng) for _ in range(100)]
    for t in cases:
        docs = mz._docs(t)
        text, _ = model_docs.concat(docs)
        if not text:
            continue
        g, lcp = model_docs.brute(docs)
        lpf, src, start, length, source = lz_check.lz(g, lcp)
        wl, ws = mz.lpf_src(g, lcp)
        assert np.array_equal(lpf, wl) and np.array_equal(src, ws), t
        assert all(np.array_equal(a, b) for a, b in zip((start, length, source), mz.factors(g, lcp)[:3])), t
        assert lz_check.decode(text, start, length, source).tobytes() == text
    with pytest.raises(ValueError):                                    # the decoder rejects a broken parse
        lz_check.decode(b"abab", np.array([0, 1, 2]), np.array([1, 1, 2]), np.array([L, L, 2]))   # source = start
