"""The device's rule for approximate positions (tests/model_approx.py: pieces, candidates, the first exactly
matching piece as the one reporter) against the definition by brute force, and the serial C statement of
tests/approx_check.c against both.  CPU only."""
import numpy as np
import pytest

from tests import approx_check, model_approx, model_docs

KS = list(range(7)) + [31]


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _queries(rng, docs, k):
    """m = 0, m <= k, m = k + 1, m > n, substrings with substitutions, and windows that end at a document end."""
    text = b"".join(docs)
    alpha = sorted(set(text)) or [97]
    rand = lambda m: bytes(int(alpha[int(x)]) for x in rng.integers(0, len(alpha), m))
    qs = [b"", rand(1), rand(max(k, 1)), rand(k + 1), rand(k + 2), text + b"a", rand(len(text) + 1)]
    nonempty = [d for d in docs if d]
    for _ in range(6):
        if not nonempty:
            break
        d = nonempty[int(rng.integers(0, len(nonempty)))]
        m = int(rng.integers(1, len(d) + 1))
        a = int(rng.integers(0, len(d) - m + 1))
        q = bytearray(d[a:a + m])
        for _ in range(int(rng.integers(0, k + 2))):
            q[int(rng.integers(0, m))] = int(alpha[int(rng.integers(0, len(alpha)))])
        qs.append(bytes(q))
        qs.append(d[len(d) - m:])                                  # ends exactly at the document end
    return qs


def _cases(rng, count):
    for _ in range(count):
        yield model_docs.random_docs(rng)
    yield []
    yield [b""]
    yield [b"", b"", b"ab", b""]
    allb = bytes(int(x) for x in rng.permutation(256))
    yield [allb[:100], b"", allb[100:], allb[:7]]
    yield [b"a" * 12, b"a" * 5]


@pytest.mark.parametrize("k", KS)
def test_model_equals_brute_force(k):
    rng = np.random.default_rng(100 + k)
    for docs in _cases(rng, 120):
        g, _ = model_docs.brute(docs)
        qs = _queries(rng, docs, k)
        want = model_approx.brute(docs, qs, k)
        assert _same(model_approx.model(docs, g, qs, k), want), (docs, qs, k)
        if len(docs) == 1:                                         # a single text is one document
            assert _same(model_approx.model([b"".join(docs)], g, qs, k), want)


def test_k0_is_exact_positions():
    rng = np.random.default_rng(7)
    for docs in _cases(rng, 60):
        text, starts = model_docs.concat(docs)
        ends = [int(x) for x in starts[1:]] + [len(text)]
        qs = _queries(rng, docs, 0)
        off, pos, mis = model_approx.brute(docs, qs, 0)
        assert not mis.any()
        for q, a, b in zip(qs, off[:-1], off[1:]):
            want = [p for s, e in zip(starts.tolist(), ends) for p in range(s, e) if q and text[p:e].startswith(q)]
            assert pos[int(a):int(b)].tolist() == want


def test_short_queries_take_every_window():
    docs = [b"abc", b"", b"de"]
    off, pos, mis = model_approx.brute(docs, [b"zz", b"zzz", b"zzzz"], 3)
    assert pos.tolist() == [0, 1, 3, 0] and mis.tolist() == [2, 2, 2, 3]
    assert off.tolist() == [0, 3, 4, 4]


@pytest.mark.parametrize("k", [0, 2, 5, 31])
def test_c_statement_equals_brute_force(k):
    rng = np.random.default_rng(200 + k)
    for docs in _cases(rng, 80):
        qs = _queries(rng, docs, k)
        text, starts = model_docs.concat(docs)
        want = model_approx.brute(docs, qs, k)
        assert _same(approx_check.approx(text, starts, qs, k), want), (docs, qs, k)
        if len(docs) == 1:
            assert _same(approx_check.approx(text, None, qs, k), want)
