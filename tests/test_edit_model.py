"""The device's rule for the edit metric of approximate positions (tests/model_edit.py: pieces, windows of starts,
the band of 4k + 1 diagonals, the least (piece, position) pair as the one reporter) against the definition, and
the serial C statement of tests/edit_check.c against it.  CPU only."""
import itertools

import numpy as np
import pytest

from tests import edit_check, model_approx, model_docs, model_edit

KS = list(range(7)) + [31]


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def edited(rng, src, edits, alpha):
    """src with `edits` random substitutions, insertions and deletions."""
    q = bytearray(src)
    for _ in range(edits):
        op = int(rng.integers(0, 3))
        x = int(rng.integers(0, len(q) + 1))
        c = int(alpha[int(rng.integers(0, len(alpha)))])
        if op == 0 and x < len(q):
            q[x] = c
        elif op == 1:
            q.insert(x, c)
        elif x < len(q):
            del q[x]
    return bytes(q)


def _queries(rng, docs, k):
    """m = 0, m <= k, m = k + 1, m > n, substrings with substitutions and indels, and substrings that start or
    end at a document end."""
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
        qs.append(edited(rng, d[a:a + m], int(rng.integers(0, k + 2)), alpha))
        qs.append(edited(rng, d[len(d) - m:], int(rng.integers(0, 2)), alpha))   # near the document end
        qs.append(d[:m])
    return qs


def _cases(rng, count):
    for _ in range(count):
        yield model_docs.random_docs(rng, alphabets=(b"ab", b"abc", b"a", b"ACGT"))
    allb = bytes(int(x) for x in rng.permutation(256))
    for _ in range(4):                                             # all byte values
        yield [bytes(int(x) for x in rng.integers(0, 256, int(rng.integers(1, 12)))) for _ in range(3)]
    yield []
    yield [b""]
    yield [b"", b"", b"ab", b""]
    yield [allb[:40], b"", allb[40:70], allb[:7]]
    yield [b"a" * 12, b"a" * 5]
    yield [b"ab" * 6, b"", b"ba" * 3]


def test_brute_force_equals_literal_definition():
    rng = np.random.default_rng(300)
    for docs in _cases(rng, 60):
        for k in (0, 1, 2, 4):
            qs = [q for q in _queries(rng, docs, k) if len(q) <= 12]
            assert _same(model_edit.brute(docs, qs, k), model_edit.literal(docs, qs, k)), (docs, qs, k)


@pytest.mark.parametrize("k", KS)
def test_model_equals_brute_force(k):
    rng = np.random.default_rng(310 + k)
    for docs in _cases(rng, 100 if k < 31 else 40):
        g, _ = model_docs.brute(docs)
        qs = _queries(rng, docs, k)
        want = model_edit.brute(docs, qs, k)
        assert _same(model_edit.model(docs, g, qs, k), want), (docs, qs, k)
        if len(docs) == 1:                                         # a single text is one document
            assert _same(model_edit.model([b"".join(docs)], g, qs, k), want)


def _strings(alpha, lo, hi):
    return [bytes(s) for m in range(lo, hi + 1) for s in itertools.product(alpha, repeat=m)]


@pytest.mark.parametrize("k", [0, 1, 2])
def test_reporter_partitions_occurrences_exhaustively(k):
    """Every text over {a, b} up to 5 bytes, as one document and cut into two at every place, with every query
    over {a, b} of 1 to 4 bytes: each occurrence has a reporter and is emitted once (model asserts no repeats)."""
    qs = _strings(b"ab", 1, 4)
    for t in _strings(b"ab", 0, 5):
        for docs in [[t]] + [[t[:x], t[x:]] for x in range(len(t) + 1)]:
            g, _ = model_docs.brute(docs)
            want = model_edit.brute(docs, qs, k)
            assert _same(model_edit.model(docs, g, qs, k), want), (docs, k)
            text, starts = model_docs.concat(docs)
            ends = [int(x) for x in starts[1:]] + [len(text)]
            off, pos = want[0], want[1]
            for q, a, b in zip(qs, off[:-1], off[1:]):
                if len(q) <= k:
                    continue
                for p in pos[int(a):int(b)].tolist():
                    d = model_docs.doc_of(starts, p)
                    assert model_edit.reporter(text, q, k, p, int(starts[d]), ends[d]) is not None, (docs, q, p)


def test_k0_is_exact_positions():
    rng = np.random.default_rng(320)
    for docs in _cases(rng, 60):
        text, starts = model_docs.concat(docs)
        ends = [int(x) for x in starts[1:]] + [len(text)]
        qs = _queries(rng, docs, 0)
        off, pos, dist = model_edit.brute(docs, qs, 0)
        assert not dist.any()
        for q, a, b in zip(qs, off[:-1], off[1:]):
            want = [p for s, e in zip(starts.tolist(), ends) for p in range(s, e) if q and text[p:e].startswith(q)]
            assert pos[int(a):int(b)].tolist() == want


@pytest.mark.parametrize("k", [1, 2, 3, 5])
def test_hamming_occurrences_are_edit_occurrences(k):
    rng = np.random.default_rng(330 + k)
    for docs in _cases(rng, 60):
        qs = _queries(rng, docs, k)
        ho, hp, hm = model_approx.brute(docs, qs, k)
        eo, ep, ed = model_edit.brute(docs, qs, k)
        for q in range(len(qs)):
            e = dict(zip(ep[int(eo[q]):int(eo[q + 1])].tolist(), ed[int(eo[q]):int(eo[q + 1])].tolist()))
            for p, mis in zip(hp[int(ho[q]):int(ho[q + 1])].tolist(), hm[int(ho[q]):int(ho[q + 1])].tolist()):
                assert p in e and e[p] <= mis, (docs, qs[q], p)


def test_short_queries_take_every_position():
    docs = [b"abc", b"", b"de"]
    off, pos, dist = model_edit.brute(docs, [b"zz", b"bc", b"zzzz"], 2)
    assert off.tolist() == [0, 5, 10, 10]
    assert pos[:5].tolist() == [0, 1, 2, 3, 4] and dist[:5].tolist() == [2, 2, 2, 2, 2]
    assert pos[5:].tolist() == [0, 1, 2, 3, 4] and dist[5:].tolist() == [1, 0, 1, 2, 2]


@pytest.mark.parametrize("k", [0, 2, 5, 31])
def test_c_statement_equals_brute_force(k):
    rng = np.random.default_rng(340 + k)
    for docs in _cases(rng, 80):
        qs = _queries(rng, docs, k)
        text, starts = model_docs.concat(docs)
        want = model_edit.brute(docs, qs, k)
        assert _same(edit_check.edit(text, starts, qs, k), want), (docs, qs, k)
        if len(docs) == 1:
            assert _same(edit_check.edit(text, None, qs, k), want)
