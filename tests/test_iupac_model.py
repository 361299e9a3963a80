"""The host statements of IUPAC queries (tests/model_iupac.py): the class table, the stretch pieces, the
device's rule against the definition for both metrics, exhaustively over small texts, and the serial C
statement of tests/iupac_check.c.  CPU only."""
import itertools

import numpy as np
import pytest

from tests import iupac_check, model_approx, model_docs, model_edit, model_iupac

CODES = b"ACGTURYSWKMBDHVN"


def _rand_query(rng, m, alpha=CODES + CODES.lower()):
    return bytes(int(alpha[int(x)]) for x in rng.integers(0, len(alpha), m))


def _text(rng, n):
    """DNA with soft-masked, N and U bytes mixed in."""
    return bytes(int(b"ACGTACGTACGTacgNU"[int(x)]) for x in rng.integers(0, 17, n))


def test_class_table():
    want = {"A": "A", "C": "C", "G": "G", "T": "T", "U": "T", "R": "AG", "Y": "CT", "S": "CG", "W": "AT",
            "K": "GT", "M": "AC", "B": "CGT", "D": "AGT", "H": "ACT", "V": "ACG", "N": "ACGT"}
    assert sorted(model_iupac.CLASSES) == sorted(want)
    for letter, bases in want.items():
        for b in (letter, letter.lower()):
            assert model_iupac.classes(b.encode()) == [frozenset(bases.encode())]
    for bad in (b"-", b".", b"X", b"x", b"Z", b"*", b"\x00", b"\xc1", b"AC-G"):
        with pytest.raises(ValueError):
            model_iupac.classes(bad)
    assert model_iupac.expansions(b"NGG") == [b + b"GG" for b in (b"A", b"C", b"G", b"T")]
    assert model_iupac.canon(b"acguRn") == b"ACGTRN"


def test_concrete_queries_get_f14_pieces():
    rng = np.random.default_rng(1)
    for _ in range(300):
        m, k = int(rng.integers(1, 60)), int(rng.integers(0, 32))
        q = _rand_query(rng, m, b"ACGTUacgtu")
        got = model_iupac.pieces(q, k)
        if m <= k:
            assert got is None
        else:
            assert got == [(a, b - a) for a, b in model_approx.pieces(m, k)], (q, k)


def test_piece_rule():
    rng = np.random.default_rng(2)
    for _ in range(2000):
        m, k = int(rng.integers(1, 50)), int(rng.integers(0, 32))
        alpha = [CODES + CODES.lower(), b"ACGTN", b"ACGTACGTACGTACGTN", b"NNNNA"][int(rng.integers(0, 4))]
        q = _rand_query(rng, m, alpha)
        ls = [L for _, L in model_iupac.stretches(q)]
        assert sum(ls) == sum(b in model_iupac.CONCRETE for b in q)
        pcs, t = model_iupac.pieces(q, k), model_iupac.piece_length(q, k)
        if sum(ls) < k + 1:
            assert pcs is None and t is None
            continue
        assert len(pcs) == k + 1
        assert sum(L // t for L in ls) >= k + 1 and sum(L // (t + 1) for L in ls) < k + 1   # t is the largest
        cover = [x for o, L in pcs for x in range(o, o + L)]
        assert len(cover) == len(set(cover))                                            # disjoint
        assert all(L >= t for _, L in pcs)
        assert all(q[x] in model_iupac.CONCRETE for x in cover)                          # concrete
        assert [o for o, _ in pcs] == sorted(o for o, _ in pcs)


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_rule_equals_definition(metric):
    rng = np.random.default_rng(3 if metric == "hamming" else 4)
    for k in (0, 1, 2, 3, 4, 31):
        for _ in range(6 if k < 31 else 3):
            n = int(rng.integers(0, 70))
            text = _text(rng, n)
            cuts = sorted(int(x) for x in rng.integers(0, n + 1, int(rng.integers(0, 4))))
            docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [n])]
            qs = [b"", _rand_query(rng, 1), b"N" * 5, b"NGG", _rand_query(rng, k + 1, b"ACGTN")]
            for _ in range(5):
                if n > 4:
                    a = int(rng.integers(0, n - 4))
                    src = bytearray(text[a:a + int(rng.integers(3, 16))].upper().replace(b"U", b"T"))
                    for x in range(len(src)):                                   # degenerate some positions
                        if rng.random() < 0.25:
                            src[x] = int(CODES[int(rng.integers(4, len(CODES)))])
                    qs.append(bytes(src))
            want = model_iupac.brute(docs, qs, k, metric)
            got = model_iupac.rule(docs, qs, k, metric)
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (docs, qs, k)


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_exhaustive_small_texts_report_each_occurrence_once(metric):
    queries = [bytes(q) for m in (1, 2, 3) for q in itertools.product(b"ACNRa", repeat=m)]
    for n in range(0, 5):
        for text in itertools.product(b"ACaN", repeat=n):
            text = bytes(text)
            doc_sets = [[text]] + ([[text[:2], text[2:]]] if n >= 3 else [])
            for docs in doc_sets:
                for k in (0, 1):
                    qs = queries if k == 0 or n <= 3 else queries[:30]
                    want = model_iupac.brute(docs, qs, k, metric)
                    got = model_iupac.rule(docs, qs, k, metric)
                    assert all(np.array_equal(a, b) for a, b in zip(got, want)), (docs, k)


def test_properties_of_the_definition():
    rng = np.random.default_rng(5)
    for _ in range(25):
        docs = [_text(rng, int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 4)))]
        plain = [_rand_query(rng, int(rng.integers(1, 8)), b"ACGT") for _ in range(4)]
        k = int(rng.integers(0, 4))
        # a query of uppercase A C G T alone is the plain definition
        assert all(np.array_equal(a, b) for a, b in zip(model_iupac.brute(docs, plain, k),
                                                         model_approx.brute(docs, plain, k)))
        assert all(np.array_equal(a, b) for a, b in zip(model_iupac.brute(docs, plain, k, "edit"),
                                                         model_edit.brute(docs, plain, k)))
        # lowercase letters act as their uppercase, U as T
        low = [q.lower().replace(b"t", b"u") for q in plain]
        for metric in ("hamming", "edit"):
            assert all(np.array_equal(a, b) for a, b in zip(model_iupac.brute(docs, low, k, metric),
                                                             model_iupac.brute(docs, plain, k, metric)))
        # k = 0: the union of the exact occurrences of every expansion
        q = _rand_query(rng, int(rng.integers(1, 5)), b"ACGTRYN")
        _, pos, _ = model_iupac.brute(docs, [q], 0)
        union = sorted(set(p for e in model_iupac.expansions(q) for p in model_approx.brute(docs, [e], 0)[1].tolist()))
        assert pos.tolist() == union, (docs, q)


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_c_statement_equals_definition(metric):
    rng = np.random.default_rng(6)
    for k in (0, 1, 2, 4, 31):
        for _ in range(8):
            n = int(rng.integers(0, 120))
            text = _text(rng, n)
            cuts = sorted(int(x) for x in rng.integers(0, n + 1, int(rng.integers(0, 5))))
            docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [n])]
            qs = [b"", _rand_query(rng, int(rng.integers(1, 12))), b"NGG", b"acgun"]
            want = model_iupac.brute(docs, qs, k, metric)
            c_text, starts = model_docs.concat(docs)
            got = iupac_check.iupac(c_text, starts, qs, k, metric)
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (docs, qs, k)
            if len(docs) == 1:
                got = iupac_check.iupac(text, None, qs, k, metric)
                assert all(np.array_equal(a, b) for a, b in zip(got, want)), (docs, qs, k)
