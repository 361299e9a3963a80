"""The host statements of fixed symbols in IUPAC queries (tests/model_fixed.py): the stated invariants on the
model, the constrained distances against the unconstrained ones, the band of the constrained walk, the bulge that
only the device's DP can place, the keyword checks, and the serial C statement of tests/fixed_check.c.  CPU
only."""
import numpy as np
import pytest

from suffix_b200 import _approx
from tests import fixed_check, model_align, model_approx_docs, model_best, model_fixed, model_iupac

CODES = b"ACGTURYSWKMBDHVN"
MIXES = [(metric, best, strands) for metric in ("hamming", "edit") for best in (None, 0, 1)
         for strands in ("forward", "both")]


def _text(rng, n):
    """DNA with soft-masked, N and U bytes mixed in."""
    return bytes(int(b"ACGTACGTACGTacgNU"[int(x)]) for x in rng.integers(0, 17, n))


def _docs(rng):
    return [_text(rng, int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 4)))]


def _mark(rng, q, where):
    """q uppercased with the positions where[x] lowercased."""
    return bytes(b | 0x20 if f else b for b, f in zip(bytes(q).upper(), where))


def _queries(rng, docs, k):
    """Substrings of the documents (non-codes as N) with degenerate symbols, marked as a PAM suffix, a prefix, a
    middle, all, none, and at random; m <= k; m = 0."""
    text = b"".join(docs).upper()
    src = bytes(b if b in CODES else ord("N") for b in text) or b"ACGT"
    out = [b"", b"ngg"[:max(1, min(3, k))], b"ACGTn"]
    for _ in range(4):
        m = int(rng.integers(1, min(len(src), 14) + 1))
        a = int(rng.integers(0, len(src) - m + 1))
        q = bytearray(src[a:a + m])
        for x in rng.integers(0, m, int(rng.integers(0, 3))):
            q[int(x)] = CODES[int(rng.integers(0, 16))]
        q = bytes(q)
        x0 = int(rng.integers(0, m))
        out += [_mark(rng, q, [x >= m - 2 for x in range(m)]), _mark(rng, q, [x < 2 for x in range(m)]),
                _mark(rng, q, [x0 <= x < x0 + 2 for x in range(m)]), q.lower(), q,
                _mark(rng, q, rng.random(m) < 0.3)]
    return out


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _split_words(packed):
    """Per query, per hit: [(p, minus, [(code, len)])] of an operation listing."""
    out = []
    off, pos, words = packed
    for q in range(len(off) - 1):
        hits = []
        for i in range(int(off[q]), int(off[q + 1])):
            p, w = int(pos[i]), int(words[i])
            key = (p, w >= model_fixed.MINUS)
            if not hits or hits[-1][:2] != key:
                hits.append((p, key[1], []))
            hits[-1][2].append((w & 15, (w & (model_fixed.MINUS - 1)) >> 4))
        out.append(hits)
    return out


def test_no_lowercase_is_the_iupac_call():
    rng = np.random.default_rng(1)
    for i in range(25):
        docs, k = _docs(rng), i % 4
        qs = [q.upper() for q in _queries(rng, docs, k)]
        for metric, best, strands in MIXES:
            want = model_approx_docs.flagless(docs, qs, k, metric, True, best, strands)
            assert _same(model_fixed.listing(docs, qs, k, metric, best, strands), want), (docs, k)
            assert _same(model_fixed.listing(docs, qs, k, metric, best, strands, documents=True),
                         model_approx_docs.brute(docs, qs, k, metric, True, best, strands))
        for metric in ("hamming", "edit"):
            got = model_fixed.listing(docs, qs, k, metric, None, "both", align_ops=True)
            want = model_align.listing(docs, qs, k, metric, True, None, "both", banded=False)
            assert _same(got, want), (docs, k)


def test_hamming_is_the_filtered_iupac_list():
    rng = np.random.default_rng(2)
    for i in range(40):
        docs, k = _docs(rng), i % 5
        qs = _queries(rng, docs, k)
        text = b"".join(docs)
        plain = model_best.lists(model_iupac.brute(docs, qs, k))
        got = model_best.lists(model_fixed.one_strand(docs, qs, k))
        for q, hp, hg in zip(qs, plain, got):
            cls, fx = model_iupac.classes(q), model_fixed.marks(q)
            keep = [(p, d) for p, d in hp
                    if all(text[p + x] in cls[x] for x in range(len(q)) if fx[x])]
            assert hg == keep, (q, k)


def test_all_fixed_is_exact_under_either_metric():
    rng = np.random.default_rng(3)
    for i in range(30):
        docs = _docs(rng)
        qs = [q.lower() for q in _queries(rng, docs, 3) if q]
        exact = model_iupac.brute(docs, qs, 0)
        for k in (0, 1, 3):
            for metric in ("hamming", "edit"):
                got = model_fixed.one_strand(docs, qs, k, metric)
                assert _same(got, exact), (docs, k, metric)


def test_alignments_keep_fixed_symbols_whole():
    rng = np.random.default_rng(4)
    seen = 0
    for i in range(30):
        docs, k = _docs(rng), 1 + i % 3
        qs = _queries(rng, docs, k)
        for metric in ("hamming", "edit"):
            for strands in ("forward", "both"):
                listing = model_fixed.listing(docs, qs, k, metric, None, strands, align_ops=True)
                for q, hits in zip(qs, _split_words(listing)):
                    for p, minus, ops in hits:
                        Q = model_align.symbols(q, True, minus)
                        fx = model_fixed.marks(Q)
                        x = 0
                        for code, n in ops:
                            for _ in range(n):
                                if code in (model_fixed.X, model_fixed.I):
                                    assert not fx[x], (q, p, ops)
                                if code == model_fixed.D:
                                    assert not fx[x] and not (x > 0 and fx[x - 1]), (q, p, ops)
                                else:
                                    x += 1
                        seen += len(ops)
    assert seen > 100


def test_constrained_distance_is_at_least_the_free_one_and_walks_in_the_band():
    rng = np.random.default_rng(5)
    for _ in range(300):
        doc = _text(rng, int(rng.integers(1, 30))).upper()
        q = _queries(rng, [doc], 2)[int(rng.integers(3, 27))]
        free = model_iupac.dists(doc, model_iupac.classes(q))
        fixed = model_fixed.dists(doc, q)
        assert (fixed >= free).all(), (doc, q)
        mis = model_align.mismatch(doc, q, True)
        for p in np.flatnonzero(fixed <= 4).tolist():
            m = model_align.mismatch(doc[p:], q, True)
            Dm = model_fixed.full_dp(m, model_fixed.marks(q))
            d = int(Dm[0, 0])
            assert d == fixed[p]
            _, _, cells = model_fixed.walk(m, model_fixed.marks(q), Dm)
            assert all(abs(u - x) <= d for x, u in cells), (doc, q, p)
        assert mis.shape == (len(q), len(doc))


def test_a_bulge_next_to_the_pam_goes_into_the_spacer():
    q, text = b"ACGTgg", b"ACGTTGG"
    cls = model_iupac.classes(q)
    assert model_iupac.dists(text, cls)[0] == 1 and model_fixed.dists(text, q)[0] == 1
    ops_free, _ = model_align.align(text, len(text), 0, q, 1, "edit", True)
    assert model_align.cigar(ops_free) == "4=1X1="                     # a substitution in the PAM
    ops, end = model_fixed.align(text, len(text), 0, q, 1, "edit")
    assert model_align.cigar(ops) == "3=1D3=" and end == 7
    off, pos, dist = model_fixed.one_strand([text], [q], 1, "edit")
    assert 0 in pos.tolist() and int(dist[pos.tolist().index(0)]) == 1
    _, hpos, _ = model_fixed.one_strand([text], [q], 1)
    assert hpos.tolist() == []              # Hamming: the window at 0 breaks gg, the one at 1 has 3 free misses


def test_keywords():
    assert _approx.FIXED == 0x2000000
    assert _approx._fixed(False, False) == 0 and _approx._fixed(False, True) == 0
    assert _approx._fixed(True, True) == _approx.FIXED and _approx._fixed(np.bool_(True), True) == _approx.FIXED
    for bad in (1, 0, None, "yes", b"", (True,)):
        with pytest.raises(ValueError):
            _approx._fixed(bad, True)
    with pytest.raises(ValueError):
        _approx._fixed(True, False)
    for kw in (dict(fixed=True), dict(fixed=1, iupac=True), dict(fixed="no", iupac=True)):
        with pytest.raises(ValueError):                                # before the table is touched
            _approx._call(None, [b"ACGT"], 1, True, **kw)


def test_c_statement_equals_the_model():
    rng = np.random.default_rng(6)
    for i in range(40):
        docs, k = _docs(rng), i % 4
        qs = _queries(rng, docs, k)
        text = b"".join(docs)
        starts = model_approx_docs.starts_of(docs)
        for metric in ("hamming", "edit"):
            got = fixed_check.fixed(text, starts.astype(np.uint32), qs, k, metric)
            want = model_fixed.one_strand(docs, qs, k, metric)
            assert _same(got, want), (docs, k, metric)
    text = _text(rng, 300).upper()
    qs = _queries(rng, [text], 2)
    for metric in ("hamming", "edit"):                               # a single text
        got = fixed_check.fixed(text, None, qs, 2, metric)
        assert _same(got, model_fixed.one_strand([text], qs, 2, metric))
