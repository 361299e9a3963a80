"""The host statements of separate budgets for substitutions, DNA and RNA bulges (tests/model_bulges.py): the model
against the serial C statement of tests/bulges_check.c, the stated properties (d = r = 0 is the Hamming call, the
hits are a subset of the edit call at t + d + r with no smaller distance, monotone budgets, canonical CIGARs within
the budgets at the hit's cost), and the keyword checks, which fail before any device work.  CPU only."""
import numpy as np
import pytest

from suffix_b200 import _approx
from tests import (bulges_check, model_align, model_approx, model_approx_docs, model_bulges, model_edit, model_fixed,
                   model_iupac, model_strand)
from tests.test_fixed_model import _docs, _queries


def _dna(rng, n, alphabet=b"ACGT"):
    return bytes(alphabet[int(x)] for x in rng.integers(0, len(alphabet), n))


def _plain_docs(rng):
    return [_dna(rng, int(rng.integers(0, 30)), b"ACGTa") for _ in range(int(rng.integers(1, 4)))]


def _plain_queries(rng, docs):
    text = b"".join(docs) or b"ACGT"
    out = [b"", b"A", b"CG"]
    for _ in range(4):
        m = int(rng.integers(1, min(len(text), 10) + 1))
        a = int(rng.integers(0, len(text) - m + 1))
        q = bytearray(text[a:a + m])
        for x in rng.integers(0, m, int(rng.integers(0, 3))):
            q[x] = b"ACGT"[int(rng.integers(0, 4))]
        out.append(bytes(q))
    return out


def _c(docs, qs, t, d, r, iupac=False, fixed=False):
    starts = model_approx_docs.starts_of(docs).astype(np.uint32)
    return bulges_check.bulges(b"".join(docs), starts, qs, t, d, r, iupac, fixed)


def _same(a, b):
    return all(np.array_equal(np.asarray(x, dtype=np.uint64), np.asarray(y, dtype=np.uint64)) for x, y in zip(a, b))


@pytest.mark.parametrize("seed", range(4))
def test_model_equals_the_c_statement(seed):
    rng = np.random.default_rng(seed)
    for _ in range(3):
        docs = _plain_docs(rng)
        qs = _plain_queries(rng, docs)
        for t, d, r in ((0, 1, 0), (0, 0, 1), (1, 1, 1), (2, 0, 2), (1, 3, 3), (0, 0, 0)):
            want = model_bulges.one_strand(docs, qs, t, d, r)
            assert _same(want, _c(docs, qs, t, d, r)), (seed, t, d, r)
        idocs = _docs(rng)
        iqs = _queries(rng, idocs, 2)
        for t, d, r in ((1, 1, 0), (0, 1, 1), (2, 1, 1)):
            for fixed in (False, True):
                want = model_bulges.one_strand(idocs, iqs, t, d, r, True, fixed)
                assert _same(want, _c(idocs, iqs, t, d, r, True, fixed)), (seed, t, d, r, fixed)


@pytest.mark.parametrize("seed", range(3))
def test_no_bulges_is_hamming(seed):
    rng = np.random.default_rng(100 + seed)
    docs = _plain_docs(rng)
    qs = _plain_queries(rng, docs)
    for t in (0, 1, 2, 4):
        assert _same(model_bulges.one_strand(docs, qs, t, 0, 0), model_approx.brute(docs, qs, t)), t
    idocs = _docs(rng)
    iqs = _queries(rng, idocs, 2)
    for t in (0, 1, 2):
        iq_upper = [q.upper() for q in iqs]
        assert _same(model_bulges.one_strand(idocs, iq_upper, t, 0, 0, True), model_iupac.brute(idocs, iq_upper, t))
        assert _same(model_bulges.one_strand(idocs, iqs, t, 0, 0, True, True), model_fixed.one_strand(idocs, iqs, t))


@pytest.mark.parametrize("seed", range(3))
def test_subset_of_edit_and_monotone(seed):
    rng = np.random.default_rng(200 + seed)
    docs = _plain_docs(rng)
    qs = _plain_queries(rng, docs)
    for t, d, r in ((0, 1, 1), (1, 1, 0), (2, 0, 1), (1, 2, 2)):
        got = model_bulges.one_strand(docs, qs, t, d, r)
        edit = model_edit.brute(docs, qs, t + d + r)
        for q, (hb, he) in enumerate(zip(_lists(got), _lists(edit))):
            ed = dict(he)
            assert all(p in ed and x >= ed[p] for p, x in hb), (t, d, r, q)
        for bigger in ((t + 1, d, r), (t, min(d + 1, 3), r), (t, d, min(r + 1, 3))):   # monotone in t, d and r
            wide = [dict(h) for h in _lists(model_bulges.one_strand(docs, qs, *bigger))]
            assert all(p in w and w[p] <= x for h, w in zip(_lists(got), wide) for p, x in h), (t, d, r, bigger)


def _lists(packed):
    off, pos, dist = packed
    return [list(zip(pos[int(off[q]):int(off[q + 1])].tolist(), dist[int(off[q]):int(off[q + 1])].tolist()))
            for q in range(len(off) - 1)]


@pytest.mark.parametrize("seed", range(3))
def test_cigars_meet_the_budgets(seed):
    rng = np.random.default_rng(300 + seed)
    docs = _docs(rng)
    qs = _queries(rng, docs, 2)
    for t, d, r in ((1, 1, 1), (0, 2, 1), (2, 1, 0)):
        for fixed in (False, True):
            off, pos, words = model_bulges.listing(docs, qs, t, d, r, True, fixed, "both", align_ops=True)
            hoff, p, dist, minus, ends, coff, cigar = _approx._hits(off, pos, words)
            for h in range(len(p)):
                ops = cigar[int(coff[h]):int(coff[h + 1])]
                n = {c: int(sum(int(w) >> 4 for w in ops if int(w) & 15 == c)) for c in (1, 2, 7, 8)}
                assert n[8] <= t and n[2] <= d and n[1] <= r, (t, d, r, ops)
                assert n[8] + n[2] + n[1] == dist[h]


def test_bulge_beside_the_pam():
    guide = b"GACGCTGACGCTGACGTTGA"
    site = guide[:15] + b"C" + guide[15:] + b"TGG"                # one text base inside the spacer
    text = b"TTTT" + site + b"AAAA"
    q = guide + b"ngg"
    E = len(text)
    assert model_bulges.dist(text, E, 4, q, 0, 1, 0, True, True) == 1
    ops, end = model_bulges.align(text, E, 4, q, 1, 0, 1, 0, True, True)
    assert model_align.cigar(ops).count("D") == 1 and end == 4 + len(site)
    assert model_bulges.dist(text, E, 4, q, 0, 0, 0, True, True) is None


def test_keyword_checks_fail_before_the_device():
    class NoDevice:                                                # any attribute access would fail
        pass

    t = NoDevice()
    for bad in ((1,), (1, 2, 3), [1, 1], (4, 0), (0, -1), (True, 0), (1.0, 0), "11", 3):
        with pytest.raises(ValueError):
            _approx.positions(t, b"ACGT", 1, metric="edit", bulges=bad)
    with pytest.raises(ValueError):
        _approx.counts(t, [b"ACGT"], 1, bulges=(1, 1))                          # needs metric="edit"
    with pytest.raises(ValueError):
        _approx.positions_batch(t, [b"ACGT"], 1, metric="edit", best=0, bulges=(1, 1))
    with pytest.raises(ValueError):
        _approx.positions(t, b"ACGT", 26, metric="edit", bulges=(3, 3))          # 32 > 31
    assert _approx._bulges(None, 31, "edit", None) == 0
    assert _approx._bulges((1, 2), 4, "edit", None) == 0x200000 | (1 << 17) | (2 << 22)
    assert model_strand.MINUS == _approx.MINUS
