"""Approximate positions on both DNA strands (tests/model_strand.py) against the one-strand definitions: the
reverse complement, plain and in IUPAC codes, the stated consequences of include/b200sa.h (B200SA_APPROX_BOTH_STRANDS)
exhaustively over small texts on {A, C, G, T} with a few other bytes, best hits over the union, the co-rank merge
rule, and the strands= argument.  CPU only."""
import itertools

import numpy as np
import pytest

from suffix_b200 import _approx
from tests import model_approx, model_best, model_iupac, model_strand

METRICS = ("hamming", "edit")
MINUS = model_strand.MINUS
CODES = b"ACGTURYSWKMBDHVN"


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _sets():
    """Every text on {A, C, G, T} of at most 3 letters, texts with N, a soft-masked base and other bytes, as one
    text and cut into documents around an empty one."""
    texts = [bytes(w) for m in range(4) for w in itertools.product(b"ACGT", repeat=m)]
    texts += [b"ACGTNACGT", b"GAATTCaattc", b"TTGCAxAC", b"NNNN", b"acgtACGT", b"AAGGTTCCAGT"]
    out = []
    for text in texts:
        out.append([text])
        if len(text) > 1:
            cut = len(text) // 2
            out.append([text[:cut], b"", text[cut:]])
    return out


PLAIN_QS = [b"", b"A", b"AC", b"GT", b"ACG", b"ACGT", b"GAATTC", b"TTG", b"aC", b"AxT", b"CCAG"]
IUPAC_QS = [b"", b"A", b"NG", b"RY", b"ACN", b"GAATTC", b"TTGa", b"MKu", b"BD", b"ACGT"]


def test_revcomp_plain_is_an_involution_on_bytes():
    allb = bytes(range(256))
    assert model_strand.revcomp(model_strand.revcomp(allb)) == allb
    for b in range(256):
        c = model_strand.comp(b)
        if b in b"ACGTacgt":
            assert c != b and c in b"ACGTacgt" and model_strand.comp(c) == b
        else:
            assert c == b, hex(b)
    assert model_strand.revcomp(b"ACCGTu") == b"uACGGT"
    assert model_strand.revcomp(b"") == b""


def test_revcomp_iupac_complements_each_class():
    base = {"A": "T", "C": "G", "G": "C", "T": "A"}
    for code in CODES + CODES.lower():
        c = model_strand.comp(code, True)
        assert (c >= 0x61) == (code >= 0x61), chr(code)                  # the case is kept
        got = set(model_iupac.CLASSES[chr(c).upper()])
        want = {ord(base[chr(b)]) for b in model_iupac.CLASSES[chr(code).upper()]}
        assert got == want, chr(code)
    assert model_strand.comp(b"U"[0], True) == b"A"[0] and model_strand.comp(b"u"[0], True) == b"a"[0]
    pairs = {"R": "Y", "K": "M", "B": "V", "D": "H", "S": "S", "W": "W", "N": "N"}
    for a, b in pairs.items():
        assert model_strand.comp(ord(a), True) == ord(b) and model_strand.comp(ord(b), True) == ord(a)
    q = b"GTGCCAGCMGCCGCGGTAA"
    assert model_strand.revcomp(q, True) == b"TTACCGCGGCKGCTGGCAC"
    no_u = bytes(b for b in CODES + CODES.lower() if b not in b"Uu")
    assert model_strand.revcomp(model_strand.revcomp(no_u, True), True) == no_u


def _check_consequences(docs, qs, k, metric, iupac):
    both = model_strand.brute(docs, qs, k, metric, iupac)
    plus = model_best.lists(model_strand.one_strand(docs, qs, k, metric, iupac))
    minus = model_best.lists(model_strand.one_strand(docs, [model_strand.revcomp(q, iupac) for q in qs], k, metric,
                                                     iupac))
    text = b"".join(docs)
    for q, h, (sp, sm), hp, hm in zip(qs, model_best.lists(both), model_strand.strand_lists(both), plus, minus):
        assert sp == hp and sm == hm, (docs, q, k)
        assert [p for p, _ in h] == sorted(p for p, _ in h)
        assert h == model_strand.merge(hp, hm)                        # the co-rank rule gives the (p, strand) order
        if model_strand.revcomp(q, iupac) == q:                       # a palindrome: every hit twice
            assert [p for p, _ in h] == sorted([p for p, _ in hp] * 2)
        if not q:
            assert h == []
        elif len(q) <= k:                                             # every window twice
            if metric == "hamming":
                want = [p for s, d in zip(*_bounds(docs)) for p in range(s, d - len(q) + 1)]
            else:
                want = list(range(len(text)))
            assert [p for p, _ in h] == sorted(want * 2), (docs, q, k)


def _bounds(docs):
    starts = np.cumsum([0] + [len(d) for d in docs[:-1]]).tolist()
    return starts, [s + len(d) for s, d in zip(starts, docs)]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("iupac", [False, True])
def test_stated_consequences(metric, iupac):
    qs = IUPAC_QS if iupac else PLAIN_QS
    for docs in _sets():
        for k in (0, 1, 2):
            _check_consequences(docs, qs, k, metric, iupac)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("iupac", [False, True])
def test_best_over_both_strands(metric, iupac):
    qs = IUPAC_QS if iupac else PLAIN_QS
    for docs in _sets():
        for k in (0, 1, 2):
            full = model_strand.brute(docs, qs, k, metric, iupac)
            assert _same(model_strand.brute(docs, qs, k, metric, iupac, best=k), full)            # s >= k
            assert _same(model_strand.brute(docs, qs, k, metric, iupac, best=k + 3), full)
            for s in range(k + 1):
                got = model_best.lists(model_strand.brute(docs, qs, k, metric, iupac, best=s))
                for q, hf, hg in zip(qs, model_best.lists(full), got):
                    if not hf:
                        assert hg == []
                        continue
                    b = min(d & (MINUS - 1) for _, d in hf)                                      # over the union
                    t = min(k, b + s)
                    assert hg == [h for h in hf if h[1] & (MINUS - 1) <= t], (docs, q, k, s)
                    if s == 0:
                        assert {d & (MINUS - 1) for _, d in hg} == {b}
        zero = model_strand.brute(docs, qs, 0, metric, iupac, best=0)                             # k = 0: exact
        assert _same(zero, model_strand.brute(docs, qs, 0, metric, iupac))
        assert not (zero[2] & (MINUS - 1)).any()


def test_only_the_minus_strand_holds_the_best_hit():
    q = b"AACCGGTTAC"
    rc = model_strand.revcomp(q)
    near = bytearray(q)
    near[3] ^= 0x02                                                    # one substitution: the plus hit at d = 1
    text = b"TTTT" + bytes(near) + b"GGGG" + rc + b"TTTT"
    for metric in METRICS:
        full = model_strand.strand_lists(model_strand.brute([text], [q], 2, metric))[0]
        assert (4, 1) in full[0] and (18, 0) in full[1]
        plus, minus = model_strand.strand_lists(model_strand.brute([text], [q], 2, metric, best=0))[0]
        assert plus == [] and minus == [(18, 0)], metric


def test_merge_rule_orders_by_position_then_strand():
    rng = np.random.default_rng(7)
    for _ in range(300):
        a = sorted(set(rng.integers(0, 30, int(rng.integers(0, 12))).tolist()))
        b = sorted(set(rng.integers(0, 30, int(rng.integers(0, 12))).tolist()))
        plus = [(p, int(rng.integers(0, 4))) for p in a]
        minus = [(p, int(rng.integers(0, 4))) for p in b]
        got = model_strand.merge(plus, minus)
        want = sorted([(p, d, 0) for p, d in plus] + [(p, d, 1) for p, d in minus], key=lambda h: (h[0], h[2]))
        assert got == [(p, d | (MINUS if s else 0)) for p, d, s in want]


def test_split():
    off, pos, d, minus = model_strand.split((np.array([0, 2], np.uint64), np.array([3, 3], np.uint32),
                                             np.array([1, 2 | MINUS], np.uint32)))
    assert d.tolist() == [1, 2] and minus.tolist() == [False, True]


def test_strands_argument():
    assert _approx._strands("forward") == 0
    assert _approx._strands("both") == _approx.BOTH_STRANDS == 0x10000000
    assert _approx.MINUS == MINUS
    for bad in ("Both", "reverse", "", None, True, 1, b"both", ("both",)):
        with pytest.raises(ValueError):
            _approx._strands(bad)


def test_model_matches_the_one_strand_rule_on_a_longer_text():
    rng = np.random.default_rng(11)
    text = bytes(rng.choice(list(b"ACGT"), 400).tolist())
    qs = [text[a:a + 12] for a in rng.integers(0, 380, 6).tolist()]
    qs += [model_strand.revcomp(q) for q in qs[:3]]
    for k in (0, 2):
        for metric in METRICS:
            got = model_strand.strand_lists(model_strand.brute([text], qs, k, metric))
            for q, (hp, hm) in zip(qs, got):
                assert hp == model_best.lists(model_strand.one_strand([text], [q], k, metric))[0]
                assert hm == model_best.lists(model_strand.one_strand([text], [model_strand.revcomp(q)], k, metric))[0]
            ham = model_approx.brute([text], qs, k)
            if metric == "hamming":
                assert all(p == hp for p, (hp, _) in zip(model_best.lists(ham), got))
