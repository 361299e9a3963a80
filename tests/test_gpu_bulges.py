"""Separate budgets for substitutions, DNA bulges and RNA bulges (B200SA_APPROX_BULGES on
b200sa_docs_approx_positions_dev, bulges= on the approximate_positions* and approximate_counts methods): bit for bit
against tests/model_bulges.py on small collections and every mix of IUPAC, FIXED, strands, documents and align;
every budget against the serial C statement; the stated properties on the device; 1 MB of DNA against the C
statement; and the argument checks and listing protocol."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib
from tests import bulges_check, model_approx_docs, model_bulges, model_strand
from tests.test_fixed_model import _docs, _queries
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
BULGES = 0x200000                               # B200SA_APPROX_BULGES
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
FIXED = 0x2000000                               # B200SA_APPROX_FIXED
ALIGN = 0x8000000                               # B200SA_APPROX_ALIGN
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
DOCS = 0x20000000                               # B200SA_APPROX_DOCUMENTS
MINUS = model_strand.MINUS
MODES = {"hits": 0, "documents": DOCS, "align": ALIGN}


def _kf(t, d, r, iupac=False, fixed=False, strands="forward", mode="hits"):
    return (t | EDIT | BULGES | (d << 17) | (r << 22) | (IUPAC if iupac else 0) | (FIXED if fixed else 0) |
            (BOTH if strands == "both" else 0) | MODES[mode])


def _starts(docs):
    return model_approx_docs.starts_of(docs).astype(np.uint32)


def _call(ctx, docs, qs, kf):
    text = b"".join(docs)
    g = DocumentSuffixTable(docs).table() if text else []
    return _fetch(ctx, text, g, qs, kf, _starts(docs))


def _substrings(rng, text, count=4, longest=9):
    src = text or b"ACGT"
    out = [b"", src[:1]]
    for _ in range(count):
        m = int(rng.integers(1, min(len(src), longest) + 1))
        a = int(rng.integers(0, len(src) - m + 1))
        q = bytearray(src[a:a + m])
        for x in rng.integers(0, m, int(rng.integers(0, 3))):
            q[x] = src[int(rng.integers(0, len(src)))]
        out.append(bytes(q))
    return out


def test_families_against_the_model():
    rng = np.random.default_rng(1)
    ctx = _lib.Context(0)
    budgets = [(0, 1, 0), (0, 0, 1), (1, 1, 1), (0, 2, 3), (2, 0, 0)]
    for i, docs in enumerate(_families(rng)[::6]):
        if not docs or not b"".join(docs):
            continue
        t, d, r = budgets[i % len(budgets)]
        qs = _substrings(rng, b"".join(docs))
        want = model_bulges.one_strand(docs, qs, t, d, r)
        assert _same(_call(ctx, docs, qs, _kf(t, d, r)), want), (i, t, d, r)
        got = DocumentSuffixTable(docs).approximate_positions_batch(qs, t, metric="edit", bulges=(d, r))
        assert _same(got, want), (i, "DocumentSuffixTable")
        if len(docs) == 1:
            got = SuffixTable(docs[0]).approximate_positions_batch(qs, t, metric="edit", bulges=(d, r))
            assert _same(got, want), (i, "SuffixTable")
    ctx.close()


def test_soft_masked_dna_with_empty_documents_and_ends():
    rng = np.random.default_rng(2)
    base = bytes(b"ACGTACGTacgN"[int(x)] for x in rng.integers(0, 12, 60))
    docs = [base[:20], b"", base[20:45], b"", base[45:]]
    qs = [base[14:20], base[40:45] + b"A", base[45:50].upper(), base[:3], b"ACGTAC"]
    st = DocumentSuffixTable(docs)
    for t, d, r in ((0, 1, 1), (1, 1, 0), (1, 0, 2)):
        want = model_bulges.one_strand(docs, qs, t, d, r)
        assert _same(st.approximate_positions_batch(qs, t, metric="edit", bulges=(d, r)), want)
        assert np.array_equal(st.approximate_counts(qs, t, metric="edit", bulges=(d, r)),
                              np.diff(want[0].astype(np.int64)).astype(np.uint64))
    one = SuffixTable(base)
    want = model_bulges.one_strand([base], qs, 1, 1, 1)
    pos, dist = one.approximate_positions(qs[0], 1, metric="edit", bulges=(1, 1))
    assert np.array_equal(pos, want[1][:int(want[0][1])]) and np.array_equal(dist, want[2][:int(want[0][1])])


def test_every_budget_and_query_length():
    rng = np.random.default_rng(3)
    text = bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, 400))
    docs = [text[:150], text[150:151], text[151:]]
    starts = _starts(docs)
    g = DocumentSuffixTable(docs).table()
    ctx = _lib.Context(0)
    qs = [text[a:a + m] for a, m in ((3, 1), (10, 2), (140, 4), (150, 3), (200, 7), (260, 10), (300, 14), (390, 10))]
    qs += [bytes(q[:x] + q[x + 1:]) for q, x in ((text[50:62], 5), (text[320:335], 9))]       # RNA bulge sites
    qs += [text[70:75] + text[76:85], text[100:106] + b"G" + text[106:114]]                   # DNA bulge, insertion
    for t in (0, 1, 2, 4):
        ham = _fetch(ctx, text, g, qs, t, starts)
        for d in range(4):
            for r in range(4):
                got = _call(ctx, docs, qs, _kf(t, d, r))
                want = bulges_check.bulges(text, starts, qs, t, d, r)
                assert _same(got, want), (t, d, r)
                if d == r == 0:
                    assert _same(got, ham), t                                   # the Hamming call
                edit = _fetch(ctx, text, g, qs, (t + d + r) | EDIT, starts)
                for q in range(len(qs)):
                    e = dict(zip(*[a[int(edit[0][q]):int(edit[0][q + 1])].tolist() for a in edit[1:]]))
                    h = zip(*[a[int(got[0][q]):int(got[0][q + 1])].tolist() for a in got[1:]])
                    assert all(p in e and x >= e[p] for p, x in h), (t, d, r, q)
    ctx.close()


@pytest.mark.parametrize("iupac,fixed", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("strands", ["forward", "both"])
@pytest.mark.parametrize("mode", ["hits", "documents", "align"])
def test_mixes_against_the_model(iupac, fixed, strands, mode):
    rng = np.random.default_rng(4)
    ctx = _lib.Context(0)
    for _ in range(3):
        docs = _docs(rng)
        if not b"".join(docs):
            continue
        qs = _queries(rng, docs, 2)
        if not iupac:
            qs = [bytes(b if b in b"ACGT" else ord("A") for b in q.upper()) for q in qs]
        elif not fixed:
            qs = [q.upper() for q in qs]
        for t, d, r in ((1, 1, 1), (0, 1, 0), (2, 0, 1)):
            want = model_bulges.listing(docs, qs, t, d, r, iupac, fixed, strands, documents=mode == "documents",
                                        align_ops=mode == "align")
            got = _call(ctx, docs, qs, _kf(t, d, r, iupac, fixed, strands, mode))
            assert _same(got, want), (docs, qs, t, d, r)
            if mode == "hits" and not fixed:
                st = DocumentSuffixTable(docs)
                res = st.approximate_positions_batch(qs, t, metric="edit", iupac=iupac, strands=strands,
                                                     bulges=(d, r))
                if strands == "both":
                    res = (res[0], res[1], res[2] | np.where(res[3], np.uint32(MINUS), np.uint32(0)))
                assert _same(res, want)
    ctx.close()


def test_fetch_protocol():
    ctx = _lib.Context(0)
    docs = [b"ACGTACGTTACGTA", b"", b"GGACGTCCA"]
    text, starts = b"".join(docs), _starts(docs)
    g = DocumentSuffixTable(docs).table()
    qs = [b"ACGTA", b"CGTC", b"", b"A"]
    for mode in MODES:
        kf = _kf(1, 1, 1, mode=mode)
        want = model_bulges.listing(docs, qs, 1, 1, 1, documents=mode == "documents", align_ops=mode == "align")
        total = int(want[0][-1])
        assert total > 2, mode
        for cap in (0, 1, total - 1):
            tot, off, pos, dist = _abi(ctx, text, g, qs, kf, cap, starts, buf=total + 5)
            assert tot == total and np.array_equal(off, want[0])
            assert (pos == MARK).all() and (dist == MARK).all(), (mode, cap)
        tot, off, pos, dist = _abi(ctx, text, g, qs, kf, total, starts, buf=total + 5)
        assert tot == total and np.array_equal(off, want[0])
        assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
    ctx.close()


def test_rejections():
    ctx = _lib.Context(0)
    text = b"ACGTACGTACGT"
    sa = SuffixTable(text).table()
    starts = np.array([0], np.uint32)

    def rejected(k, single=False):
        with pytest.raises(_lib.B200SAError) as e:
            if single:
                _abi(ctx, text, sa, [b"ACG"], k, 0)
            else:
                _abi(ctx, text, sa, [b"ACG"], k, 0, starts)
        assert e.value.code == BAD_ARG
        return str(e.value)

    assert "B200SA_APPROX_BULGES" in rejected(1 | BULGES | (1 << 17))                     # without EDIT
    msg = rejected(_kf(1, 1, 1), single=True)                                             # single-text entry
    assert "B200SA_APPROX_BULGES" in msg and "B200SA_APPROX_MAX_K" in msg
    msg = rejected(1 | EDIT | BEST | BULGES | (1 << 17))                                  # with BEST
    assert "B200SA_APPROX_BULGES" in msg and "B200SA_APPROX_BEST" in msg
    assert "B200SA_APPROX_BULGES" in rejected(_kf(26, 3, 3))                              # t + d + r = 32
    for bit in (17, 18, 22, 23):                                                          # a field without the flag
        msg = rejected(1 | EDIT | (1 << bit))
        assert "B200SA_APPROX_MAX_K" in msg and "BULGES" not in msg, bit
    assert _fetch(ctx, text, sa, [b"ACG"], _kf(25, 3, 3), starts)[0][-1] == len(text)   # t + d + r = 31 is fine
    with pytest.raises(ValueError):
        SuffixTable(text).approximate_positions(b"ACG", 1, bulges=(1, 1))
    ctx.close()


def test_one_megabase_against_the_c_statement():
    rng = np.random.default_rng(5)
    text = bytearray(b"ACGT"[int(x)] for x in rng.integers(0, 4, 1 << 20))
    guides = [bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, 20)) for _ in range(200)]
    for i, gd in enumerate(guides[:60]):                                       # plant bulged and mismatched sites
        at = int(rng.integers(0, len(text) - 30))
        x = int(rng.integers(3, 17))
        site = {0: gd[:x] + b"T" + gd[x:], 1: gd[:x] + gd[x + 1:], 2: gd[:x] + b"A" + gd[x + 1:]}[i % 3]
        text[at:at + len(site)] = site
    text = bytes(text)
    st = SuffixTable(text)
    off, pos, dist = st.approximate_positions_batch(guides, 1, metric="edit", bulges=(1, 1))
    assert int(off[-1]) >= 60
    for q0 in (0, 57, 190):                                # the serial statement on a sample of the guides
        o, p, x = bulges_check.bulges(text, None, guides[q0:q0 + 3], 1, 1, 1)
        a, b = int(off[q0]), int(off[q0 + 3])
        assert np.array_equal(o + off[q0], off[q0:q0 + 4]) and np.array_equal(pos[a:b], p) and np.array_equal(dist[a:b], x)


def test_bulge_beside_the_pam():
    guide = b"GACGCTGACGCTGACGTTGA"
    site = guide[:15] + b"C" + guide[15:] + b"TGG"
    text = b"TTTTT" + site + b"AAAAACCCC"
    st = SuffixTable(text)
    q = guide + b"ngg"
    pos, dist = st.approximate_positions(q, 0, metric="edit", iupac=True, fixed=True, bulges=(1, 0))
    assert pos.tolist() == [5] and dist.tolist() == [1]
    assert len(st.approximate_positions(q, 0, metric="edit", iupac=True, fixed=True, bulges=(0, 0))[0]) == 0
    ctx = _lib.Context(0)
    off, p, words = _fetch(ctx, text, st.table(), [q], _kf(0, 1, 0, True, True, mode="align"), np.array([0], np.uint32))
    cig = "".join("%d%s" % (int(w) >> 4, "MIDNSHP=X"[int(w) & 15]) for w in words)
    assert cig == "15=1D8=", cig
    ctx.close()
