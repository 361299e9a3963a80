"""One hit per locus (B200SA_APPROX_LOCI on b200sa_docs_approx_positions_dev, loci= on the approximate_positions*
and approximate_counts methods): against tests/model_loci.py applied to the listings of the existing models, for
every mix of the edit metric, best hits, IUPAC, fixed symbols, both strands and bulges, on families with empty
documents; the count against the fetch; alignments against the plain alignment listing cut to the kept hits; the
rejections; a chain as long as the text; a periodic text; and 1 MB of DNA against the serial C statements."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import (bulges_check, edit_check, fixed_check, model_approx_docs, model_bulges, model_fixed, model_loci,
                   model_strand)
from tests.test_fixed_model import _docs as _fixed_docs
from tests.test_fixed_model import _queries as _fixed_queries
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_iupac import _masked_dna
from tests.test_gpu_iupac import _queries as _iupac_queries
from tests.test_gpu_strand import _dna_queries

pytestmark = pytest.mark.gpu

BAD_ARG = -1
LOCI = 0x80                                     # B200SA_APPROX_LOCI
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
BULGES = 0x200000                               # B200SA_APPROX_BULGES
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
FIXED = 0x2000000                               # B200SA_APPROX_FIXED
ALIGN = 0x8000000                               # B200SA_APPROX_ALIGN
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
DOCS = 0x20000000                               # B200SA_APPROX_DOCUMENTS
MINUS = model_strand.MINUS

# (metric, iupac, fixed, best, strands, bulges)
MIXES = ([(metric, iupac, False, best, strands, None) for metric in ("hamming", "edit") for iupac in (False, True)
          for best in (None, 1) for strands in ("forward", "both")] +
         [(metric, True, True, best, strands, None) for metric in ("hamming", "edit") for best in (None, 0)
          for strands in ("forward", "both")] +
         [("edit", iupac, fixed, None, strands, (1, 1)) for iupac, fixed in ((False, False), (True, False), (True, True))
          for strands in ("forward", "both")])


def _kf(k, metric, iupac, fixed, best, strands, bulges, loci=True):
    kf = (k | (EDIT if metric == "edit" else 0) | (IUPAC if iupac else 0) | (FIXED if fixed else 0) |
          (0 if best is None else (best << 8) | BEST) | (BOTH if strands == "both" else 0) | (LOCI if loci else 0))
    if bulges is not None:
        kf |= BULGES | (bulges[0] << 17) | (bulges[1] << 22)
    return kf


def _plain(docs, qs, k, metric, iupac, fixed, best, strands, bulges):
    """L(q): the model listing of the call without the flag."""
    if bulges is not None:
        return model_bulges.flagless(docs, qs, k, bulges[0], bulges[1], iupac, fixed, strands)
    if fixed:
        return model_fixed.flagless(docs, qs, k, metric, best, strands)
    return model_approx_docs.flagless(docs, qs, k, metric, iupac, best, strands)


def _queries(rng, docs, k, iupac, fixed):
    if fixed:
        return _fixed_queries(rng, docs, k)
    if iupac:
        return [q.upper() for q in _iupac_queries(rng, docs, k)]
    text = b"".join(docs)
    return _dna_queries(rng, docs, k) + [text[:6], text[2:9]]


def _packed(res, strands):
    """(offsets, pos, d | MINUS) of what a method returns for strands=."""
    if strands == "forward":
        return res
    off, pos, dist, minus = res
    return off, pos, dist | np.where(minus, np.uint32(MINUS), np.uint32(0))


def _sets(rng, mix):
    metric, iupac, fixed, best, strands, bulges = mix
    if fixed or bulges is not None:                  # the bulge model is slow: small collections only
        return [_fixed_docs(rng) for _ in range(6)] + [[_masked_dna(rng, 60).upper(), b"", _masked_dna(rng, 30)]]
    dna = [[_u8(gen.dna(int(rng.integers(1, 80)), seed=int(rng.integers(1, 1 << 30)))) for _ in range(3)]
           for _ in range(4)]
    return ([s for s in _families(rng)[::25] if b"".join(s)] + dna +
            [[_masked_dna(rng, 70), b"", _masked_dna(rng, 40), b""]])


@pytest.mark.parametrize("mix", MIXES, ids=lambda m: "-".join(str(x) for x in m))
def test_mixes_against_the_model(mix):
    metric, iupac, fixed, best, strands, bulges = mix
    rng = np.random.default_rng(7000 + MIXES.index(mix))
    ctx = _lib.Context(0)
    kw = dict(metric=metric, iupac=iupac, fixed=fixed, best=best, strands=strands, bulges=bulges)
    for i, docs in enumerate(_sets(rng, mix)):
        k = [1, 2, 0, 3][i % 4] if bulges is None else [0, 1][i % 2]
        qs = _queries(rng, docs, k, iupac, fixed)
        text, starts = b"".join(docs), model_approx_docs.starts_of(docs).astype(np.uint32)
        g = DocumentSuffixTable(docs).table()
        want = model_loci.collapse(_plain(docs, qs, k, metric, iupac, fixed, best, strands, bulges), qs, starts)
        got = _fetch(ctx, text, g, qs, _kf(k, metric, iupac, fixed, best, strands, bulges), starts)
        assert _same(got, want), (docs, qs, k)
        plain = _fetch(ctx, text, g, qs, _kf(k, metric, iupac, fixed, best, strands, bulges, loci=False), starts)
        assert _same(model_loci.collapse(plain, qs, starts), want), (docs, qs, k)       # the device's own L(q)
        st = DocumentSuffixTable(docs)
        assert _same(_packed(st.approximate_positions_batch(qs, k, loci=True, **kw), strands), want), (docs, k)
        cnt = st.approximate_counts(qs, k, loci=True, **kw)
        assert cnt.dtype == np.uint64 and np.array_equal(cnt, np.diff(want[0].astype(np.int64))), (docs, k)
        if len(docs) == 1:
            one = SuffixTable(docs[0])
            assert _same(_packed(one.approximate_positions_batch(qs, k, loci=True, **kw), strands), want), docs
            a, b = int(want[0][-2]), int(want[0][-1])
            res = one.approximate_positions(qs[-1], k, loci=True, **kw)
            assert _same(_packed((None,) + tuple(res), strands)[1:], (want[1][a:b], want[2][a:b])), docs
    ctx.close()


def test_count_and_fetch_protocol():
    ctx = _lib.Context(0)
    docs = [b"ACGTACGTTACGTAACGTA", b"", b"GGACGTCCACGTA"]
    text, starts = b"".join(docs), model_approx_docs.starts_of(docs).astype(np.uint32)
    g = DocumentSuffixTable(docs).table()
    qs = [b"ACGTA", b"CGTC", b"", b"A", b"TACGT"]
    for kf in (1 | EDIT | LOCI, 1 | EDIT | BOTH | LOCI, 2 | EDIT | BEST | LOCI, 0 | EDIT | BULGES | (1 << 17) | LOCI):
        want = _fetch(ctx, text, g, qs, kf, starts)                           # asserts the count call's total
        total = int(want[0][-1])
        assert total > 2 and total == len(want[1]), hex(kf)
        for cap in (0, 1, total - 1):                                        # offsets only
            tot, off, pos, dist = _abi(ctx, text, g, qs, kf, cap, starts, buf=total + 5)
            assert tot == total and np.array_equal(off, want[0])
            assert (pos == MARK).all() and (dist == MARK).all(), (hex(kf), cap)
        tot, off, pos, dist = _abi(ctx, text, g, qs, kf, total, starts, buf=total + 5)
        assert tot == total and np.array_equal(off, want[0])
        assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
        tot, off, pos, _ = _abi(ctx, text, g, qs, kf, total + 5, starts, with_mis=False, buf=total + 5)
        assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all()
    for empty_starts in ([0], [0, 0, 0]):                                    # n = 0 and nq = 0
        tot, off, _, _ = _abi(ctx, b"", [], [b"AC", b""], 1 | EDIT | LOCI, 4, np.array(empty_starts, np.uint32))
        assert tot == 0 and off.tolist() == [0, 0, 0]
    tot, off, _, _ = _abi(ctx, text, g, [], 1 | EDIT | LOCI, 0, starts)
    assert tot == 0 and off.tolist() == [0]
    ctx.close()


@pytest.mark.parametrize("kf", [2 | EDIT, 1, 1 | EDIT | BOTH, 2 | EDIT | BEST | (1 << 8) | BOTH,
                                1 | EDIT | BULGES | (1 << 17) | (1 << 22) | BOTH,
                                1 | EDIT | IUPAC | FIXED | BOTH], ids=hex)
def test_alignments_are_the_kept_hits_words(kf):
    rng = np.random.default_rng(7100)
    docs = [_masked_dna(rng, 400).upper(), b"", _masked_dna(rng, 250).upper()]
    text, starts = b"".join(docs), model_approx_docs.starts_of(docs).astype(np.uint32)
    g = DocumentSuffixTable(docs).table()
    up = text.replace(b"N", b"A").replace(b"U", b"C")
    qs = [up[a:a + 12] for a in rng.integers(0, len(up) - 12, 20).tolist()] + [b"", b"ACGTn", up[5:25] + b"ngg"]
    if not kf & IUPAC:
        qs = [bytes(b if b in b"ACGT" else 65 for b in q.upper()) for q in qs]
    ctx = _lib.Context(0)
    kept = _fetch(ctx, text, g, qs, kf | LOCI, starts)
    plain_ops = _fetch(ctx, text, g, qs, kf | ALIGN, starts)
    got = _fetch(ctx, text, g, qs, kf | ALIGN | LOCI, starts)
    assert int(kept[0][-1]) >= 20
    assert _same(got, model_loci.keep_ops(plain_ops, kept))
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

    for extra in (0, EDIT, BOTH, EDIT | BEST | (1 << 8)):
        msg = rejected(1 | LOCI | DOCS | extra)
        assert "B200SA_APPROX_LOCI" in msg and "B200SA_APPROX_DOCUMENTS" in msg, hex(extra)
    for extra in (0, EDIT, BOTH, EDIT | IUPAC):                              # bit 7 is a threshold bit there
        assert "k above B200SA_APPROX_MAX_K" in rejected(1 | LOCI | extra, single=True), hex(extra)
    for k in (32 | LOCI, 0x60 | LOCI | EDIT, (1 << 8) | LOCI):               # other threshold bits still count
        assert "k above B200SA_APPROX_MAX_K" in rejected(k), hex(k)
    for k in (32 | LOCI | BEST, 0x7F | LOCI | BEST, 1 | LOCI | BEST | (32 << 8)):
        assert "B200SA_APPROX_MAX_K" in rejected(k), hex(k)
    msg = rejected(1 | LOCI | (1 << 19))                                     # an unknown bit beside the flag
    assert all(w in msg for w in ("B200SA_APPROX_MAX_K", "B200SA_APPROX_DOCUMENTS", "B200SA_APPROX_LOCI")), msg
    assert _fetch(ctx, text, sa, [b"ACG"], 31 | LOCI | EDIT, starts)[0][-1] == 1      # threshold 31 is fine
    assert _fetch(ctx, text, sa, [b"ACG"], 31 | LOCI | EDIT | BEST | (31 << 8), starts)[0][-1] == 1
    for bad in (1, 0, None, "True", 1.0):
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_positions(b"ACG", 1, loci=bad)
        with pytest.raises(ValueError):
            DocumentSuffixTable([text]).approximate_counts([b"ACG"], 1, metric="edit", loci=bad)
    ctx.close()


def test_chain_as_long_as_the_text():
    text = b"A" * 200_000
    st = SuffixTable(text)
    q = b"A" * 20
    pos, dist, minus = st.approximate_positions(q, 2, metric="edit", strands="both", loci=True)
    assert pos.tolist() == [0] and dist.tolist() == [0] and minus.tolist() == [False]
    assert st.approximate_counts([q, b"T" * 20], 2, metric="edit", strands="both", loci=True).tolist() == [1, 1]
    off, pos, dist, minus = st.approximate_positions_batch([q, b"T" * 20], 2, metric="edit", strands="both", loci=True)
    assert pos.tolist() == [0, 0] and dist.tolist() == [0, 0] and minus.tolist() == [False, True]
    docs = DocumentSuffixTable([text[:100_000], text[100_000:]])                     # one locus per document
    assert docs.approximate_positions(q, 2, metric="edit", loci=True)[0].tolist() == [0, 100_000]


def test_periodic_text_under_hamming():
    text = b"ACG" * 10_000 + b"T" * 50 + b"ACG" * 100
    st = SuffixTable(text)
    pos, dist = st.approximate_positions(b"ACGACG", 0, loci=True)
    assert pos.tolist() == [0, 30_050] and dist.tolist() == [0, 0]
    for k in (1, 2):
        for q in (b"ACGACG", b"ACGTCG", b"CGACGA"):
            plain = st.approximate_positions_batch([q], k)
            got = st.approximate_positions_batch([q], k, loci=True)
            assert _same(got, model_loci.collapse(plain, [q])), (k, q)
    pos, _ = st.approximate_positions(b"ACG", 0, loci=True)                           # starts 3 apart: no merging
    assert len(pos) == 10_100


def test_one_megabase_against_the_c_statements():
    rng = np.random.default_rng(7200)
    t = gen.dna(1 << 20)
    text = _u8(t)
    guides, sites = [], rng.integers(0, len(text) - 30, 150).tolist()
    for a in sites:                                                                # sites with a substitution
        g = bytearray(text[a:a + 20])
        g[int(rng.integers(0, 20))] = b"ACGT"[int(rng.integers(0, 4))]
        guides.append(bytes(g))
    guides += [bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, 20)) for _ in range(50)]
    cuts = np.unique(rng.integers(1, len(text), 300))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(text)])]
    one, many = SuffixTable(text), DocumentSuffixTable(docs)
    for st, s in ((one, None), (many, starts)):
        want = model_loci.collapse(edit_check.edit(text, s, guides, 2), guides, s)
        assert int(want[0][-1]) >= 140                                             # a site may cross a cut
        assert _same(st.approximate_positions_batch(guides, 2, metric="edit", loci=True), want)
        assert np.array_equal(st.approximate_counts(guides, 2, metric="edit", loci=True),
                              np.diff(want[0].astype(np.int64)))
    pam = [g + text[a + 20:a + 23].lower() for g, a in zip(guides[:6], sites)]           # the site's own PAM, fixed
    want = model_loci.collapse(fixed_check.fixed(text, None, pam, 2, "edit"), pam)
    assert int(want[0][-1]) >= 6
    assert _same(one.approximate_positions_batch(pam, 2, metric="edit", iupac=True, fixed=True, loci=True), want)
    sample = guides[:3] + guides[-2:]
    want = model_loci.collapse(bulges_check.bulges(text, starts, sample, 1, 1, 1), sample, starts)
    assert _same(many.approximate_positions_batch(sample, 1, metric="edit", bulges=(1, 1), loci=True), want)
