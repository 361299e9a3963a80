"""The alignments of approximate hits (B200SA_APPROX_ALIGN) on the host: the stated properties of every hit's
operations on small collections of DNA and of bytes with documents, the band lemma (the full-DP walk equals the
banded walk the device runs), the walk's cost against tests/model_edit.py and the Hamming count, hand-made cases
with known CIGARs, the host's recovery of hits from an operation listing, and the Python argument checks."""
import itertools

import numpy as np
import pytest

from suffix_b200 import _approx, cigar_string
from tests import model_align, model_approx, model_approx_docs, model_edit, model_strand

MINUS = model_strand.MINUS
MIXES = [(metric, iupac, best, strands) for metric in ("hamming", "edit") for iupac in (False, True)
         for best in (None, 0, 1) for strands in ("forward", "both")]
PLAIN_QS = [b"", b"A", b"AC", b"GT", b"ACG", b"ACGT", b"GAATTC", b"TTG", b"aC", b"AxT", b"CCAGTTGCAAGT"]
IUPAC_QS = [b"", b"A", b"NG", b"RY", b"ACN", b"GAATTC", b"TTGa", b"MKu", b"BD", b"ACGT", b"NNNNNNNNNNNNN"]


def _collections(rng):
    pieces = [b"", b"A", b"C", b"G", b"T", b"AC", b"GT"]
    out = [list(c) for m in (1, 2) for c in itertools.product(pieces, repeat=m)]
    out += [[b"ACGTNACGT", b"", b"GAATTCaattc"], [b"TTGCAxAC", b"A", b"", b"AAGGTTCCAGT"], [b"NNNN", b"acgtACGT"]]
    for _ in range(6):                                              # random DNA in documents, some empty
        out.append([bytes(rng.choice(list(b"ACGT"), int(rng.integers(0, 40)))) for _ in range(int(rng.integers(1, 5)))])
    for _ in range(4):                                              # bytes
        out.append([bytes(rng.integers(0, 4, int(rng.integers(0, 30))).astype(np.uint8)) for _ in range(3)])
    return out


def _queries(rng, docs, iupac):
    qs = list(IUPAC_QS if iupac else PLAIN_QS)
    text = b"".join(docs)
    for _ in range(3):
        if len(text) > 3:
            a = int(rng.integers(0, len(text) - 3))
            q = bytearray(text[a:a + int(rng.integers(3, 15))])
            if iupac:
                q = bytearray(b if b in b"ACGT" else ord("N") for b in q)
            qs.append(bytes(q))
    return qs


def _hits(docs, qs, k, metric, iupac, best, strands):
    return model_approx_docs.flagless(docs, qs, k, metric, iupac, best, strands)


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_properties_and_band_lemma(metric, iupac, best, strands):
    rng = np.random.default_rng(500 + MIXES.index((metric, iupac, best, strands)))
    for i, docs in enumerate(_collections(rng)):
        k = [0, 1, 2, 3][i % 4]
        qs = _queries(rng, docs, iupac)
        text = b"".join(docs)
        starts = model_approx_docs.starts_of(docs)
        ends = model_approx._ends(starts, len(text))
        off, pos, dist = _hits(docs, qs, k, metric, iupac, best, strands)
        for qi, q in enumerate(qs):
            for i in range(int(off[qi]), int(off[qi + 1])):
                p, d = int(pos[i]), int(dist[i])
                minus, d = d >= MINUS, d & (MINUS - 1)
                E = ends[model_approx_docs.doc_of(starts, p)]
                ops, end = model_align.align(text, E, p, q, d, metric, iupac, minus)
                lens = {c: sum(n for cc, n in ops if cc == c) for c in (1, 2, 7, 8)}
                assert lens[8] + lens[1] + lens[2] == d, (docs, q, p)
                assert lens[7] + lens[8] + lens[1] == len(q)
                assert lens[7] + lens[8] + lens[2] == end - p
                assert end <= E and ops[-1][0] != model_align.D and len(ops) <= 2 * d + 1
                assert all(a[0] != b[0] for a, b in zip(ops, ops[1:]))            # merged
                if metric == "edit":                                           # the band lemma
                    assert model_align.align(text, E, p, q, d, metric, iupac, minus, banded=True) == (ops, end)


def test_cost_equals_the_distance():
    rng = np.random.default_rng(520)
    for _ in range(40):
        docs = [bytes(rng.choice(list(b"ACGT"), int(rng.integers(1, 30)))) for _ in range(int(rng.integers(1, 4)))]
        text = b"".join(docs)
        qs = [bytes(rng.choice(list(b"ACGT"), int(rng.integers(1, 9)))) for _ in range(4)]
        starts = model_approx_docs.starts_of(docs)
        ends = model_approx._ends(starts, len(text))
        for metric, brute in (("edit", model_edit.brute), ("hamming", model_approx.brute)):
            off, pos, dist = brute(docs, qs, 3)
            for qi, q in enumerate(qs):
                for i in range(int(off[qi]), int(off[qi + 1])):
                    p = int(pos[i])
                    E = ends[model_approx_docs.doc_of(starts, p)]
                    ops, end = model_align.align(text, E, p, q, int(dist[i]), metric)
                    cost = sum(n for c, n in ops if c != model_align.EQ)
                    assert cost == int(dist[i])
                    if metric == "edit":
                        assert cost == model_edit.levenshtein(q, text[p:end])
                    else:
                        assert cost == model_approx.hamming(text[p:end], q)


def _one(text, p, q, d, metric="edit", E=None, **kw):
    ops, end = model_align.align(text, len(text) if E is None else E, p, q, d, metric, **kw)
    return model_align.cigar(ops), end


def test_hand_made_cigars():
    t = b"TTTTACGTACGTTTTT"
    assert _one(t, 4, b"ACGAACGT", 1, "hamming") == ("3=1X4=", 12)
    assert _one(t, 4, b"ACGAACGT", 1) == ("3=1X4=", 12)                    # a substitution
    assert _one(t, 4, b"ACGTCCGT", 1) == ("4=1X3=", 12)
    # an insertion: the walk prefers the diagonal, so of the equal places for the extra A it takes the last
    assert _one(t, 4, b"ACGTAACGT", 1) == ("5=1I3=", 12)
    assert _one(t, 4, b"ACGTAGCGT", 1) == ("5=1I3=", 12)
    assert _one(t, 4, b"ACGACGT", 1) == ("3=1D4=", 12)                     # a deletion
    # an exact hit at 4 puts 3 and 5 at distance 1: a leading D, or a leading I
    assert _one(t, 3, b"ACGTACGT", 1) == ("1D8=", 12)
    assert _one(t, 5, b"ACGTACGT", 1) == ("1I7=", 12)
    assert _one(b"ACGTAC", 2, b"GTACG", 1) == ("4=1I", 6)                  # cut by the document end
    assert _one(b"ACGTACxx", 2, b"GTACG", 1, E=6) == ("4=1I", 6)
    assert _one(b"ACGT", 1, b"GG", 2, "hamming") == ("1X1=", 3)
    # m <= k: the whole query against the text, or m insertions when no byte matches
    assert _one(b"ACGT", 2, b"GT", 0) == ("2=", 4)
    assert _one(b"AAAA", 0, b"CC", 2) == ("2X", 2)
    assert _one(b"AAAA", 3, b"CC", 2) == ("1X1I", 4)
    assert _one(b"AAAA", 3, b"CCC", 3) == ("1X2I", 4)
    assert _one(b"T", 0, b"GG", 2) == ("1X1I", 1)
    assert _one(b"ACGTAC", 5, b"GG", 2) == ("1X1I", 6)
    assert _one(b"AC", 1, b"GG", 2, E=2) == ("1X1I", 2)
    # minus hits: rc(q) against the text, in text order
    assert _one(t, 4, model_strand.revcomp(b"ACGTACGT"), 0, minus=True) == ("8=", 12)
    assert _one(t, 4, b"NCGT", 0, "hamming", iupac=True) == ("4=", 8)
    assert _one(t, 4, b"ACGN", 0, iupac=True, minus=True) == ("4=", 8)      # rc(ACGN) = NCGT
    assert _one(t, 4, b"ACGTACGG", 1, "hamming", minus=True) == ("1X7=", 12)  # rc = CCGTACGT


def test_insertions_only_alignment():
    # D(x, E) = m - x: at the document end only insertions remain, so an empty text aligns as mI.  A hit has
    # p < E, and there the last query byte takes the diagonal (cost at most 1), so a hit always has = or X.
    ops, end = model_align.align(b"AC", 2, 1, b"GG", 2, "edit")
    assert model_align.cigar(ops) == "1X1I" and end == 2
    mis = model_align.mismatch(b"", b"GGG")
    moves, u = model_align.walk(lambda x, uu: int(model_align.full_dp(mis)[x, uu]), mis)
    assert model_align.cigar(model_align.merge(moves)) == "3I" and u == 0


def test_bam_words_and_cigar_string():
    ops = [(model_align.EQ, 12), (model_align.X, 1), (model_align.EQ, 7), (model_align.I, 1), (model_align.EQ, 2)]
    w = model_align.words(ops)
    assert w == [12 << 4 | 7, 1 << 4 | 8, 7 << 4 | 7, 1 << 4 | 1, 2 << 4 | 7]
    assert cigar_string(w) == model_align.cigar(ops) == "12=1X7=1I2="
    assert cigar_string(model_align.words(ops, minus=True)) == "12=1X7=1I2="
    assert cigar_string([3 << 4 | 2]) == "3D" and cigar_string([]) == ""


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES[::3])
def test_hits_recovered_from_the_listing(metric, iupac, best, strands):
    """_approx._hits turns the listing back into the hits of the call without the flag, distances and ends
    included, and the cigar offsets into each hit's words."""
    rng = np.random.default_rng(530)
    for docs in _collections(rng)[-10:]:
        qs = _queries(rng, docs, iupac)
        for k in (1, 3):
            off, pos, w = model_align.listing(docs, qs, k, metric, iupac, best, strands)
            hoff, p, dist, minus, ends, coff, cig = _approx._hits(off, pos, np.asarray(w, np.uint32))
            want = _hits(docs, qs, k, metric, iupac, best, strands)
            assert np.array_equal(hoff, want[0]) and np.array_equal(p, want[1])
            assert np.array_equal(dist | np.where(minus, np.uint32(MINUS), np.uint32(0)), want[2])
            assert not (cig & MINUS).any() and coff[-1] == len(w) and (np.diff(coff.astype(np.int64)) > 0).all()
            assert (ends >= p).all()


def test_listing_of_plain_hits_is_one_op_per_run():
    off, pos, w = model_align.listing([b"ACGTACGT"], [b"ACGT", b"AxGT"], 1)
    assert off.tolist() == [0, 2, 8]
    assert pos.tolist() == [0, 4, 0, 0, 0, 4, 4, 4]
    assert [cigar_string([x]) for x in w] == ["4=", "4=", "1=", "1X", "2=", "1=", "1X", "2="]


class _NoTable:
    _device = 0

    def __len__(self):
        raise AssertionError("the argument checks let the call through")

    def _bwt_arrays(self):
        raise AssertionError("the argument checks let the call through")


@pytest.mark.parametrize("fn", [_approx.alignments, _approx.alignments_batch])
def test_argument_checks(fn):
    assert _approx.ALIGN == 0x8000000
    q = b"ACG" if fn is _approx.alignments else [b"ACG"]
    for kw in (dict(k=32), dict(k=-1), dict(k=1, metric="levenshtein"), dict(k=1, best=True), dict(k=1, best=32),
               dict(k=1, iupac=1), dict(k=1, strands="Both")):
        kw = dict(kw)
        k = kw.pop("k")
        with pytest.raises(ValueError):
            fn(_NoTable(), q, k, **kw)


def test_methods_on_both_tables():
    import inspect

    from suffix_b200 import DocumentSuffixTable, SuffixTable
    for cls in (SuffixTable, DocumentSuffixTable):
        for name in ("approximate_alignments", "approximate_alignments_batch"):
            sig = inspect.signature(getattr(cls, name))
            assert [p for p in sig.parameters if sig.parameters[p].kind == inspect.Parameter.KEYWORD_ONLY] == \
                ["metric", "best", "iupac", "strands"], name


@pytest.mark.parametrize("metric,iupac,strands", [(m, i, s) for m in ("hamming", "edit") for i in (False, True)
                                                  for s in ("forward", "both")])
def test_serial_c_statement_equals_model(metric, iupac, strands):
    from tests import align_check
    rng = np.random.default_rng(540)
    for docs in _collections(rng)[-10:]:
        qs = _queries(rng, docs, iupac)
        text = b"".join(docs)
        for k in (1, 3):
            off, pos, dist = _hits(docs, qs, k, metric, iupac, None, strands)
            want = model_align.listing(docs, qs, k, metric, iupac, None, strands)
            hq = np.repeat(np.arange(len(qs)), np.diff(off.astype(np.int64)))
            cnt, w = align_check.align_hits(text, model_approx_docs.starts_of(docs), qs, hq, pos, dist,
                                            metric == "edit", iupac)
            assert np.array_equal(w, want[2]) and int(cnt.sum()) == len(want[2]), (docs, k)
