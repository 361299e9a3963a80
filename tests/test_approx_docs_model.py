"""The approximate document listing (tests/model_approx_docs.py) against the hit lists it reduces: the stated
consequences of include/b200sa.h (B200SA_APPROX_DOCUMENTS) exhaustively over small collections with empty and
one-byte documents, queries longer than every document, ties between the strands and best= cut at the global
t(q); the device's mark-scan-minimum rule; and the Python argument checks.  CPU only."""
import itertools

import numpy as np
import pytest

from suffix_b200 import _approx
from tests import model_approx_docs, model_best, model_strand

METRICS = ("hamming", "edit")
MINUS = model_strand.MINUS
MIXES = [(metric, iupac, best, strands) for metric in METRICS for iupac in (False, True) for best in (None, 1)
         for strands in ("forward", "both")]


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _collections():
    """Every collection of at most three documents over {"", "A", "C", "G", "T", "AC", "GT"}, and a few longer ones
    with N, soft-masked bases and other bytes, empty documents among them."""
    pieces = [b"", b"A", b"C", b"G", b"T", b"AC", b"GT"]
    out = [list(c) for m in (1, 2, 3) for c in itertools.product(pieces, repeat=m)]
    out += [[b"ACGTNACGT", b"", b"GAATTCaattc"], [b"TTGCAxAC", b"A", b"", b"AAGGTTCCAGT"], [b"NNNN", b"acgtACGT"],
            [b"GAATTC", b"GAATTC", b"", b"C"]]
    return out


PLAIN_QS = [b"", b"A", b"AC", b"GT", b"ACG", b"ACGT", b"GAATTC", b"TTG", b"aC", b"AxT", b"CCAGTTGCAAGT"]
IUPAC_QS = [b"", b"A", b"NG", b"RY", b"ACN", b"GAATTC", b"TTGa", b"MKu", b"BD", b"ACGT", b"NNNNNNNNNNNNN"]


def _check(docs, qs, k, metric, iupac, best, strands):
    starts = model_approx_docs.starts_of(docs)
    hits = model_approx_docs.flagless(docs, qs, k, metric, iupac, best, strands)
    got = model_approx_docs.brute(docs, qs, k, metric, iupac, best, strands)
    assert _same(got, model_approx_docs.group(hits, starts)), (docs, k)
    hit_off, got_off = hits[0].astype(np.int64), got[0].astype(np.int64)
    assert (np.diff(got_off) <= np.diff(hit_off)).all()                          # documents <= hits
    for q, h, listed in zip(qs, model_best.lists(hits), model_best.lists(got)):
        ds = [d for d, _ in listed]
        assert ds == sorted(set(ds))                                             # ascending, distinct
        assert all(docs[d] for d in ds)                                          # empty documents never listed
        assert set(ds) == {model_approx_docs.doc_of(starts, p) for p, _ in h}
        for d, w in listed:
            mine = [e for p, e in h if model_approx_docs.doc_of(starts, p) == d]
            least = min(e & (MINUS - 1) for e in mine)
            assert w & (MINUS - 1) == least
            plus_reaches = any(e == least for e in mine)                         # a + entry at the least distance
            assert bool(w & MINUS) == (not plus_reaches), (docs, q, d)
        if strands == "both" and model_strand.revcomp(q, iupac) == q:            # a palindrome: never MINUS
            assert all(w < MINUS for _, w in listed), (docs, q)
        if len(q) > max(len(d) for d in docs) + k:                              # longer than every document
            assert listed == []
    if k == 0 and metric == "hamming" and strands == "forward" and not iupac:
        for q, listed in zip(qs, model_best.lists(got)):                        # the exact documents
            want = [d for d, x in enumerate(docs) if q and q in x]
            assert listed == [(d, 0) for d in want], (docs, q)


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_stated_consequences(metric, iupac, best, strands):
    qs = IUPAC_QS if iupac else PLAIN_QS
    for docs in _collections():
        for k in (0, 1, 2):
            _check(docs, qs, k, metric, iupac, best, strands)


def test_ties_between_strands():
    q = b"AACCGGTTAC"
    rc = model_strand.revcomp(q)
    near = bytearray(q)
    near[3] ^= 0x02                                                    # the plus hit at d = 1
    docs = [b"TTTT" + rc + b"GG",                                      # a minus hit at 0 only
            b"GG" + bytes(near) + b"TT" + model_strand.revcomp(bytes(near)),   # + and - both at 1: + wins the tie
            b"CC" + bytes(near) + b"A" + rc,                           # + at 1, - at 0
            b"", b"AC" + q]                                            # + at 0
    for metric in METRICS:
        off, ds, dist = model_approx_docs.brute(docs, [q], 2, metric, strands="both")
        got = list(zip(ds.tolist(), dist.tolist()))
        assert got[:3] == [(0, MINUS), (1, 1), (2, MINUS)] and got[-1] == (4, 0), (metric, got)
        fw = model_approx_docs.brute(docs, [q], 2, metric)
        assert fw[1].tolist()[:1] == [0] and fw[2].tolist()[0] > 0 and all(d < MINUS for d in fw[2].tolist())


def test_best_cuts_at_the_global_threshold():
    q = b"ACGTACGTTG"
    one = bytearray(q)
    one[4] = ord("G")
    two = bytearray(one)
    two[8] = ord("A")
    docs = [b"TT" + bytes(two) + b"TT", b"GG" + q + b"CC", b"CC" + bytes(one) + b"AA", b"T" * 12]
    for metric in METRICS:
        full = model_best.lists(model_approx_docs.brute(docs, [q], 2, metric))[0]
        assert [d for d, _ in full] == [0, 1, 2], (metric, full)
        zero = model_best.lists(model_approx_docs.brute(docs, [q], 2, metric, best=0))[0]
        assert zero == [(1, 0)], metric                                # best(q) = 0 over the collection
        slack1 = model_best.lists(model_approx_docs.brute(docs, [q], 2, metric, best=1))[0]
        assert [d for d, _ in slack1] == [1, 2], metric                # document 0 holds nothing within t(q) = 1
        no_exact = [docs[0], docs[2], docs[3]]
        zero = model_best.lists(model_approx_docs.brute(no_exact, [q], 2, metric, best=0))[0]
        assert zero == [(1, 1)], metric                                # best(q) = 1: only the d = 1 document


def test_one_byte_documents_and_long_queries():
    docs = [b"A", b"", b"C", b"A", b"G", b"T", b""]
    for metric in METRICS:
        for k in (0, 1, 2):
            _check(docs, [b"A", b"AC", b"ACGT", b"N", b""], k, metric, False, None, "both")
            _check(docs, [b"N", b"NN", b"R"], k, metric, True, None, "forward")
        one = model_best.lists(model_approx_docs.brute(docs, [b"A"], 0, metric))[0]
        assert one == [(0, 0), (3, 0)]


@pytest.mark.parametrize("metric,iupac,best,strands", MIXES)
def test_device_rule_equals_the_definition(metric, iupac, best, strands):
    rng = np.random.default_rng(MIXES.index((metric, iupac, best, strands)))
    qs = IUPAC_QS if iupac else PLAIN_QS
    for docs in _collections()[::7]:
        for k in (0, 2):
            starts = model_approx_docs.starts_of(docs)
            hits = model_approx_docs.flagless(docs, qs, k, metric, iupac, best, strands)
            assert _same(model_approx_docs.device_rule(hits, starts),
                         model_approx_docs.brute(docs, qs, k, metric, iupac, best, strands)), (docs, k)
    text = bytes(rng.choice(list(b"ACGT"), 600).tolist())
    cuts = sorted(set(rng.integers(0, 600, 40).tolist()))
    docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [600])]
    qs = [text[a:a + 9] for a in rng.integers(0, 590, 8).tolist()]
    hits = model_approx_docs.flagless(docs, qs, 2, metric, iupac, best, strands)
    assert _same(model_approx_docs.device_rule(hits, model_approx_docs.starts_of(docs)),
                 model_approx_docs.brute(docs, qs, 2, metric, iupac, best, strands))


class _NoTable:
    """A stand-in that fails if the call gets past its argument checks."""

    def __len__(self):
        raise AssertionError("the argument checks let the call through")

    def _bwt_arrays(self):
        raise AssertionError("the argument checks let the call through")


@pytest.mark.parametrize("fn", [_approx.documents, _approx.documents_batch, _approx.document_frequencies])
def test_argument_checks(fn):
    assert _approx.DOCUMENTS == 0x20000000
    q = b"ACG" if fn is _approx.documents else [b"ACG"]
    for kw in (dict(k=32), dict(k=-1), dict(k=1, metric="levenshtein"), dict(k=1, best=True), dict(k=1, best=32),
               dict(k=1, best=-1), dict(k=1, best=1.0), dict(k=1, iupac=1), dict(k=1, iupac="yes"),
               dict(k=1, strands="Both"), dict(k=1, strands=None)):
        kw = dict(kw)
        k = kw.pop("k")
        with pytest.raises(ValueError):
            fn(_NoTable(), q, k, **kw)


def test_methods_on_document_tables_only():
    import inspect

    from suffix_b200 import DocumentSuffixTable, SuffixTable
    for name in ("approximate_documents", "approximate_documents_batch", "approximate_document_frequencies"):
        sig = inspect.signature(getattr(DocumentSuffixTable, name))
        assert [p for p in sig.parameters if sig.parameters[p].kind == inspect.Parameter.KEYWORD_ONLY] == \
            ["metric", "best", "iupac", "strands"], name
        assert not hasattr(SuffixTable, name)
