"""The host statement of one hit per locus (tests/model_loci.py): hand cases of the definition (a planted site under
the edit metric, m = 1, transitive chains, document ends, strands, ties), its stated properties on the listings of
the existing models (a subset at equal distances, collapsing twice equals collapsing once, nothing merges when the
hits are at least m apart), and the keyword checks, which fail before any device work.  CPU only."""
import inspect

import numpy as np
import pytest

from suffix_b200 import _approx
from tests import model_approx, model_approx_docs, model_best, model_bulges, model_edit, model_fixed, model_loci
from tests import model_strand
from tests.test_fixed_model import _docs, _queries

MINUS = model_loci.MINUS


def _pack(lists):
    return model_approx._pack(lists)


def _lists(packed):
    return model_best.lists(packed)


def _dna(rng, n):
    return bytes(b"ACGT"[int(x)] for x in rng.integers(0, 4, n))


def test_planted_exact_site_under_edit_collapses_to_its_start():
    rng = np.random.default_rng(1)
    q = _dna(rng, 20)
    text = _dna(rng, 300) + q + _dna(rng, 300)
    plain = model_edit.brute([text], [q], 2)
    assert int(plain[0][-1]) >= 3                                   # the run around p = 300
    got = model_loci.collapse(plain, [q])
    assert _lists(got) == [[(300, 0)]]


def test_length_one_never_merges():
    packed = _pack([[(0, 0), (1, 0), (2, 1), (5, 0)], [(3, 0)]])
    got = model_loci.collapse(packed, [b"A", b"C"])
    assert all(np.array_equal(a, b) for a, b in zip(got, packed))


def test_transitive_chain_is_one_locus():
    m, p = 5, 10
    packed = _pack([[(p, 2), (p + m - 1, 1), (p + 2 * m - 2, 2), (p + 3 * m - 2, 0)]])
    assert _lists(model_loci.collapse(packed, [m])) == [[(p + m - 1, 1), (p + 3 * m - 2, 0)]]


def test_document_end_splits():
    packed = _pack([[(8, 1), (9, 0), (10, 0), (11, 1)]])
    assert _lists(model_loci.collapse(packed, [4], np.array([0, 10, 10]))) == [[(9, 0), (10, 0)]]
    assert _lists(model_loci.collapse(packed, [4])) == [[(9, 0)]]


def test_strands_stay_apart_and_keep_their_order():
    packed = _pack([[(4, 1), (4, 0 | MINUS), (5, 0), (5, 1 | MINUS), (6, 2 | MINUS)]])
    assert _lists(model_loci.collapse(packed, [6])) == [[(4, 0 | MINUS), (5, 0)]]


def test_ties_go_to_the_leftmost():
    packed = _pack([[(3, 1), (4, 1), (5, 1)], [(7, 2 | MINUS), (8, 2 | MINUS)]])
    assert _lists(model_loci.collapse(packed, [3, 3])) == [[(3, 1)], [(7, 2 | MINUS)]]


def _random_listings(rng):
    """(name, packed, queries, starts) from the existing models on small random collections."""
    docs = [_dna(rng, int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 4)))]
    text = b"".join(docs) or b"ACGT"
    qs = [b"", b"A", text[:3]]
    for _ in range(4):
        m = int(rng.integers(1, min(len(text), 9) + 1))
        a = int(rng.integers(0, len(text) - m + 1))
        qs.append(text[a:a + m])
    starts = model_approx_docs.starts_of(docs)
    out = [("hamming", model_approx_docs.flagless(docs, qs, 1), qs, starts),
           ("edit_both", model_strand.brute(docs, qs, 2, "edit"), qs, starts),
           ("best", model_best.select(docs, qs, 2, 0, "edit"), qs, starts),
           ("bulges", model_bulges.listing(docs, qs, 1, 1, 1, strands="both"), qs, starts)]
    fdocs = _docs(rng)
    fqs = _queries(rng, fdocs, 2)
    out.append(("fixed", model_fixed.flagless(fdocs, fqs, 2, "edit", strands="both"), fqs,
                model_approx_docs.starts_of(fdocs)))
    return out


@pytest.mark.parametrize("seed", range(6))
def test_properties_on_model_listings(seed):
    rng = np.random.default_rng(100 + seed)
    for name, packed, qs, starts in _random_listings(rng):
        got = model_loci.collapse(packed, qs, starts)
        plain, loci = _lists(packed), _lists(got)
        for q, (hp, hl) in enumerate(zip(plain, loci)):
            assert set(hl) <= set(hp), (name, q)                                        # a subset, equal distances
            assert [h for h in hp if h in set(hl)] == hl, (name, q)                     # in the plain order
            assert bool(hp) == bool(hl), (name, q)
        again = model_loci.collapse(got, qs, starts)
        assert all(np.array_equal(a, b) for a, b in zip(again, got)), name             # idempotent
        # spread: every hit of a strand at least m after the previous one of its query
        spread = []
        for q, hp in zip(qs, plain):
            last, keep = {}, []
            for p, d in hp:
                s = d >= MINUS
                if s not in last or p - last[s] >= len(q):
                    keep.append((p, d))
                    last[s] = p
            spread.append(keep)
        spread = _pack(spread)
        same = model_loci.collapse(spread, qs, starts)
        assert all(np.array_equal(a, b) for a, b in zip(same, spread)), name


def test_keep_ops_filters_to_the_kept_hits():
    ops = _pack([[(3, 5 << 4 | 7), (4, 2 << 4 | 7), (4, 1 << 4 | 8), (4, 1 << 4 | 7 | MINUS)], [(0, 4 << 4 | 7)]])
    kept = _pack([[(4, 1), (4, 0 | MINUS)], []])
    got = model_loci.keep_ops(ops, kept)
    assert _lists(got) == [[(4, 2 << 4 | 7), (4, 1 << 4 | 8), (4, 1 << 4 | 7 | MINUS)], []]


def test_keyword_checks_fail_before_the_device():
    class NoDevice:                                                # any attribute access would fail
        pass

    t = NoDevice()
    for bad in (1, 0, None, "yes", 1.0):
        with pytest.raises(ValueError):
            _approx.positions(t, b"ACGT", 1, loci=bad)
        with pytest.raises(ValueError):
            _approx.counts(t, [b"ACGT"], 1, metric="edit", loci=bad)
    assert _approx._loci(True) == 0x80 and _approx._loci(False) == 0 and _approx.LOCI == 0x80

    from suffix_b200 import DocumentSuffixTable, SuffixTable
    for cls in (SuffixTable, DocumentSuffixTable):
        for name in ("approximate_positions", "approximate_positions_batch", "approximate_counts"):
            sig = inspect.signature(getattr(cls, name))
            assert sig.parameters["loci"].kind == inspect.Parameter.KEYWORD_ONLY, (cls, name)
            assert sig.parameters["loci"].default is False, (cls, name)
