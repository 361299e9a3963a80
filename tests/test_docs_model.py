"""CPU checks of the separator-free generalized suffix array's device formulation
(suffix_b200/csrc/docs.cuh): the numpy model of tests/model_docs.py on SA + LCP of the
concatenation against the definition, on random small document sets."""
import numpy as np
import pytest

from oracle import oracle
from tests import model_docs


def _check(docs):
    text, _ = model_docs.concat(docs)
    sa = oracle.sais(text) if text else np.zeros(0, np.uint32)
    lcp = oracle.lcp_kasai(text, sa) if text else np.zeros(0, np.uint32)
    g, glcp, na = model_docs.model(docs, sa, lcp)
    want_g, want_lcp = model_docs.brute(docs)
    assert np.array_equal(g, want_g), docs
    assert np.array_equal(glcp, want_lcp), docs
    return na


@pytest.mark.parametrize("seed", range(8))
def test_model_matches_definition_random(seed):
    rng = np.random.default_rng(1000 + seed)
    crossing = 0
    for _ in range(300):
        crossing += _check(model_docs.random_docs(rng)) > 0
    assert crossing > 50          # the sorted set A is exercised, not only the rank-order set U


@pytest.mark.parametrize("docs", [
    [], [b""], [b"", b""], [b"x"], [b"", b"x", b""], [b"banana"], [b"a", b"a", b"a"],
    [b"ACGT"] * 50, [b"ab", b"a", b"abab", b"b", b""], [bytes(range(256)), bytes(range(255, -1, -1))],
    [b"\x00", b"\x00\x00", b"\x00\xff\x00"], [b"mississippi", b"ssi", b"issi", b"ppi"],
])
def test_model_matches_definition_cases(docs):
    _check(docs)


def test_single_document_is_the_suffix_table():
    for t in (b"banana", b"aaaaaaaa", b"abracadabra", bytes(range(200))):
        sa = oracle.sais(t)
        lcp = oracle.lcp_kasai(t, sa)
        g, glcp, na = model_docs.model([t], sa, lcp)
        assert na == 0
        assert np.array_equal(g, sa) and np.array_equal(glcp, lcp)


def test_document_table_shares_the_context_lock():
    # DocumentSuffixTable and SuffixTable use the same per-device default context, so they must
    # serialise on the same lock
    from suffix_b200 import docs, table, tree
    assert docs._lock is table._lock is tree._lock
