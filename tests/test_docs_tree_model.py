"""CPU checks of the generalized suffix tree's formulation (include/b200sa.h, b200sa_docs_tree):
the rules model of tests/model_docs_tree.py against the definition, a brute-force compressed trie
of the document suffixes, and against the single-text model for one document."""
import itertools

import numpy as np
import pytest

from oracle import oracle
from tests import model_docs, model_docs_tree, model_tree


def _check(docs):
    text, starts = model_docs.concat(docs)
    g, glcp = model_docs.brute(docs)
    got = model_docs_tree.tree_arrays(g, glcp, starts, len(text))
    want = model_docs_tree.brute(docs)
    for f in model_docs_tree.FIELDS:
        assert np.array_equal(got[f], want[f]), (docs, f, got[f], want[f])
    # doc_count is the size of the node's document set, and the root's is the non-empty documents
    assert [len(s) for s in want["doc_sets"]] == want["doc_count"].tolist()
    assert int(got["doc_count"][0]) == sum(1 for d in docs if d)
    return got


def test_every_ab_set_of_up_to_three_documents():
    by_len = [[bytes(t) for t in itertools.product(b"ab", repeat=k)] for k in range(9)]
    count = 0
    for k in (1, 2, 3):
        for lens in itertools.product(range(9), repeat=k):
            if sum(lens) > 8:
                continue
            for docs in itertools.product(*(by_len[m] for m in lens)):
                _check(list(docs))
                count += 1
    assert count == 511 + 4097 + 18943


@pytest.mark.parametrize("seed", range(8))
def test_random_document_sets(seed):
    rng = np.random.default_rng(2000 + seed)
    for _ in range(300):
        _check(model_docs.random_docs(rng))


@pytest.mark.parametrize("docs", [
    [], [b""], [b"", b""], [b"x"], [b"", b"x", b""], [b"a", b"a", b"a"], [b"ACGT"] * 20,
    [b"ab", b"a", b"abab", b"b", b""], [bytes(range(256)), bytes(range(255, -1, -1))],
    [b"\x00", b"\x00\x00", b"\x00\xff\x00"], [b"mississippi", b"ssi", b"issi", b"ppi"],
])
def test_cases(docs):
    _check(docs)


def test_single_document_is_the_suffix_tree():
    rng = np.random.default_rng(7)
    texts = [b"banana", b"aaaaaaaa", b"abracadabra", bytes(range(200)), b"x"]
    texts += [bytes(rng.integers(0, int(rng.integers(1, 4)), int(rng.integers(1, 50))).astype(np.uint8) + 97)
              for _ in range(300)]
    for t in texts:
        sa = oracle.sais(t)
        lcp = oracle.lcp_kasai(t, sa)
        got = model_docs_tree.tree_arrays(sa, lcp, np.zeros(1, np.uint32), len(t))
        want = model_tree.tree_arrays(sa, lcp)
        for f in model_tree.FIELDS:
            assert np.array_equal(got[f], want[f]), (t, f)
        term = got["sa_lo"] + (got["depth"] == len(t) - sa[np.minimum(got["sa_lo"], len(t) - 1)])
        term[0] = 0
        assert np.array_equal(got["term_end"], term.astype(np.uint32)), t
        assert (got["doc_count"] == 1).all(), t


def test_serial_checker_matches_definition():
    # tests/docs_tree_check.c, which checks the GPU tree at scale, against the definition
    from tests import docs_tree_check
    rng = np.random.default_rng(77)
    sets = [model_docs.random_docs(rng) for _ in range(600)]
    sets += [[b"x"], [b"", b"x", b""], [b"a", b"a", b"a"], [b"ACGT"] * 30, [b"ab", b"a", b"abab", b"b", b""]]
    for docs in sets:
        text, starts = model_docs.concat(docs)
        if not text:
            continue
        g, glcp = model_docs.brute(docs)
        got = docs_tree_check.tree(g, glcp, starts)
        want = model_docs_tree.brute(docs)
        for f in model_docs_tree.FIELDS:
            assert np.array_equal(got[f], want[f]), (docs, f)
