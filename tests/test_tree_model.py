"""CPU checks of the suffix tree formulation: the rules-1-8 model (tests/model_tree.py)
against the C restatement of the reference's insertion loop (tests/tree_oracle.c), and
that restatement against a literal Python one on small strings."""
import itertools

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import gen
from tests import families, model_tree, tree_oracle

KAT = families.kat()


def _sa_lcp(t: bytes):
    sa = oracle.sais(t)
    return sa, oracle.lcp_quadratic(t, sa)


def _check_model(t: bytes):
    sa, lcp = _sa_lcp(t)
    want = tree_oracle.suffix_tree(sa, lcp)
    got = model_tree.tree_arrays(sa, lcp)
    for f in model_tree.FIELDS:
        assert np.array_equal(got[f], want[f]), (t[:40], f)
    # label bytes: the model's offsets and the oracle's own offsets name the same bytes
    lens = tree_oracle.label_lengths(want)
    assert np.array_equal(want["own_end"] - want["own_start"], lens)
    assert tree_oracle.labels_differ(t, got["label_start"], want["own_start"], lens) == -1, t[:40]


def test_all_ab_strings_up_to_12():
    for k in range(13):
        for tup in itertools.product(b"ab", repeat=k):
            _check_model(bytes(tup))


def test_random_small_alphabets():
    rng = np.random.default_rng(8)
    for _ in range(2000):
        sigma = int(rng.integers(1, 5))
        t = bytes(rng.integers(0, sigma, int(rng.integers(0, 60))).astype(np.uint8) + 97)
        _check_model(t)


@pytest.mark.parametrize("case", KAT["kat"], ids=lambda c: repr(c["text"])[:24])
def test_kats(case):
    _check_model(case["text"].encode("utf-8"))


@pytest.mark.parametrize("name", ["AP009048_10000.fasta", "AP009048_100000.fasta"])
def test_fixtures(name):
    _check_model(gen.fixture(name).tobytes())


# ---- the oracle against a literal restatement of to_suffix_tree (suffix_tree/src/lib.rs:392-505)
class _N:
    def __init__(self, start, end, terms):
        self.parent, self.children, self.suffixes = None, {}, terms
        self.start, self.end, self.path_len = start, end, 0

    def add_parent(self, p):
        self.parent = p
        self.path_len = p.path_len + (self.end - self.start)


def _brute(t: bytes):
    sa, lcp = _sa_lcp(t)
    n = len(t)
    root = _N(0, 0, [n])
    last = root
    for i, s in enumerate(int(x) for x in sa):
        L = int(lcp[i])
        v = last
        while v.path_len > L and v.parent is not None:
            v = v.parent
        if v.path_len == L:
            leaf = _N(s + L, n, [s])
            leaf.add_parent(v)
            assert t[leaf.start] not in v.children
            v.children[t[leaf.start]] = leaf
        else:
            rkey = max(v.children)
            r = v.children.pop(rkey)
            p = int(sa[i - 1])
            w = _N(p + v.path_len, p + L, [])
            w.add_parent(v)
            r.start, r.end = p + L, p + r.path_len
            r.add_parent(w)
            leaf = _N(s + L, n, [s])
            leaf.add_parent(w)
            w.children[t[r.start]] = r
            w.children[t[leaf.start]] = leaf
            v.children[t[w.start]] = w
        last = leaf
    return sa, lcp, root


def _flatten(root):
    out, stack, ids = [], [root], {}
    while stack:
        v = stack.pop()
        ids[id(v)] = len(out)
        out.append(v)
        stack.extend(v.children[k] for k in sorted(v.children, reverse=True))
    return out, ids


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_literal_insertion_loop(seed):
    rng = np.random.default_rng(100 + seed)
    texts = [b"", b"a", b"banana", b"mississippi", b"aaaa", b"abab", b"abaca", b"babc", b"apple"]
    texts += [bytes(rng.integers(0, int(rng.integers(1, 5)), int(rng.integers(0, 40))).astype(np.uint8) + 97)
              for _ in range(300)]
    for t in texts:
        sa, lcp, root = _brute(t)
        nodes, ids = _flatten(root)
        got = tree_oracle.suffix_tree(sa, lcp)
        assert len(got["parent"]) == len(nodes), t
        for k, v in enumerate(nodes):
            assert got["parent"][k] == (model_tree.NONE if v.parent is None else ids[id(v.parent)]), t
            assert got["depth"][k] == v.path_len, t
            assert (got["own_start"][k], got["own_end"][k]) == (v.start, v.end), t
            term = got["terminal"][k]
            assert ([] if term == model_tree.NONE else [int(term)]) == v.suffixes, t
            ch = [ids[id(c)] for _, c in sorted(v.children.items())]
            assert ch == list(model_tree.children(got, k)), t
        # subtree ranges hold exactly the suffixes of the leaf walk below the node
        for k, v in enumerate(nodes):
            walk = [s for u in _flatten(v)[0] if u.end > u.start for s in u.suffixes]
            assert walk == sa[got["sa_lo"][k]:got["sa_hi"][k]].tolist(), t
