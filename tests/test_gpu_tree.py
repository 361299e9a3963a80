"""The suffix tree built on the GPU (b200sa_suffix_tree[_dev], suffix_b200.SuffixTree) against
the C restatement of the reference's insertion loop (tests/tree_oracle.c), the reference's
own quickcheck properties (suffix_tree/src/lib.rs:528-566) and its Debug output."""
import ctypes

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import SuffixTable, SuffixTree, _lib, gen
from tests import tree_oracle

pytestmark = pytest.mark.gpu

FIELDS = tree_oracle.FIELDS


def _u8(t) -> bytes:
    return t if isinstance(t, bytes) else np.ascontiguousarray(t, dtype=np.uint8).tobytes()


def _check_against_oracle(t: bytes, st: SuffixTree = None):
    st = SuffixTree(t) if st is None else st
    sa = oracle.sais(t)
    assert np.array_equal(st._table, sa)
    want = tree_oracle.suffix_tree(sa, oracle.lcp_kasai(t, sa))
    got = st.arrays()
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), f
    lens = tree_oracle.label_lengths(want)
    assert np.array_equal(want["own_end"] - want["own_start"], lens)
    assert tree_oracle.labels_differ(t, got["label_start"], want["own_start"], lens) == -1
    return st


CASES = {
    "n0": lambda: b"",
    "n1": lambda: b"x",
    "n2": lambda: b"ab",
    "banana": lambda: b"banana",
    "mississippi": lambda: b"mississippi",
    "apple": lambda: b"apple",
    "a3000": lambda: b"a" * 3000,
    "a100k": lambda: b"a" * 100_000,
    "nul_ff": lambda: bytes([0, 255, 0, 0, 255, 1, 0, 255, 255, 0] * 500),
    "bytes200k": lambda: _u8(gen.rand_bytes(200_000)),
    "english150k": lambda: _u8(gen.english(150_000)),
    "fixture100k": lambda: _u8(gen.fixture("AP009048_100000.fasta")),
    "tiled": lambda: _u8(gen.tiled(gen.fixture("AP009048_10000.fasta"), 300_000)),
    "dna1m": lambda: _u8(gen.dna(1_000_000)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_tree_matches_oracle(name):
    _check_against_oracle(CASES[name]())


def test_empty_and_single():
    st = SuffixTree(b"")
    r = st.root()
    assert len(st) == 1 and r.len() == 0 and r.suffixes() == [0] and r.has_terminals()
    assert list(r.children()) == [] and list(r.leaves()) == [] and r.suffix_indices().tolist() == []
    st = SuffixTree(b"x")
    assert [st.label(c) for c in st.root().children()] == [b"x"]
    assert st.root().suffixes() == [1]


def test_quickcheck_properties_through_node_api():
    """qc_n_leaves, qc_internals_have_at_least_two_children, qc_tree_enumerates_suffixes
    (suffix_tree/src/lib.rs:528-566), plus child order and the ancestor chain."""
    rng = np.random.default_rng(5)
    for k in range(60):
        sigma = [1, 2, 4, 26, 256][k % 5]
        n = int(rng.integers(0, 300))
        t = bytes(rng.integers(0, sigma, n).astype(np.uint8) + (97 if sigma < 256 else 0))
        st = SuffixTree(t)
        root = st.root()
        assert sum(1 for _ in root.leaves()) == n
        for v in root.preorder():
            ch = list(v.children())
            if not v.has_terminals():
                assert len(ch) >= 2
            keys = [st.label(c)[0] for c in ch]
            assert keys == sorted(set(keys))
            anc = list(v.ancestors())
            assert anc[0] == v and anc[-1] == root and v.depth() == len(anc) - 1
            assert sum(a.len() for a in anc) == int(st.arrays()["depth"][v.id])
        sa = st._table
        idx = root.suffix_indices()
        assert np.array_equal(idx, sa)
        for i, s in enumerate(idx.tolist()):
            assert t[s:] == t[int(sa[i]):]
        walk = [s for leaf in root.leaves() for s in leaf.suffixes()]
        assert walk == sa.tolist()
        terms = sorted(s for v in root.preorder() for s in v.suffixes())
        assert terms == list(range(n + 1))


def test_debug_banana():
    want = ("\n-----------------------------------------\n"
            "SUFFIX TREE\n"
            "text: banana\n"
            "ROOT\n"
            "  [97]\n"
            "    [110, 97]\n"
            "      [110, 97]\n"
            "  [98, 97, 110, 97, 110, 97]\n"
            "  [110, 97]\n"
            "    [110, 97]\n"
            "-----------------------------------------\n")
    assert repr(SuffixTree("banana")) == want


def test_from_suffix_table_of_parts():
    t = _u8(gen.english(20_000))
    tab = SuffixTable.from_parts(t, oracle.sais(t))
    st = SuffixTree.from_suffix_table(tab)
    _check_against_oracle(t, st)
    assert st.text() == t


# ---- the device entry point and its input checks
def _dev_tree(ctx, sa, lcp, cap=None):
    import torch
    n = len(sa)
    cap = max(1, 2 * n) if cap is None else cap
    dev = torch.device("cuda:0")
    d_sa = torch.from_numpy(np.asarray(sa, dtype=np.int64)).to(dev).to(torch.int32)
    d_lcp = torch.from_numpy(np.asarray(lcp, dtype=np.int64)).to(dev).to(torch.int32)
    outs = [torch.empty(max(cap, 1), dtype=torch.int32, device=dev) for _ in FIELDS]
    N = ctx.suffix_tree_dev(n, d_sa.data_ptr(), d_lcp.data_ptr(), [o.data_ptr() for o in outs], cap,
                            torch.cuda.current_stream().cuda_stream)
    return {f: o[:N].cpu().numpy().view(np.uint32) for f, o in zip(FIELDS, outs)}


def test_device_entry_and_phase_times():
    ctx = _lib.Context(0)
    t = _u8(gen.dna(300_000))
    sa = oracle.sais(t)
    lcp = oracle.lcp_kasai(t, sa)
    ctx.set_timing(True)
    got = _dev_tree(ctx, sa, lcp)
    names = [p for p, _ in ctx.phase_times()]
    for p in ("tree_ansv", "tree_emit", "tree_sort", "tree_first", "tree_nodes"):
        assert p in names
    want = tree_oracle.suffix_tree(sa, lcp)
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), f
    root = _dev_tree(ctx, [], [])
    assert {f: a.tolist() for f, a in root.items()} == \
        {"parent": [0xFFFFFFFF], "depth": [0], "sa_lo": [0], "sa_hi": [0], "label_start": [0], "subtree_end": [1]}
    ctx.close()


def _bad_inputs():
    t = b"mississippi"
    sa = oracle.sais(t)
    lcp = oracle.lcp_quadratic(t, sa)
    n = len(t)
    out = []
    s = sa.copy(); s[3] = n; out.append(("sa_out_of_range", s, lcp))
    lc = lcp.copy(); lc[0] = 1; out.append(("lcp0", sa, lc))
    lc = lcp.copy(); lc[1] = n; out.append(("lcp_too_long", sa, lc))
    # passes the per-rank checks, but rank 3 starts no node: not the LCP array of that table
    out.append(("rank_without_node", np.array([3, 2, 4, 1, 0], np.uint32), np.array([0, 1, 1, 1, 4], np.uint32)))
    return out


@pytest.mark.parametrize("case", _bad_inputs(), ids=lambda c: c[0])
def test_input_checks_return_bad_arg(case):
    _, sa, lcp = case
    ctx = _lib.Context(0)
    with pytest.raises(_lib.B200SAError) as e:
        ctx.suffix_tree(sa, lcp)
    assert e.value.code == -1
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, sa, lcp)
    assert e.value.code == -1
    t = b"mississippi"                               # the context still works afterwards
    good = oracle.sais(t)
    assert len(ctx.suffix_tree(good, oracle.lcp_quadratic(t, good))["parent"]) > 1
    ctx.close()


def test_cap_and_size_limits():
    ctx = _lib.Context(0)
    t = b"banana"
    sa = oracle.sais(t)
    lcp = oracle.lcp_quadratic(t, sa)
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, sa, lcp, cap=2 * len(t) - 1)
    assert e.value.code == -1
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, [], [], cap=0)
    assert e.value.code == -1
    p = ctypes.c_void_p(8)
    tr = _lib.Tree(*([p.value] * 6))
    N = ctypes.c_uint64(0)
    rc = _lib.lib().b200sa_suffix_tree_dev(ctx._h, 1 << 31, p, p, ctypes.byref(tr), 1 << 33, ctypes.byref(N), None)
    assert rc == -2
    ctx.close()


# ---- full size
@pytest.mark.slow
@pytest.mark.parametrize("maker", ["dna", "english"])
def test_tree_10mb_against_oracle(maker):
    t = _u8(gen.dna(10_000_000) if maker == "dna" else gen.english(10_000_000))
    _check_against_oracle(t)


@pytest.mark.slow
def test_tree_100mb_dna_structure():
    t = _u8(gen.dna(100_000_000))
    tab = SuffixTable(t)
    st = SuffixTree.from_suffix_table(tab)
    a = {f: v.astype(np.int64) for f, v in st.arrays().items()}
    sa = tab.table().astype(np.int64)
    lcp = tab.lcp_lens().astype(np.int64)
    n, N = len(t), len(a["parent"])
    v = np.arange(1, N)
    p = a["parent"][1:]
    assert a["parent"][0] == 0xFFFFFFFF
    assert (p < v).all()                                   # parents precede children
    assert (a["depth"][1:] > a["depth"][p]).all()          # depth strictly increases downwards
    assert (a["sa_lo"][p] <= a["sa_lo"][1:]).all() and (a["sa_hi"][1:] <= a["sa_hi"][p]).all()
    assert (a["sa_lo"] < a["sa_hi"]).all() and (a["subtree_end"][1:] > v).all()
    # rule 4: N = 1 + #internal + n - #merged; the internal nodes are the distinct LCP intervals
    _, psv, nsv = tab.lcp_intervals(lcp.astype(np.uint32))
    pos = np.nonzero(lcp[1:] > 0)[0] + 1
    internal = len(np.unique((psv[pos].astype(np.int64) << 32) | nsv[pos].astype(np.int64)))
    merged = int(np.count_nonzero(lcp[1:] == n - sa[:-1]))
    assert N == 1 + internal + n - merged
    # every rank (and so every suffix) is the terminal of exactly one node
    term = a["depth"][1:] == n - sa[a["sa_lo"][1:]]
    ranks = a["sa_lo"][1:][term]
    assert len(ranks) == n and (np.bincount(ranks, minlength=n) == 1).all()
