"""The generalized suffix tree with document counts (b200sa_docs_tree[_dev], b200sa_docs_tree_counts_dev,
suffix_b200.DocumentSuffixTree) against the rules model of tests/model_docs_tree.py on small sets,
b200sa_suffix_tree on single documents, and the serial builder of tests/docs_tree_check.c at scale."""
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, DocumentSuffixTree, SuffixTable, SuffixTree, _lib, gen
from tests import docs_tree_check, model_docs, model_docs_tree
from tests.test_gpu_docs import _families

pytestmark = pytest.mark.gpu

FIELDS = model_docs_tree.FIELDS
BAD_ARG = -1


def _u8(t) -> bytes:
    return t if isinstance(t, bytes) else np.ascontiguousarray(t, dtype=np.uint8).tobytes()


def _check_model(docs):
    st = DocumentSuffixTree(docs)
    dt = st.document_table()
    want = model_docs_tree.tree_arrays(dt.table(), dt.lcp_lens(), dt.doc_starts(), len(dt.text()))
    got = st.arrays()
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), (docs, f)
    return st


def test_small_sets_against_model():
    rng = np.random.default_rng(51)
    sets = _families(rng)
    assert len(sets) >= 300
    for docs in sets:
        _check_model(docs)
    # the definition itself on a sample
    for docs in [d for d in sets if sum(map(len, d)) <= 60][::5]:
        got = DocumentSuffixTree(docs).arrays()
        want = model_docs_tree.brute(docs)
        for f in FIELDS:
            assert np.array_equal(got[f], want[f]), (docs, f)


def test_empty_and_single_byte():
    for docs in ([], [b""], [b"", b""]):
        st = DocumentSuffixTree(docs)
        assert {f: a.tolist() for f, a in st.arrays().items()} == {
            "parent": [0xFFFFFFFF], "depth": [0], "sa_lo": [0], "sa_hi": [0], "label_start": [0],
            "subtree_end": [1], "term_end": [0], "doc_count": [0]}
        assert st.root().suffixes() == [] and not st.root().has_terminals()
        assert st.longest_common_substring(1) == b""
    st = DocumentSuffixTree([b"", b"z", b""])
    assert [st.label(c) for c in st.root().children()] == [b"z"]
    (c,) = list(st.root().children())
    assert c.suffixes() == [0] and c.terminals().tolist() == [[1, 0]] and c.doc_count() == 1
    assert st.root().doc_count() == 1


SINGLE = {
    "banana": lambda: b"banana",
    "a3000": lambda: b"a" * 3000,
    "dna": lambda: _u8(gen.dna(300_000)),
    "english": lambda: _u8(gen.english(100_000)),
    "bytes": lambda: _u8(gen.rand_bytes(100_000)),
    "fixture100k": lambda: _u8(gen.fixture("AP009048_100000.fasta")),
}


@pytest.mark.parametrize("name", list(SINGLE))
def test_single_document_is_the_suffix_tree(name):
    t = SINGLE[name]()
    got = DocumentSuffixTree([t]).arrays()
    want = SuffixTree(t).arrays()
    for f in model_docs_tree.FIELDS[:6]:
        assert np.array_equal(got[f], want[f]), f
    sa = SuffixTable(t).table().astype(np.int64)
    lo = got["sa_lo"].astype(np.int64)
    term = lo + (got["depth"].astype(np.int64) == len(t) - sa[np.minimum(lo, len(t) - 1)])
    term[0] = 0
    assert np.array_equal(got["term_end"], term.astype(np.uint32))
    assert (got["doc_count"] == 1).all()


# ---- at scale: the serial builder of tests/docs_tree_check.c
def _check_scale(docs):
    st = DocumentSuffixTree(docs)
    dt = st.document_table()
    want = docs_tree_check.tree(dt.table(), dt.lcp_lens(), dt.doc_starts())
    got = st.arrays()
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), f
    return st


@pytest.mark.slow
def test_scale_dna_cut_with_duplicates():
    rng = np.random.default_rng(21)
    t = _u8(gen.dna(4 << 20))
    cuts = np.unique(rng.integers(1, len(t), 3000))
    docs = [t[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for k in rng.integers(0, len(docs), 40):
        docs.insert(int(rng.integers(0, len(docs) + 1)), docs[int(k)])
    docs.insert(5, b"")
    _check_scale(docs)


def test_docs_tree_acgt_copies():
    docs = [b"ACGT"] * 100_000
    st = _check_scale(docs)
    # four nodes below the root, one per suffix string, each the terminal of every copy
    assert len(st) == 5 and st.arrays()["doc_count"].tolist() == [100_000] * 5
    assert st.longest_common_substring(100_000) == b"ACGT"


@pytest.mark.slow
def test_scale_fixture_lines():
    lines = _u8(gen.fixture("AP009048_100000.fasta")).split(b"\n")
    _check_scale(lines)


@pytest.mark.slow
def test_scale_wide_keys():
    docs = [_u8(gen.dna(1 << 21))] + [bytes([b]) for b in _u8(gen.dna(1 << 21))]
    _check_scale(docs)


# ---- the Node API
def test_node_api_properties():
    rng = np.random.default_rng(61)
    for k in range(40):
        docs = model_docs.random_docs(rng) if k % 2 else [
            bytes(rng.choice(list(b"abc"), int(rng.integers(0, 40)))) for _ in range(int(rng.integers(1, 6)))]
        st = DocumentSuffixTree(docs)
        dt = st.document_table()
        text, starts = dt.text(), dt.doc_starts()
        ends = np.append(starts[1:], len(text))
        root = st.root()
        for p in range(len(text)):                          # every T_p is spelled from the root
            d = int(np.searchsorted(starts, p, side="right")) - 1
            s = text[p:int(ends[d])]
            v, depth = root, 0
            while depth < len(s):
                nxt = [c for c in v.children() if st.label(c)[:1] == s[depth:depth + 1]]
                assert len(nxt) == 1, (docs, p)
                v = nxt[0]
                lab = st.label(v)
                assert s[depth:depth + len(lab)] == lab
                depth += len(lab)
            assert depth == len(s) and p in v.suffixes(), (docs, p)
            assert [d, p - int(starts[d])] in v.terminals().tolist()
        for v in root.preorder():
            ch = list(v.children())
            keys = [st.label(c)[0] for c in ch]
            assert keys == sorted(set(keys))
            if not v.has_terminals() and v.id != 0:         # the root is a node even with one child
                assert len(ch) >= 2
            idx = v.suffix_indices().astype(np.int64)
            docs_below = set((np.searchsorted(starts, idx, side="right") - 1).tolist())
            assert v.doc_count() == len(docs_below)
        assert sorted(p for v in root.preorder() for p in v.suffixes()) == list(range(len(text)))
        assert all(v.has_terminals() for v in root.preorder() if v.id and not list(v.children()))


def test_debug_output():
    st = DocumentSuffixTree([b"ab", b"b"])
    want = ("\n-----------------------------------------\n"
            "SUFFIX TREE\n"
            "text: abb\n"
            "ROOT\n"
            "  [97, 98]\n"
            "  [98]\n"
            "-----------------------------------------\n")
    assert repr(st) == want
    assert st.root().children().__next__().suffixes() == [0]
    assert [c.suffixes() for c in st.root().children()] == [[0], [1, 2]]


# ---- queries
def _brute_doc_count(docs, q):
    return sum(1 for d in docs if q and q in d)


def test_document_counts_against_brute_force():
    rng = np.random.default_rng(71)
    alpha = b"ACG\x00"
    docs = [bytes(alpha[int(c)] for c in rng.integers(0, 4, int(rng.integers(0, 600)))) for _ in range(30)]
    docs += [docs[3], docs[7][:50], b"", b"\x00\x00\x00", docs[3]]
    st = DocumentSuffixTree(docs)
    text, starts = st.text(), st.document_table().doc_starts()
    nonempty = [d for d in range(len(docs)) if docs[d]]
    qs = []
    for k in range(50_000):
        r = k % 3
        if r == 0:
            d = docs[nonempty[int(rng.integers(0, len(nonempty)))]]
            a = int(rng.integers(0, len(d)))
            qs.append(d[a:a + int(rng.integers(1, 12))])
        elif r == 1:
            s = int(starts[nonempty[int(rng.integers(1, len(nonempty)))]])
            qs.append(text[max(0, s - int(rng.integers(1, 6))):s + int(rng.integers(1, 6))])
        else:
            qs.append(bytes(alpha[int(c)] for c in rng.integers(0, 4, int(rng.integers(1, 8)))))
    qs.append(b"")
    memo = {}
    want = [memo.setdefault(q, _brute_doc_count(docs, q)) for q in qs]
    got = st.document_counts(qs)
    assert got.tolist() == want
    assert st.document_counts(qs[:100]).tolist() == want[:100]          # device arrays kept for a second batch
    assert len(st.document_counts([])) == 0


def _brute_lcs(docs, k):
    best = b""
    subs = {}
    for d, doc in enumerate(docs):
        for a in range(len(doc)):
            for b in range(a + 1, len(doc) + 1):
                subs.setdefault(doc[a:b], set()).add(d)
    for s, ds in subs.items():
        if len(ds) >= k and (len(s) > len(best) or (len(s) == len(best) and s < best)):
            best = s
    return best


def test_longest_common_substring_against_brute_force():
    rng = np.random.default_rng(81)
    for it in range(60):
        docs = model_docs.random_docs(rng) if it % 2 else [
            bytes(rng.choice(list(b"ab"), int(rng.integers(0, 25)))) for _ in range(int(rng.integers(1, 6)))]
        st = DocumentSuffixTree(docs)
        for k in range(1, len(docs) + 2):
            # ties go to the lowest preorder id, which is the lexicographically smallest string
            assert st.longest_common_substring(k) == _brute_lcs(docs, k), (docs, k)


# ---- entry points
def _dev_tree(ctx, g, glcp, starts, cap=None, n=None):
    n = len(g) if n is None else n
    cap = max(1, 2 * n) if cap is None else cap
    dev = torch.device("cuda:0")
    up = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int64)).to(dev).to(torch.int32) if len(a) else \
        torch.zeros(1, dtype=torch.int32, device=dev)
    d_g, d_l, d_s = up(g), up(glcp), up(starts)
    outs = [torch.full((max(cap, 1),), -7, dtype=torch.int32, device=dev) for _ in FIELDS]
    N = ctx.docs_tree_dev(n, d_g.data_ptr(), d_l.data_ptr(), d_s.data_ptr() if len(starts) else 0, len(starts),
                          [o.data_ptr() for o in outs], cap, torch.cuda.current_stream().cuda_stream)
    return {f: o[:N].cpu().numpy().view(np.uint32) for f, o in zip(FIELDS, outs)}


def test_device_entry_equals_host_entry():
    ctx = _lib.Context(0)
    rng = np.random.default_rng(91)
    sets = [model_docs.random_docs(rng) for _ in range(30)]
    t = _u8(gen.dna(200_001))
    sets += [[t[:1000], t[1000:1001], b"", t[1001:150_000], t[1000:1001], t[150_000:]], [b"x"], [], [b""]]
    for docs in sets:
        dt = DocumentSuffixTable(docs)
        host = ctx.docs_tree(dt.table(), dt.lcp_lens(), dt.doc_starts())
        dev = _dev_tree(ctx, dt.table(), dt.lcp_lens(), dt.doc_starts())
        for f in FIELDS:
            assert np.array_equal(host[f], dev[f]), (docs, f)
    ctx.set_timing(True)
    dt = DocumentSuffixTable(sets[-4])
    _dev_tree(ctx, dt.table(), dt.lcp_lens(), dt.doc_starts())
    names = [p for p, _ in ctx.phase_times()]
    ctx.set_timing(False)
    for p in ("docs_check", "dtree_len", "tree_ansv", "tree_emit", "tree_sort", "tree_first", "tree_nodes",
              "dtree_term", "dtree_sort", "dtree_pairs", "dtree_count"):
        assert p in names, names
    ctx.close()


def _bad_cases():
    docs = [b"mississippi", b"ssi", b"", b"pi"]
    g, l = model_docs.brute(docs)                       # on the host: this runs at collection
    s = model_docs.concat(docs)[1]
    n = len(g)
    out = []
    x = g.copy(); x[3] = n; out.append(("g_out_of_range", x, l, s, "sa[r] >= n"))
    x = l.copy(); x[0] = 1; out.append(("glcp0", g, x, s, "lcp[0]"))
    x = l.copy(); x[1] = 12; out.append(("glcp_too_long", g, x, s, "longer than"))
    out.append(("starts_not_ascending", g, l, np.array([0, 11, 9, 14], np.uint32), "doc_starts"))
    out.append(("starts_first", g, l, np.array([1, 11, 14, 14], np.uint32), "doc_starts"))
    out.append(("no_docs", g, l, np.zeros(0, np.uint32), "doc_starts"))
    return out


@pytest.mark.parametrize("case", _bad_cases(), ids=lambda c: c[0])
def test_bad_inputs_return_bad_arg(case):
    _, g, l, s, detail = case
    ctx = _lib.Context(0)
    with pytest.raises(_lib.B200SAError) as e:
        ctx.docs_tree(g, l, s)
    assert e.value.code == BAD_ARG and detail in str(e.value)
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, g, l, s)
    assert e.value.code == BAD_ARG and detail in str(e.value)
    dt = DocumentSuffixTable([b"abab", b"ab"])          # the context stays usable
    assert len(ctx.docs_tree(dt.table(), dt.lcp_lens(), dt.doc_starts())["parent"]) > 1
    ctx.close()


def test_cap_and_range_checks():
    ctx = _lib.Context(0)
    dt = DocumentSuffixTable([b"banana", b"ana"])
    g, l, s = dt.table(), dt.lcp_lens(), dt.doc_starts()
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, g, l, s, cap=2 * len(g) - 1)
    assert e.value.code == BAD_ARG and "cap" in str(e.value)
    with pytest.raises(_lib.B200SAError) as e:
        _dev_tree(ctx, [], [], [], cap=0)
    assert e.value.code == BAD_ARG
    # a range that no node has
    a = {f: torch.from_numpy(v.view(np.int32).copy()).cuda() for f, v in ctx.docs_tree(g, l, s).items()}
    d_s = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    d_e = torch.tensor([0, 2], dtype=torch.int32, device="cuda")
    d_c = torch.empty(2, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.B200SAError) as e:
        ctx.docs_tree_counts_dev(a["sa_lo"].data_ptr(), a["sa_hi"].data_ptr(), a["doc_count"].data_ptr(),
                                 len(a["sa_lo"]), d_s.data_ptr(), d_e.data_ptr(), 2, d_c.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    assert e.value.code == BAD_ARG and "no node" in str(e.value)
    ctx.close()


def test_concurrent_with_suffix_tree():
    docs = [_u8(gen.dna(100_000, seed=s)) for s in (1, 2)] + [b"ACGT" * 2000]
    t = _u8(gen.english(150_000))
    want_d = DocumentSuffixTree(docs).arrays()
    want_t = SuffixTree(t).arrays()
    errors = []

    def run(fn):
        try:
            for _ in range(4):
                fn()
        except Exception as e:               # reported in the main thread
            errors.append(e)

    def build_docs():
        got = DocumentSuffixTree(docs).arrays()
        assert all(np.array_equal(got[f], want_d[f]) for f in FIELDS)

    def build_tree():
        got = SuffixTree(t).arrays()
        assert all(np.array_equal(got[f], want_t[f]) for f in want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (build_docs, build_tree)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
