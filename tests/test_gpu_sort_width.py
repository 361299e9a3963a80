"""Every one-sweep radix sort gives the same arrays with either tile width.  Each stage that sorts runs at item
counts just below and at 2^20, where the default width changes, with no switch, B200SA_SORT_NARROW=1,
B200SA_SORT_ITEMS=8 and B200SA_SORT_ITEMS=16 (INTEGRATION.md section 6), and the four outputs must be equal."""
import numpy as np
import pytest
import torch

from oracle import oracle
from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen, inverse_bwt_documents
from tests import tree_oracle
from tests.test_gpu_lms_sort import _text_with_m

pytestmark = pytest.mark.gpu

WIDE_FROM = 1 << 20
SIDES = {"below": WIDE_FROM - 1, "at": WIDE_FROM}
SWITCHES = [{}, {"B200SA_SORT_NARROW": "1"}, {"B200SA_SORT_ITEMS": "8"}, {"B200SA_SORT_ITEMS": "16"}]


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _same_under_switches(monkeypatch, run):
    """run() under each switch; its outputs (a tuple of arrays) must not depend on the switch."""
    outs = []
    for env in SWITCHES:
        monkeypatch.delenv("B200SA_SORT_NARROW", raising=False)
        monkeypatch.delenv("B200SA_SORT_ITEMS", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        outs.append(run())
    for env, out in zip(SWITCHES[1:], outs[1:]):
        assert len(out) == len(outs[0])
        for i, (a, b) in enumerate(zip(outs[0], out)):
            assert np.array_equal(a, b), (env, i)
    return outs[0]


def _smallest_prefix(count, lo, hi, target):
    """The shortest prefix length in [lo, hi] whose count() reaches target (count grows with the prefix)."""
    assert count(lo) < target <= count(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if count(mid) >= target:
            hi = mid
        else:
            lo = mid
    return hi


@pytest.mark.parametrize("side", SIDES)
@pytest.mark.parametrize("text, env", [("dna", {}), ("dna", {"B200SA_LMS_SORT4": "1"}),
                                       ("dna", {"B200SA_NO_DIRECT": "1"}), ("english", {})],
                         ids=["dna_bucketed", "dna_four_pass", "dna_robust", "english"])
def test_lms_sort_and_rank_doubling(ctx, monkeypatch, side, text, env):
    # m LMS suffixes: the LMS sort (direct path) or the rank doubling of the reduced string (robust path)
    m = SIDES[side]
    base = gen.english(int(m * 3.6) + 1000, seed=gen.SEED_ENGLISH + m) if text == "english" else None
    t = _text_with_m(m, base)
    for k, v in env.items():
        monkeypatch.setenv(k, v)

    def run():
        sa, lcp = ctx.build_lcp(t)
        assert ctx.stats()["m"] == m
        return sa, lcp

    sa, _ = _same_under_switches(monkeypatch, run)
    assert np.array_equal(sa, oracle.sais(t))


@pytest.mark.parametrize("side", SIDES)
def test_suffix_tree(ctx, monkeypatch, side):
    # the tree sorts its N nodes: the shortest prefix of G_dna with N >= 2^20, and that prefix less one byte
    base = gen.dna(700_000)

    def nodes(n):
        sa = oracle.sais(base[:n])
        return len(tree_oracle.suffix_tree(sa, oracle.lcp_kasai(base[:n], sa))["parent"])

    n = _smallest_prefix(nodes, 645_500, 646_500, WIDE_FROM) - (side == "below")
    t = base[:n]
    sa, lcp = ctx.build_lcp(t)
    a = _same_under_switches(monkeypatch, lambda: tuple(ctx.suffix_tree(sa, lcp).values()))
    assert (len(a[0]) >= WIDE_FROM) == (side == "at")


def _crossing(docs):
    """|A| of b200sa_docs_build: the ranks of the concatenation whose LCP reaches their document's end."""
    text = np.frombuffer(b"".join(docs), np.uint8)
    starts = np.cumsum([0] + [len(d) for d in docs[:-1]])
    ends = np.append(starts[1:], len(text))
    sa = oracle.sais(text)
    rem = ends[np.searchsorted(starts, sa, side="right") - 1] - sa
    return int((oracle.lcp_kasai(text, sa) >= rem).sum())


@pytest.mark.parametrize("side", SIDES)
@pytest.mark.parametrize("two_stage", [False, True])
def test_document_array(monkeypatch, side, two_stage):
    # 1024 copies of one document cross their ends about 1023 * 1024 times; a prefix of it put in front adds
    # one crossing per byte
    d = gen.dna(1024, seed=7).tobytes()
    copies = [d] * 1024
    x = SIDES[side] - _crossing(copies)
    assert 0 < x <= len(d)
    docs = [d[:x]] + copies
    assert _crossing(docs) == SIDES[side]
    if two_stage:
        monkeypatch.setenv("B200SA_DOCS_SORT2", "1")

    def run():
        dt = DocumentSuffixTable(docs)
        return dt.table(), dt.lcp_lens()

    _same_under_switches(monkeypatch, run)


@pytest.mark.parametrize("side", SIDES)
def test_document_tree_and_listing_index(ctx, monkeypatch, side):
    # both sort the n ranks of G by document
    n = SIDES[side]
    text = gen.dna(n, seed=11)
    rng = np.random.default_rng(n)
    starts = np.unique(np.concatenate([[0], rng.integers(1, n, 2000)])).astype(np.uint32)
    gsa, glcp = ctx.docs_build(text, starts)
    d_g = torch.from_numpy(gsa.view(np.int32).copy()).cuda()
    d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()

    def run():
        tree = ctx.docs_tree(gsa, glcp, starts)
        byd = torch.empty(n, dtype=torch.int32, device="cuda")
        prev = torch.empty(n, dtype=torch.int32, device="cuda")
        ctx.docs_list_index_dev(n, d_g.data_ptr(), d_s.data_ptr(), len(starts), byd.data_ptr(), prev.data_ptr(),
                                torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return tuple(tree.values()) + (byd.cpu().numpy(), prev.cpu().numpy())

    _same_under_switches(monkeypatch, run)


@pytest.mark.parametrize("side", SIDES)
def test_bwt_inverse(monkeypatch, side):
    # one byte per document: the inverse sorts as many term rows as bytes
    k = SIDES[side]
    docs = [bytes([c]) for c in gen.dna(k, seed=13).tolist()]
    bwt, term = DocumentSuffixTable(docs).bwt()

    def run():
        out = inverse_bwt_documents(bwt, term)
        return np.frombuffer(b"".join(out), np.uint8), np.array([len(x) for x in out])

    text, lens = _same_under_switches(monkeypatch, run)
    assert text.tobytes() == b"".join(docs) and np.all(lens == 1)


@pytest.mark.parametrize("side", SIDES)
def test_approximate_hits(monkeypatch, side):
    # a 24-mer planted h times, asked r times: the search sorts h * r hits (k = 0 keeps h exact)
    h, r = (1025, 1023) if side == "below" else (1024, 1024)
    rng = np.random.default_rng(h)
    q = gen.dna(24, seed=17).tobytes()
    text = bytearray(gen.dna(64 * h, seed=19).tobytes())
    for p in rng.choice(np.arange(0, len(text) - 24, 32), h, replace=False).tolist():
        text[p:p + 24] = q
    text = bytes(text)
    assert sum(1 for i in range(len(text) - 23) if text.startswith(q, i)) == h
    st = SuffixTable(text)

    off, _, _ = _same_under_switches(monkeypatch, lambda: st.approximate_positions_batch([q] * r, 0))
    assert int(off[-1]) == SIDES[side]
