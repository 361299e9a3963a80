"""Top-k document retrieval (b200sa_docs_topk_dev, DocumentSuffixTable.top_documents*) against the model of
tests/model_docs_topk.py, brute force over the documents of G[s:e], and the listing route (documents_batch
followed by a host sort by (-count, document))."""
import os
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import model_docs, model_docs_list, model_docs_topk
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_docs_list import _scale_docs

pytestmark = pytest.mark.gpu

BAD_ARG = -1
MARK = 0xFFFFFFFF
KS = (1, 2, 3, 1024)


def _topk_ranges(ctx, st, s, e, k):
    """The C-ABI on explicit ranges: (count, docs, tf), docs / tf as nq x k arrays pre-filled with MARK."""
    byd, prev = st._list_arrays()
    _, d_g, d_s = st._device_arrays()
    s = np.asarray(s, np.uint32)
    e = np.asarray(e, np.uint32)
    nq = len(s)
    d_start = torch.from_numpy(s.view(np.int32).copy()).cuda()
    d_end = torch.from_numpy(e.view(np.int32).copy()).cuda()
    d_count = torch.full((max(nq, 1),), -1, dtype=torch.int32, device="cuda")
    d_docs = torch.full((max(nq * k, 1),), -1, dtype=torch.int32, device="cuda")
    d_tf = torch.full((max(nq * k, 1),), -1, dtype=torch.int32, device="cuda")
    ctx.docs_topk_dev(len(st), d_g.data_ptr(), d_s.data_ptr(), len(st.doc_starts()), byd.data_ptr(), prev.data_ptr(),
                      d_start.data_ptr(), d_end.data_ptr(), nq, k, d_count.data_ptr(), d_docs.data_ptr(),
                      d_tf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return (d_count.cpu().numpy().view(np.uint32)[:nq], d_docs.cpu().numpy().view(np.uint32)[:nq * k].reshape(nq, k),
            d_tf.cpu().numpy().view(np.uint32)[:nq * k].reshape(nq, k))


def _check_abi(count, docs, tf, want):
    """want: per query [(d, tf), ...]; slots past count[q] keep MARK."""
    assert count.tolist() == [len(w) for w in want]
    for q, w in enumerate(want):
        c = len(w)
        assert list(zip(docs[q, :c].tolist(), tf[q, :c].tolist())) == w, q
        assert (docs[q, c:] == MARK).all() and (tf[q, c:] == MARK).all(), q


def _check_batch(got, want):
    off, dd, tf = got
    assert np.diff(off.astype(np.int64)).tolist() == [len(w) for w in want] and off[0] == 0
    assert list(zip(dd.tolist(), tf.tolist())) == [r for w in want for r in w]


def _brute(st, s, e, k):
    """Per range the top-k by brute force: np.unique over the documents of G[s:e]."""
    doc = np.searchsorted(st.doc_starts(), st.table(), side="right") - 1
    out = []
    for a, b in zip(s, e):
        d, cnt = np.unique(doc[int(a):int(b)], return_counts=True)
        o = np.lexsort((d, -cnt))[:k]
        out.append(list(zip(d[o].tolist(), cnt[o].tolist())))
    return out


def _listing_route(st, qs, k):
    """documents_batch, then per query a host sort by (-count, document), cut to k."""
    off, dd, tf = st.documents_batch(qs)
    out = []
    for q in range(len(qs)):
        a, b = int(off[q]), int(off[q + 1])
        o = np.lexsort((dd[a:b], -tf[a:b].astype(np.int64)))[:k]
        out.append(list(zip(dd[a:b][o].tolist(), tf[a:b][o].tolist())))
    return out


def test_families_against_model():
    rng = np.random.default_rng(31)
    ctx = _lib.Context(0)
    sets = _families(rng)
    assert len(sets) >= 300
    for docs in sets:
        st = DocumentSuffixTable(docs)
        qs = sorted({x[a:a + m] for x in docs for m in range(1, 4) for a in range(len(x) - m + 1)})
        qs += [b"", b"zz", b"\x01\x02"]
        g, doc, byd, prev = model_docs_list.index(docs)
        text, starts = model_docs.concat(docs)
        ranges = [model_docs_list.query_range(docs, g, q) for q in qs]
        s_arr, e_arr = st.positions_batch(qs)
        for k in KS:
            want = [model_docs_topk.top_k(starts, len(text), doc, byd, prev, a, b, k) for a, b in ranges]
            _check_abi(*_topk_ranges(ctx, st, s_arr, e_arr, k), want)
            _check_batch(st.top_documents_batch(qs, k), want)
    ctx.close()


def _edge_docs(df, rng):
    """Documents in which b"x" occurs in exactly df of them, 1 to 3 times each (distinct and tied counts),
    among documents without it."""
    docs = []
    for _ in range(df):
        docs.append(b"x" * int(rng.integers(1, 4)) + b"y")
        if rng.random() < 0.3:
            docs.append(b"yy")
    return docs


# TOPK_WARP = 32 and TOPK_TILE = 4096 separate the warp, block and multi-tile classes; with k = 1024,
# 16384 = 4 * 4096 is the last df whose candidates fit one tile after the first level (4 * 1024).
@pytest.mark.parametrize("T", [32, 4096, 16384])
def test_class_edges(T):
    rng = np.random.default_rng(T)
    ctx = _lib.Context(0)
    for df in (T - 1, T, T + 1):
        st = DocumentSuffixTable(_edge_docs(df, rng))
        qs = [b"x", b"xx", b"xxx", b"y", b"xy", b"z"]
        s, e = st.positions_batch(qs)
        assert int(e[0]) - int(s[0]) >= df
        for k in sorted({1, 2, 31, 32, 33, 1000, 1024, min(df - 1, 1024), min(df, 1024)}):
            want = _brute(st, s, e, k)
            assert len(want[0]) == min(k, df)
            _check_abi(*_topk_ranges(ctx, st, s, e, k), want)
        _check_batch(st.top_documents_batch(qs, 7), _brute(st, s, e, 7))
    ctx.close()


def test_ties_acgt_copies():
    st = DocumentSuffixTable([b"ACGT"] * 100_000)
    for k in (1, 10, 1024):
        rows = st.top_documents(b"A", k)
        assert rows.shape == (k, 2)
        assert np.array_equal(rows[:, 0], np.arange(k)) and (rows[:, 1] == 1).all()
    off, dd, tf = st.top_documents_batch([b"A", b"ACGTA", b"GT", b""], 5)
    assert off.tolist() == [0, 5, 5, 10, 10]
    assert dd.tolist() == [0, 1, 2, 3, 4] * 2 and (tf == 1).all()


def _scale_queries():
    t, docs = _scale_docs()
    rng = np.random.default_rng(22)
    qs = []
    for _ in range(50_000):
        a = int(rng.integers(0, len(t) - 16))
        qs.append(t[a:a + int(rng.integers(4, 17))])
    return docs, qs + [b"A", b"C"]


def test_scale_against_listing_route():
    docs, qs = _scale_queries()
    st = DocumentSuffixTable(docs)
    df = st.document_frequencies(qs)
    for k in (1, 10, 1024):
        off, dd, tf = st.top_documents_batch(qs, k)
        assert np.array_equal(np.diff(off.astype(np.int64)), np.minimum(df, k))
        _check_batch((off, dd, tf), _listing_route(st, qs, k))


def test_rounds_equal_one_round():
    docs, qs = _scale_queries()
    st = DocumentSuffixTable(docs)
    s, e = st.positions_batch(qs)
    budget = 3000
    df = st.document_frequencies(qs)
    assert df.max() > budget                                      # b"A" alone is larger than a round
    ctx = _lib.Context(0)
    for k in (1, 10, 1024):
        want = _topk_ranges(ctx, st, s, e, k)
        os.environ["B200SA_TOPK_ROUND"] = str(budget)
        try:
            ctx.set_timing(True)
            got = _topk_ranges(ctx, st, s, e, k)
            rounds = [p for p, _ in ctx.phase_times()].count("topk_emit")
            ctx.set_timing(False)
            got_py = st.top_documents_batch(qs, k)
        finally:
            del os.environ["B200SA_TOPK_ROUND"]
        assert rounds >= 10                                       # phase_times shows the first 64 phases
        for x, y in zip(got, want):
            assert np.array_equal(x, y)
        _check_batch(got_py, [list(zip(want[1][q, :c].tolist(), want[2][q, :c].tolist()))
                              for q, c in enumerate(want[0].tolist())])
    ctx.close()


def test_arguments():
    _, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:300])
    s, e = st.positions_batch([b"ACG", b"T"])
    n = len(st)
    ctx = _lib.Context(0)
    for k in (0, 1025):
        with pytest.raises(_lib.B200SAError) as ex:
            _topk_ranges(ctx, st, s, e, k)
        assert ex.value.code == BAD_ARG and "docs topk" in str(ex.value)
    for bad_s, bad_e in ((5, 4), (0, n + 1), (n, n + 7)):
        with pytest.raises(_lib.B200SAError) as ex:
            _topk_ranges(ctx, st, [0, bad_s], [3, bad_e], 4)
        assert ex.value.code == BAD_ARG and "docs list" in str(ex.value)
    byd, prev = st._list_arrays()
    _, d_g, d_s = st._device_arrays()
    buf = torch.full((64,), -1, dtype=torch.int32, device="cuda")
    p = buf.data_ptr()
    full = [n, d_g.data_ptr(), d_s.data_ptr(), len(st.doc_starts()), byd.data_ptr(), prev.data_ptr(), p, p + 8, 2, 4,
            p + 16, p + 32, p + 64, 0]
    for i in (1, 2, 4, 5, 6, 7, 10, 11, 12):                      # one null pointer at a time
        args = list(full)
        args[i] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.docs_topk_dev(*args)
        assert ex.value.code == BAD_ARG
    with pytest.raises(ValueError):
        st.top_documents_batch([b"A"], 0)
    with pytest.raises(ValueError):
        st.top_documents(b"A", 1025)
    # the context still works, and reports the phases
    ctx.set_timing(True)
    count, _, _ = _topk_ranges(ctx, st, s, e, 4)
    names = [q for q, _ in ctx.phase_times()]
    ctx.set_timing(False)
    assert count.tolist() == [min(4, x) for x in st.document_frequencies([b"ACG", b"T"]).tolist()]
    for q in ("dlist_levels", "dlist_count", "dlist_scan", "topk_emit", "topk_select"):
        assert q in names, names
    # nq = 0 writes nothing
    args = list(full)
    args[8] = 0
    ctx.docs_topk_dev(*args)
    torch.cuda.synchronize()
    assert (buf == -1).all()
    ctx.close()


def test_empty_and_tiny_tables():
    e = DocumentSuffixTable([])
    off, dd, tf = e.top_documents_batch([b"a", b""], 3)
    assert off.tolist() == [0, 0, 0] and len(dd) == 0 and len(tf) == 0
    assert e.top_documents(b"a", 1).shape == (0, 2)
    ctx = _lib.Context(0)
    count, docs, _ = _topk_ranges(ctx, e, [0, 0], [0, 0], 2)
    assert count.tolist() == [0, 0] and (docs == MARK).all()
    ctx.close()
    one = DocumentSuffixTable([b"", b"zz", b"", b"z"])
    assert one.top_documents(b"z", 5).tolist() == [[1, 2], [3, 1]]
    assert one.top_documents(b"z", 1).tolist() == [[1, 2]]
    assert one.top_documents_batch([], 4)[0].tolist() == [0]


def test_concurrent_topk_with_suffix_table_builds():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:800])
    rng = np.random.default_rng(5)
    qs = []
    for _ in range(3000):
        a = int(rng.integers(0, len(t) - 12))
        qs.append(t[a:a + int(rng.integers(3, 12))])
    want = st.top_documents_batch(qs, 10)
    text = _u8(gen.english(300_000))
    want_t = SuffixTable(text).table()
    errors = []

    def run(fn):
        try:
            for _ in range(5):
                fn()
        except Exception as ex:
            errors.append(ex)

    def topk():
        got = st.top_documents_batch(qs, 10)
        assert all(np.array_equal(x, y) for x, y in zip(got, want))

    def build():
        assert np.array_equal(SuffixTable(text).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (topk, topk, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
