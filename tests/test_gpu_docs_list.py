"""Document listing (b200sa_docs_list_index_dev, b200sa_docs_list_dev, DocumentSuffixTable.documents*) against
the numpy model of tests/model_docs_list.py, brute force, and the occurrence route (positions_batch + locate +
np.unique), which shares no kernel with the listing."""
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, DocumentSuffixTree, SuffixTable, _lib, gen
from tests import model_docs, model_docs_list
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG = -1


def _u32(t, n):
    return t.cpu().numpy().view(np.uint32)[:n]


def _list_ranges(ctx, st, s, e, cap, with_tf=True, fill=-1):
    """The C-ABI on explicit ranges: (total, offsets, docs, tf) with docs / tf buffers of max(cap, 1) entries
    pre-filled with `fill` (returned whole, so that writes past the listing show)."""
    byd, prev = st._list_arrays()
    _, d_g, d_s = st._device_arrays()
    s = np.asarray(s, np.uint32)
    e = np.asarray(e, np.uint32)
    nq = len(s)
    d_start = torch.from_numpy(s.view(np.int32).copy()).cuda()
    d_end = torch.from_numpy(e.view(np.int32).copy()).cuda()
    d_off = torch.full((nq + 1,), -1, dtype=torch.int64, device="cuda")
    d_docs = torch.full((max(cap, 1),), fill, dtype=torch.int32, device="cuda")
    d_tf = torch.full((max(cap, 1),), fill, dtype=torch.int32, device="cuda")
    total = ctx.docs_list_dev(len(st), d_g.data_ptr(), d_s.data_ptr(), len(st.doc_starts()), byd.data_ptr(),
                              prev.data_ptr(), d_start.data_ptr(), d_end.data_ptr(), nq, d_off.data_ptr(),
                              d_docs.data_ptr() if cap else 0, d_tf.data_ptr() if cap and with_tf else 0, cap,
                              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return (total, d_off.cpu().numpy().view(np.uint64), d_docs.cpu().numpy().view(np.uint32),
            d_tf.cpu().numpy().view(np.uint32))


def _want_ranges(st, s, e):
    """Listing of ranges of G by first occurrence: (docs, tf) per range, in rank order of first occurrence."""
    starts = st.doc_starts()
    doc = np.searchsorted(starts, st.table(), side="right") - 1
    out = []
    for a, b in zip(s, e):
        d, first, cnt = np.unique(doc[int(a):int(b)], return_index=True, return_counts=True)
        o = np.argsort(first)
        out.append((d[o].astype(np.uint32), cnt[o].astype(np.uint32)))
    return out


def _check_ranges(ctx, st, s, e):
    want = _want_ranges(st, s, e)
    tot = sum(len(d) for d, _ in want)
    for with_tf in (True, False):
        total, off, docs, tf = _list_ranges(ctx, st, s, e, tot, with_tf)
        assert total == tot
        assert np.array_equal(np.diff(off.astype(np.int64)), [len(d) for d, _ in want]) and off[0] == 0
        assert np.array_equal(docs[:tot], np.concatenate([d for d, _ in want] + [np.zeros(0, np.uint32)]))
        if with_tf:
            assert np.array_equal(tf[:tot], np.concatenate([t for _, t in want] + [np.zeros(0, np.uint32)]))
        else:
            assert (tf == 0xFFFFFFFF).all()                       # d_tf NULL: nothing written


def test_index_equals_model_on_families():
    rng = np.random.default_rng(11)
    sets = _families(rng)
    assert len(sets) >= 300
    for docs in sets:
        st = DocumentSuffixTable(docs)
        g, _, byd, prev = model_docs_list.index(docs)
        assert np.array_equal(st.table(), g), docs
        d_byd, d_prev = st._list_arrays()
        assert np.array_equal(_u32(d_byd, len(g)), byd), docs
        assert np.array_equal(_u32(d_prev, len(g)), prev), docs


def test_listing_against_brute_force_on_families():
    rng = np.random.default_rng(12)
    ctx = _lib.Context(0)
    for docs in _families(rng):
        st = DocumentSuffixTable(docs)
        qs = sorted({x[a:a + m] for x in docs for m in range(1, 4) for a in range(len(x) - m + 1)})
        qs += [b"", b"zz", b"\x01\x02"]
        g, doc, byd, prev = model_docs_list.index(docs)
        text, starts = model_docs.concat(docs)
        ranges = [model_docs_list.query_range(docs, g, q) for q in qs]
        s_arr, e_arr = st.positions_batch(qs)
        for (a, b), (ws, we) in zip(zip(s_arr.tolist(), e_arr.tolist()), ranges):
            assert (a, b) == (ws, we) or (a == b and ws == we), docs   # an empty range may sit anywhere
        want = [model_docs_list.listing(starts, len(text), doc, byd, prev, a, b) for a, b in ranges]
        tot = sum(len(w) for w in want)
        # the C-ABI order (rank order), with and without tf
        for with_tf in (True, False):
            total, off, d_docs, d_tf = _list_ranges(ctx, st, s_arr, e_arr, tot, with_tf)
            assert total == tot
            assert np.diff(off.astype(np.int64)).tolist() == [len(w) for w in want]
            assert d_docs[:tot].tolist() == [d for w in want for _, d, _ in w], docs
            if with_tf:
                assert d_tf[:tot].tolist() == [t for w in want for _, _, t in w], docs
        # the Python API: document order, counts by brute force
        off, dd, tf = st.documents_batch(qs)
        for k, q in enumerate(qs):
            rows = list(zip(dd[off[k]:off[k + 1]].tolist(), tf[off[k]:off[k + 1]].tolist()))
            brute = [(d, _count(x, q)) for d, x in enumerate(docs) if q and q in x]
            assert rows == brute, (docs, q)
        assert st.document_frequencies(qs).tolist() == [len(w) for w in want]
    ctx.close()


def _count(doc: bytes, q: bytes) -> int:
    k, i = 0, doc.find(q)
    while i >= 0:
        k += 1
        i = doc.find(q, i + 1)
    return k


@pytest.mark.parametrize("n", [31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769])
def test_chunk_and_level_edges(n):
    rng = np.random.default_rng(n)
    t = bytes(rng.choice(list(b"ab"), n))
    cuts = np.unique(rng.integers(1, n, max(1, n // 40)))
    docs = [t[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, n])]
    docs.insert(1, b"")
    st = DocumentSuffixTable(docs)
    assert len(st) == n
    pts = {0, n}
    for m in list(range(1024, n + 2, 1024)) + [int(x) * 32 for x in rng.integers(1, n // 32 + 2, 24)]:
        pts |= {m - 1, m, m + 1}
    pts = sorted(p for p in pts if 0 <= p <= n)
    pairs = [(a, b) for a in pts for b in pts if a <= b]
    if len(pairs) > 3000:
        pairs = [pairs[int(k)] for k in rng.choice(len(pairs), 3000, replace=False)]
    pairs.append((0, n))                                           # all of G
    s, e = zip(*pairs)
    ctx = _lib.Context(0)
    _check_ranges(ctx, st, s, e)
    ctx.close()


def test_acgt_copies():
    st = DocumentSuffixTable([b"ACGT"] * 100_000)
    off, docs, tf = st.documents_batch([b"A", b"ACGTA", b"GT"])
    assert off.tolist() == [0, 100_000, 100_000, 200_000]
    assert np.array_equal(docs[:100_000], np.arange(100_000)) and (tf == 1).all()
    # the C-ABI order of b"A" is already document order (equal suffixes sort by document)
    ctx = _lib.Context(0)
    s, e = st.positions_batch([b"A"])
    total, _, d_docs, _ = _list_ranges(ctx, st, s, e, 100_000)
    assert total == 100_000 and np.array_equal(d_docs, np.arange(100_000))
    ctx.close()
    assert st.document_frequencies([b"A", b"ACGTA", b"", b"CGTAC"]).tolist() == [100_000, 0, 0, 0]
    rows = st.documents(b"CG")
    assert rows.shape == (100_000, 2) and (rows[:, 1] == 1).all()


def _scale_docs():
    rng = np.random.default_rng(21)
    t = _u8(gen.dna(4 << 20))
    cuts = np.unique(rng.integers(1, len(t), 3000))
    docs = [t[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for k in rng.integers(0, len(docs), 40):
        docs.insert(int(rng.integers(0, len(docs) + 1)), docs[int(k)])
    docs.insert(5, b"")
    return t, docs


def test_scale_mixed_batch_against_occurrences():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs)
    rng = np.random.default_rng(22)
    qs = []
    for _ in range(50_000):
        a = int(rng.integers(0, len(t) - 16))
        qs.append(t[a:a + int(rng.integers(4, 17))])
    qs += [b"A", b"C"]
    off, dd, tf = st.documents_batch(qs)
    # the occurrence route: every occurrence located, then (query, document) counted
    s, e = st.positions_batch(qs)
    lens = (e.astype(np.int64) - s)
    qid = np.repeat(np.arange(len(qs), dtype=np.int64), lens)
    ranks = np.concatenate([np.arange(a, b) for a, b in zip(s.tolist(), e.tolist())])
    loc = st.locate(st.table()[ranks])
    key, cnt = np.unique((qid << 32) | loc[:, 0].astype(np.int64), return_counts=True)
    assert len(dd) == len(key) and int(off[-1]) == len(key)
    assert np.array_equal((key >> 32), np.repeat(np.arange(len(qs)), np.diff(off.astype(np.int64))))
    assert np.array_equal(dd, (key & 0xFFFFFFFF).astype(np.uint32))
    assert np.array_equal(tf, cnt.astype(np.uint32))
    nonempty = sum(1 for d in docs if d)
    assert np.diff(off.astype(np.int64))[-2] <= nonempty and np.diff(off.astype(np.int64))[-2] > nonempty // 2
    # document frequencies without the tree equal the tree's
    df = st.document_frequencies(qs)
    assert np.array_equal(df, np.diff(off.astype(np.int64)).astype(np.uint32))
    tree = DocumentSuffixTree.from_document_table(st)
    assert np.array_equal(df, tree.document_counts(qs))


def test_cap_paths_and_bad_ranges():
    t, docs = _scale_docs()
    docs = docs[:300]
    st = DocumentSuffixTable(docs)
    s, e = st.positions_batch([b"ACG", b"T", b"GGGGGGGGGGGGGGGGGGGGGG", b"CA"])
    ctx = _lib.Context(0)
    total, off0, docs0, _ = _list_ranges(ctx, st, s, e, 0)
    assert total > 0 and int(off0[-1]) == total
    for cap in (total - 1, 1):                                     # too small: offsets only
        tot, off, dd, tf = _list_ranges(ctx, st, s, e, cap)
        assert tot == total and np.array_equal(off, off0)
        assert (dd == 0xFFFFFFFF).all() and (tf == 0xFFFFFFFF).all()
    tot, off, dd, tf = _list_ranges(ctx, st, s, e, total)
    assert tot == total and np.array_equal(off, off0)
    assert np.array_equal(dd, np.concatenate([w[0] for w in _want_ranges(st, s, e)]))
    n = len(st)
    for bad_s, bad_e in ((5, 4), (0, n + 1), (n, n + 7)):
        with pytest.raises(_lib.B200SAError) as ex:
            _list_ranges(ctx, st, [0, bad_s], [3, bad_e], 16)
        assert ex.value.code == BAD_ARG and "docs list" in str(ex.value)
    # the context still works, and reports the phases
    ctx.set_timing(True)
    tot, off, dd, _ = _list_ranges(ctx, st, s, e, total)
    names = [p for p, _ in ctx.phase_times()]
    ctx.set_timing(False)
    assert tot == total and np.array_equal(off, off0)
    for p in ("dlist_levels", "dlist_count", "dlist_scan", "dlist_emit"):
        assert p in names, names
    # nq = 0 writes offsets[0] = 0
    tot, off, _, _ = _list_ranges(ctx, st, [], [], 4)
    assert tot == 0 and off.tolist() == [0]
    ctx.close()


def test_index_entry_checks_doc_starts():
    ctx = _lib.Context(0)
    text = b"abcdef"
    g = torch.zeros(6, dtype=torch.int32, device="cuda")
    out = torch.empty(12, dtype=torch.int32, device="cuda")
    for starts in ([1, 3], [0, 4, 2], [0, 3, 7]):
        d_s = torch.tensor(starts, dtype=torch.int32, device="cuda")
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.docs_list_index_dev(len(text), g.data_ptr(), d_s.data_ptr(), len(starts), out.data_ptr(),
                                    out.data_ptr() + 24, torch.cuda.current_stream().cuda_stream)
        assert ex.value.code == BAD_ARG and "doc_starts" in str(ex.value)
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.docs_list_index_dev(6, g.data_ptr(), 0, 0, out.data_ptr(), out.data_ptr() + 24, 0)
    assert ex.value.code == BAD_ARG
    ctx.set_timing(True)
    st = DocumentSuffixTable([b"abc", b"", b"cab"])
    d_g, d_s = st._device_arrays()[1:]
    ctx.docs_list_index_dev(6, d_g.data_ptr(), d_s.data_ptr(), 3, out.data_ptr(), out.data_ptr() + 24,
                            torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    names = [p for p, _ in ctx.phase_times()]
    for p in ("docs_check", "dlist_len", "dlist_sort", "dlist_prev"):
        assert p in names, names
    _, _, byd, prev = model_docs_list.index([b"abc", b"", b"cab"])
    assert np.array_equal(_u32(out, 6), byd) and np.array_equal(out.cpu().numpy().view(np.uint32)[6:], prev)
    ctx.close()


def test_empty_and_tiny_tables():
    e = DocumentSuffixTable([])
    off, dd, tf = e.documents_batch([b"a", b""])
    assert off.tolist() == [0, 0, 0] and len(dd) == 0 and len(tf) == 0
    assert e.document_frequencies([b"a"]).tolist() == [0]
    assert e.documents(b"a").shape == (0, 2)
    one = DocumentSuffixTable([b"", b"z", b""])
    assert one.documents(b"z").tolist() == [[1, 1]] and one.documents(b"").shape == (0, 2)
    assert one.documents_batch([]) [0].tolist() == [0]


def test_wrapper_keeps_index_and_retries_small_cap():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:500])
    qs = [b"ACGT", b"A", b"TTT", b"GATTACA"]
    a = st.documents_batch(qs)
    idx = st._dlist
    b = st.documents_batch(qs, _cap_guess=1)                      # too small: the second call sizes the buffers
    assert st._dlist is idx
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_concurrent_listing_with_suffix_table_builds():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:800])
    rng = np.random.default_rng(5)
    qs = []
    for _ in range(3000):
        a = int(rng.integers(0, len(t) - 12))
        qs.append(t[a:a + int(rng.integers(3, 12))])
    want = st.documents_batch(qs)
    want_df = st.document_frequencies(qs)
    text = _u8(gen.english(300_000))
    want_t = SuffixTable(text).table()
    errors = []

    def run(fn):
        try:
            for _ in range(5):
                fn()
        except Exception as ex:
            errors.append(ex)

    def listing():
        got = st.documents_batch(qs)
        assert all(np.array_equal(x, y) for x, y in zip(got, want))
        assert np.array_equal(st.document_frequencies(qs), want_df)

    def build():
        assert np.array_equal(SuffixTable(text).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (listing, listing, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
