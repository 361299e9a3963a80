"""Repeat lengths, runs and duplicate spans (b200sa_repeat_lens_dev, b200sa_repeat_runs_dev,
b200sa_duplicate_spans_dev, SuffixTable / DocumentSuffixTable .repeat_lengths, .repeated_substrings,
.duplicate_spans, .duplicated_bytes) against the numpy model of tests/model_repeats.py and, at scale, the
serial C statement of tests/repeats_check.c."""
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import model_docs, model_repeats as mr, repeats_check
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_docs_list import _scale_docs

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
MARK = 0xA5A5A5A5
SCAN_CHUNK = 4096
NAMES = ("any", "earlier", "other_document", "earlier_document")


def _dev(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return torch.from_numpy((a if len(a) else np.zeros(1, np.uint32)).view(np.int32).copy()).cuda()


def _marked(k):
    return torch.full((max(k, 1),), MARK - (1 << 32), dtype=torch.int32, device="cuda")


def _host(t):
    return t.cpu().numpy().view(np.uint32)


class _Abi:
    """The C-ABI on host arrays: the table and its LCP array go to the device once."""

    def __init__(self, ctx, g, lcp, starts=None):
        self.ctx, self.n = ctx, len(g)
        self.g, self.lcp = _dev(g), _dev(lcp)
        self.starts = None if starts is None else _dev(starts)
        self.ndocs = 0 if starts is None else len(starts)
        self.stream = torch.cuda.current_stream().cuda_stream       # 0: the context's own stream, which does not
        torch.cuda.synchronize()                                     # wait for torch's -- hence the synchronises

    def lens(self):
        out = _marked(self.n)
        torch.cuda.synchronize()
        self.ctx.repeat_lens_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), out.data_ptr(), self.stream)
        torch.cuda.synchronize()
        return _host(out)[:self.n]

    def runs(self, L, cap=None, ends=True):
        """(total, start, end, first, last): buffers of max(cap, 1) entries pre-filled with MARK; cap = None
        counts first and fetches into buffers of exactly that size."""
        if cap is None:
            cap = self.ctx.repeat_runs_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), L, stream=self.stream)
        out = [_marked(cap) for _ in range(4)]
        ptrs = [o.data_ptr() if cap and (ends or k < 2) else 0 for k, o in enumerate(out)]
        torch.cuda.synchronize()
        total = self.ctx.repeat_runs_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), L, *ptrs, cap, self.stream)
        return (total,) + tuple(_host(o) for o in out)

    def spans(self, L, mode, cap=None):
        """(total, covered, begin, end), the buffers as for runs."""
        args = (self.n, self.g.data_ptr(), self.lcp.data_ptr(), self.starts.data_ptr() if self.ndocs else 0, self.ndocs,
                L, mode)
        if cap is None:
            cap = self.ctx.duplicate_spans_dev(*args, stream=self.stream)[0]
        b, e = _marked(cap), _marked(cap)
        torch.cuda.synchronize()
        total, cov = self.ctx.duplicate_spans_dev(*args, b.data_ptr() if cap else 0, e.data_ptr() if cap else 0, cap,
                                                  self.stream)
        return total, cov, _host(b), _host(e)


def _check_abi(abi, g, lcp, starts, lens, modes, want_spans=None):
    """Every entry point of `abi` against the model (or want_spans(L, mode)) at every L and mode."""
    assert np.array_equal(abi.lens(), mr.repeat_lens(g, lcp))
    for L in lens:
        want = mr.runs(g, lcp, L)
        got = abi.runs(L)
        k = len(want[0])
        assert got[0] == k and all(np.array_equal(a[:k], b) for a, b in zip(got[1:], want)), L
        for m in modes:
            wb, we, wcov = want_spans(L, m) if want_spans else mr.duplicate_spans(g, lcp, starts, L, m)
            total, cov, b, e = abi.spans(L, m)
            assert (total, cov) == (len(wb), wcov), (L, m)
            assert np.array_equal(b[:total], wb) and np.array_equal(e[:total], we), (L, m)


def _rows(starts, begin, end):
    """(document, begin_offset, end_offset) rows of spans given in coordinates of the concatenation."""
    d = np.searchsorted(starts, begin, side="right") - 1
    s = np.asarray(starts, dtype=np.uint32)[d] if len(begin) else np.zeros(0, np.uint32)
    return np.stack([d.astype(np.uint32), begin - s, end - s], axis=1).astype(np.uint32).reshape(-1, 3)


def _check_docs_class(st, docs, lens):
    g, lcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    assert np.array_equal(st.repeat_lengths(), mr.repeat_lens(g, lcp)), docs
    for L in lens:
        want = mr.runs(g, lcp, L)
        assert all(np.array_equal(a, b) for a, b in zip(st.repeated_substrings(L, with_ends=True), want)), (docs, L)
        assert all(np.array_equal(a, b) for a, b in zip(st.repeated_substrings(L), want[:2])), (docs, L)
        for m, name in enumerate(NAMES):
            wb, we, wcov = mr.duplicate_spans(g, lcp, starts, L, m) if len(g) else (g, g, 0)
            assert np.array_equal(st.duplicate_spans(L, name), _rows(starts, wb, we)), (docs, L, name)
            assert st.duplicated_bytes(L, name) == wcov, (docs, L, name)


def test_abi_and_classes_equal_model_on_families():
    rng = np.random.default_rng(81)
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for docs in sets:
        g, glcp = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        n = len(text)
        lens = sorted({1, 2, 3, 8, max(n, 1), n + 1})
        if len(docs):
            _check_abi(_Abi(ctx, g, glcp, starts), g, glcp, starts, lens, mr.MODES)
        _check_docs_class(DocumentSuffixTable(docs), docs, (1, 3, n + 1))
        if len(docs) == 1:                                     # one document is the single text
            sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
            assert np.array_equal(sa, g) and np.array_equal(lcp, glcp)
            _check_abi(_Abi(ctx, sa, lcp), sa, lcp, None, lens, (mr.ANY, mr.EARLIER))
            t1, st = SuffixTable(text), DocumentSuffixTable(docs)
            assert np.array_equal(t1.repeat_lengths(), st.repeat_lengths())
            for L in (1, 2, 3):
                assert all(np.array_equal(a, b) for a, b in zip(t1.repeated_substrings(L, True),
                                                                st.repeated_substrings(L, True)))
                for name in NAMES[:2]:
                    b, e = t1.duplicate_spans(L, name)
                    assert np.array_equal(_rows([0], b, e), st.duplicate_spans(L, name)), (docs, L, name)
                    assert t1.duplicated_bytes(L, name) == st.duplicated_bytes(L, name)
    ctx.close()


def test_definition_on_a_sample_of_the_families():
    rng = np.random.default_rng(82)
    for docs in [d for d in _families(rng) if 0 < sum(map(len, d)) <= 40][::4]:
        st = DocumentSuffixTable(docs)
        assert np.array_equal(st.repeat_lengths(), mr.brute_repeat_lens(docs)), docs
        for L in (1, 2, 4):
            flags = mr.brute_flags(docs, L)
            for m, name in enumerate(NAMES):
                wb, we, wcov = mr.spans_of_flags(docs, flags[m], L)
                assert np.array_equal(st.duplicate_spans(L, name), _rows(st.doc_starts(), wb, we)), (docs, L, name)


def test_one_run_over_everything():
    ctx = _lib.Context(0)
    for text in (b"a" * 70_001, b"ab" * 35_000):
        sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
        n = len(text)
        _check_abi(_Abi(ctx, sa, lcp), sa, lcp, None, (1, 2, 5000, n - 1, n, n + 1, 0xFFFFFFFF), (mr.ANY, mr.EARLIER),
                   want_spans=lambda L, m: repeats_check.spans(sa, lcp, None, L, m))
        abi = _Abi(ctx, sa, lcp)
        total, start, end, first, last = abi.runs(1)
        if text[:2] == b"aa":                                  # one run of n ranks
            assert (total, start[0], end[0], first[0], last[0]) == (1, 0, n, 0, n - 1)
            assert abi.spans(3, mr.ANY)[:2] == (1, n) and abi.spans(3, mr.EARLIER)[:2] == (1, n - 1)
    # 10^5 copies of ACGT: one run per gram, spanning every document
    docs = [b"ACGT"] * 100_000
    st = DocumentSuffixTable(docs)
    g, lcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    n = len(g)
    abi = _Abi(ctx, g, lcp, starts)
    for L in (1, 2, 4):
        total, start, end, first, last = abi.runs(L)
        assert total == 5 - L and np.all(end[:total] - start[:total] == 100_000)
        assert sorted(first[:total].tolist()) == list(range(5 - L)) and np.all(last[:total] - first[:total] == n - 4)
        assert abi.spans(L, mr.OTHER_DOC)[:2] == (100_000, n)              # everything, one span per document
        total, cov, b, e = abi.spans(L, mr.EARLIER_DOC)                    # everything but document 0
        assert (total, cov, b[0], e[total - 1]) == (99_999, n - 4, 4, n)
    assert abi.spans(5, mr.ANY)[:2] == (0, 0)
    _check_abi(abi, g, lcp, starts, (1, 3, 4), mr.MODES)
    assert st.duplicated_bytes(4, "earlier_document") == n - 4
    rows = st.duplicate_spans(4, "earlier")
    assert len(rows) == 99_999 and rows[0].tolist() == [1, 0, 4] and rows[-1].tolist() == [99_999, 0, 4]
    ctx.close()


def _synthetic(rng, n, L, runs):
    """A random permutation as the table and an LCP array whose runs at L are exactly `runs` ([a, b) rank
    ranges) plus random short ones elsewhere: the entry points take the arrays as given."""
    g = rng.permutation(n).astype(np.uint32)
    lcp = np.where(rng.random(n) < 0.3, L, rng.integers(0, L, n)).astype(np.uint32)
    for a, b in runs:
        lcp[a] = 0
        lcp[a + 1:b] = rng.integers(L, L + 3, max(b - a - 1, 0))
        if b < n:
            lcp[b] = L - 1
    lcp[0] = 0
    return g, lcp


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 255, 256, 257, 1023, 1025, SCAN_CHUNK - 1, SCAN_CHUNK, SCAN_CHUNK + 1,
                               2 * SCAN_CHUNK - 1, 2 * SCAN_CHUNK + 1, 32767, 32769])
def test_lengths_and_tile_edges(n):
    """Runs that start, end and straddle exactly at the scan's tile edges, and one over all ranks: the
    segment's extremes have to arrive across any number of tiles."""
    rng = np.random.default_rng(83 + n)
    ctx = _lib.Context(0)
    T = SCAN_CHUNK
    shapes = [[], [(0, n)],
              [(a, b) for a, b in ((T - 7, T), (T, T + 9), (2 * T - 3, 2 * T + 3), (2 * T + 3, 5 * T), (5 * T + 1, 6 * T - 1))
               if b <= n],
              [(a, b) for a, b in ((0, T + 1), (T + 1, 3 * T), (3 * T, 3 * T + 2), (7 * T - 1, n)) if a + 2 <= b <= n]]
    for runs in shapes:
        g, lcp = _synthetic(rng, n, 4, runs)
        cuts = np.unique(np.r_[0, rng.integers(0, n + 1, 6), 0 if n < T else T]).astype(np.uint32)
        _check_abi(_Abi(ctx, g, lcp, cuts), g, lcp, cuts, (4,), mr.MODES)
        _check_abi(_Abi(ctx, g, lcp), g, lcp, None, (3, 4, 5), (mr.ANY, mr.EARLIER))
    ctx.close()


def test_touching_spans_and_empty_documents():
    for docs, want in (([b"abab"], [(0, 0, 4)]), ([b"ab", b"ab"], [(0, 0, 2), (1, 0, 2)]),
                       ([b"", b"ab", b"", b"", b"ab", b""], [(1, 0, 2), (4, 0, 2)]),
                       ([b"", b"xabx", b"", b"yaby", b""], [(1, 1, 3), (3, 1, 3)])):
        st = DocumentSuffixTable(docs)
        assert st.duplicate_spans(2).tolist() == [list(w) for w in want], docs
        assert st.duplicated_bytes(2) == 4
        assert st.duplicate_spans(2, "earlier_document").tolist() == ([list(want[-1])] if len(docs) > 1 else [])
    t = SuffixTable(b"abcabcXabc")
    assert [x.tolist() for x in t.duplicate_spans(3)] == [[0, 7], [6, 10]]
    assert [x.tolist() for x in t.duplicate_spans(3, "earlier")] == [[3, 7], [6, 10]]
    assert t.duplicated_bytes(3, "earlier") == 6 and t.duplicated_bytes(0xFFFFFFFF) == 0 and t.duplicated_bytes(1 << 40) == 0


def test_scale_against_the_serial_checker():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs)
    g, lcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    ctx = _lib.Context(0)
    abi = _Abi(ctx, g, lcp, starts)
    assert np.array_equal(abi.lens(), mr.repeat_lens(g, lcp))
    for L in (12, 20, 50):
        want = repeats_check.runs(g, lcp, L)
        got = abi.runs(L)
        assert got[0] == len(want[0]) and all(np.array_equal(a, b) for a, b in zip(got[1:], want)), L
        for m in mr.MODES:
            wb, we, wcov = repeats_check.spans(g, lcp, starts, L, m)
            total, cov, b, e = abi.spans(L, m)
            assert (total, cov) == (len(wb), wcov) and np.array_equal(b, wb) and np.array_equal(e, we), (L, m)
    rows = st.duplicate_spans(50, "earlier_document")
    wb, we, wcov = repeats_check.spans(g, lcp, starts, 50, mr.EARLIER_DOC)
    assert np.array_equal(rows, _rows(starts, wb, we)) and wcov > 40 * 50     # the planted copies
    assert st.duplicated_bytes(50, "earlier_document") == wcov
    # the single text
    t1 = SuffixTable(t)
    sa, lcp1 = t1.table(), t1.lcp_lens()
    assert np.array_equal(t1.repeat_lengths(), mr.repeat_lens(sa, lcp1))
    for L in (12, 20):
        assert all(np.array_equal(a, b) for a, b in zip(t1.repeated_substrings(L, True), repeats_check.runs(sa, lcp1, L)))
        for m, name in enumerate(NAMES[:2]):
            wb, we, wcov = repeats_check.spans(sa, lcp1, None, L, m)
            b, e = t1.duplicate_spans(L, name)
            assert np.array_equal(b, wb) and np.array_equal(e, we) and t1.duplicated_bytes(L, name) == wcov
    ctx.close()


def test_fixture_100k():
    t = _u8(gen.fixture("AP009048_100000.fasta"))
    t1 = SuffixTable(t)
    sa, lcp = t1.table(), t1.lcp_lens()
    assert np.array_equal(t1.repeat_lengths(), mr.repeat_lens(sa, lcp))
    for L in (8, 12, 20):
        assert all(np.array_equal(a, b) for a, b in zip(t1.repeated_substrings(L, True), mr.runs(sa, lcp, L)))
        for m, name in enumerate(NAMES[:2]):
            wb, we, wcov = repeats_check.spans(sa, lcp, None, L, m)
            mb, me, mcov = mr.duplicate_spans(sa, lcp, None, L, m)
            assert np.array_equal(wb, mb) and np.array_equal(we, me) and wcov == mcov    # the two statements agree
            b, e = t1.duplicate_spans(L, name)
            assert np.array_equal(b, wb) and np.array_equal(e, we) and t1.duplicated_bytes(L, name) == wcov


def test_runs_are_position_ranges_and_feed_the_listing():
    t, docs = _scale_docs()
    docs = docs[:600]
    st = DocumentSuffixTable(docs)
    text, g = st.text(), st.table()
    rng = np.random.default_rng(84)
    for L in (6, 12):
        start, end, first, last = st.repeated_substrings(L, with_ends=True)
        pick = np.sort(rng.choice(len(start), min(len(start), 3000), replace=False))
        qs = [text[int(p):int(p) + L] for p in first[pick]]
        s, e = st.positions_batch(qs)
        assert np.array_equal(s, start[pick]) and np.array_equal(e, end[pick]), L
        assert all(np.array_equal(a, b) for a, b in zip(st.documents_for_ranges(start[pick], end[pick]),
                                                        st.documents_batch(qs)))
        assert all(np.array_equal(a, b) for a, b in zip(st.top_documents_for_ranges(start[pick], end[pick], 3),
                                                        st.top_documents_batch(qs, 3)))
    with pytest.raises(ValueError):
        st.duplicate_spans(0)
    with pytest.raises(ValueError):
        st.duplicate_spans(3, "later")
    with pytest.raises(ValueError):
        st.repeated_substrings(-1)
    with pytest.raises(ValueError):
        SuffixTable(b"abab").duplicate_spans(2, "other_document")
    with pytest.raises(ValueError):
        SuffixTable(b"abab").duplicated_bytes(0)


def test_cap_protocol():
    ctx = _lib.Context(0)
    docs = [b"abcabc", b"", b"bcabca", b"zz"]
    g, lcp = model_docs.brute(docs)
    _, starts = model_docs.concat(docs)
    abi = _Abi(ctx, g, lcp, starts)
    want = mr.runs(g, lcp, 2)
    k = len(want[0])
    assert k >= 3
    for cap in (0, 1, k - 1):                                  # too small: the total and nothing else
        got = abi.runs(2, cap)
        assert got[0] == k and all(np.all(a == MARK) for a in got[1:]), cap
    for cap in (k, k + 3):                                     # exact and larger: nothing past the total
        got = abi.runs(2, cap)
        assert got[0] == k and all(np.array_equal(a[:k], b) and np.all(a[k:] == MARK) for a, b in zip(got[1:], want))
    got = abi.runs(2, k, ends=False)                           # first / last are optional
    assert np.array_equal(got[1], want[0]) and np.array_equal(got[2], want[1])
    assert np.all(got[3] == MARK) and np.all(got[4] == MARK)
    for m in mr.MODES:
        wb, we, wcov = mr.duplicate_spans(g, lcp, starts, 2, m)
        k = len(wb)
        assert k >= 1
        for cap in sorted({0, k - 1}):
            total, cov, b, e = abi.spans(2, m, cap)
            assert (total, cov) == (k, wcov) and np.all(b == MARK) and np.all(e == MARK), (m, cap)
        for cap in (k, k + 5):
            total, cov, b, e = abi.spans(2, m, cap)
            assert (total, cov) == (k, wcov) and np.array_equal(b[:k], wb) and np.array_equal(e[:k], we)
            assert np.all(b[k:] == MARK) and np.all(e[k:] == MARK)
    ctx.close()


def test_abi_errors_and_empty_inputs():
    ctx = _lib.Context(0)
    d = torch.zeros(64, dtype=torch.int32, device="cuda")
    d[1] = 3                                                   # doc_starts = [0, 3, 0, ...] is not ascending
    p = d.data_ptr()
    for k in (1, 2, 3):                                        # (n, sa, lcp, rl)
        args = [8, p, p, p]
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.repeat_lens_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), k
    for k in (1, 2, 4, 5):                                     # (n, sa, lcp, min_len, start, end, first, last, cap)
        args = [8, p, p, 2, p, p, 0, 0, 4]
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.repeat_runs_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), k
    for k in (1, 2, 7, 8):                                     # (n, sa, lcp, starts, ndocs, min_len, mode, begin, end, cap)
        args = [8, p, p, p, 1, 2, 0, p, p, 4]
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.duplicate_spans_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), k
    for args, word in (([8, p, p, p, 1, 0, 0, p, p, 4], "min_len"), ([8, p, p, p, 1, 2, 4, p, p, 4], "mode"),
                       ([8, p, p, p, 1, 2, -1, p, p, 4], "mode"), ([8, p, p, 0, 0, 2, 2, p, p, 4], "doc_starts"),
                       ([8, p, p, 0, 0, 2, 3, p, p, 4], "doc_starts"), ([8, p, p, 0, 1, 2, 0, p, p, 4], "null"),
                       ([8, p, p, p, 0, 2, 0, p, p, 4], "ndocs == 0"), ([8, p, p, p, 3, 2, 0, p, p, 4], "doc_starts"), ([8, p, p, p, 3, 2, 3, 0, 0, 0], "doc_starts")):
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.duplicate_spans_dev(*args)
        assert ex.value.code == BAD_ARG and word in str(ex.value), args
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.repeat_runs_dev(8, p, p, 0, p, p, 0, 0, 4)
    assert ex.value.code == BAD_ARG and "min_len" in str(ex.value)
    for call in (lambda: ctx.repeat_lens_dev(1 << 33, p, p, p), lambda: ctx.repeat_runs_dev(1 << 33, p, p, 2, p, p, 0, 0, 4),
                 lambda: ctx.duplicate_spans_dev(1 << 33, p, p, 0, 0, 2, 0, p, p, 4)):
        with pytest.raises(_lib.B200SAError) as ex:
            call()
        assert ex.value.code == TOO_LARGE
    # the context still works; n = 0 gives totals 0; the phases have names of their own
    g, lcp = model_docs.brute([b"abab", b"ab"])
    abi = _Abi(ctx, g, lcp, [0, 4])
    _check_abi(abi, g, lcp, np.asarray([0, 4]), (1, 2), mr.MODES)
    assert ctx.repeat_runs_dev(0, 0, 0, 2) == 0 and ctx.duplicate_spans_dev(0, 0, 0, 0, 0, 2, 0) == (0, 0)
    assert ctx.duplicate_spans_dev(0, 0, 0, p, 2, 2, 3) == (0, 0)
    ctx.repeat_lens_dev(0, 0, 0, 0)
    ctx.set_timing(True)
    abi.lens()
    assert [x for x, _ in ctx.phase_times()] == ["rep_lens"]
    abi.runs(2)
    assert [x for x, _ in ctx.phase_times()] == ["rep_count", "rep_segments", "rep_emit"]
    abi.spans(2, mr.ANY)
    assert [x for x, _ in ctx.phase_times()] == ["rep_check", "rep_flag", "rep_cover", "rep_count", "rep_emit"]
    abi.spans(2, mr.OTHER_DOC, 0)
    assert [x for x, _ in ctx.phase_times()] == ["rep_check", "rep_segments", "rep_flag", "rep_cover", "rep_count"]
    ctx.close()
    # the classes on empty tables
    for e in (DocumentSuffixTable([]), DocumentSuffixTable([b"", b""]), SuffixTable(b"")):
        assert len(e.repeat_lengths()) == 0 and e.duplicated_bytes(1) == 0
        assert [len(x) for x in e.repeated_substrings(1, True)] == [0, 0, 0, 0]
        assert len(e.duplicate_spans(1)[0]) == 0 if isinstance(e, SuffixTable) else e.duplicate_spans(1).shape == (0, 3)


def test_concurrent_spans_with_suffix_table_builds():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:800])
    g, glcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    want = {m: repeats_check.spans(g, glcp, starts, 12, m) for m in mr.MODES}
    want_runs = repeats_check.runs(g, glcp, 12)
    etext = _u8(gen.english(300_000))
    want_t = SuffixTable(etext).table()
    errors = []

    def run(fn):
        try:
            for _ in range(4):
                fn()
        except Exception as ex:
            errors.append(ex)

    def spans():                                                   # a context of its own per thread
        ctx = _lib.Context(0)
        abi = _Abi(ctx, g, glcp, starts)
        for m in mr.MODES:
            total, cov, b, e = abi.spans(12, m)
            assert (total, cov) == (len(want[m][0]), want[m][2])
            assert np.array_equal(b, want[m][0]) and np.array_equal(e, want[m][1])
        got = abi.runs(12)
        assert all(np.array_equal(a, b) for a, b in zip(got[1:], want_runs))
        ctx.close()

    def build():
        assert np.array_equal(SuffixTable(etext).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (spans, spans, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
