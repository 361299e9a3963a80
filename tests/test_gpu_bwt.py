"""The Burrows-Wheeler transform and its inverse (b200sa_bwt_dev, b200sa_unbwt_dev, SuffixTable /
DocumentSuffixTable .bwt and .bwt_runs, suffix_b200.inverse_bwt and .inverse_bwt_documents) against the
brute-force rotation sort and the numpy model of tests/model_bwt.py and, at scale, the serial C statement of
tests/bwt_check.c."""
import os
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen, inverse_bwt, inverse_bwt_documents
from tests import bwt_check, model_bwt as mb, model_docs
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_lz import _planted_docs

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
MARK8, MARK32 = 0xA5, 0xA5A5A5A5


class _ruler:
    """Forces the ruler spacing of the inverse (B200SA_BWT_RULER)."""

    def __init__(self, s):
        self.s = s

    def __enter__(self):
        os.environ["B200SA_BWT_RULER"] = str(self.s)

    def __exit__(self, *a):
        del os.environ["B200SA_BWT_RULER"]


def _dev32(a, size=None):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    buf = np.full(max(size or len(a), 1), MARK32, np.uint32)
    buf[:len(a)] = a
    return torch.from_numpy(buf.view(np.int32)).cuda()


def _dev8(b, size=None):
    b = np.frombuffer(bytes(b), dtype=np.uint8)
    buf = np.full(max(size or len(b), 1), MARK8, np.uint8)
    buf[:len(b)] = b
    return torch.from_numpy(buf).cuda()


def _host32(t):
    return t.cpu().numpy().view(np.uint32)


class _Abi:
    """Both entry points on host arrays, with output buffers pre-filled with markers and `pad` entries
    past the end."""

    def __init__(self, ctx, pad=5):
        self.ctx, self.pad = ctx, pad
        self.stream = torch.cuda.current_stream().cuda_stream

    def bwt(self, text, g, starts=None, runs=True):
        n = len(text)
        k = 1 if starts is None else len(starts)
        d_t, d_g = _dev8(text), _dev32(g)
        d_s = _dev32(starts) if starts is not None else None
        out, term = _dev8(b"", n + self.pad), _dev32([], k + self.pad)
        torch.cuda.synchronize()
        r = self.ctx.bwt_dev(n, d_t.data_ptr(), d_g.data_ptr(), d_s.data_ptr() if d_s is not None else 0,
                             0 if starts is None else len(starts), out.data_ptr(), term.data_ptr(), runs, self.stream)
        torch.cuda.synchronize()
        o, t = out.cpu().numpy(), _host32(term)
        assert np.all(o[n:] == MARK8) and np.all(t[k:] == MARK32)           # nothing past n bytes or k entries
        return o[:n].tobytes(), t[:k].tolist(), r

    def unbwt(self, bwt, term_rows, with_starts=True):
        """(text, starts) or the B200SAError; on an error the outputs must be untouched."""
        n, k = len(bwt), len(term_rows)
        d_b, d_t = _dev8(bwt), _dev32(term_rows)
        out, st = _dev8(b"", n + self.pad), _dev32([], k + self.pad)
        torch.cuda.synchronize()
        try:
            self.ctx.unbwt_dev(n, k, d_b.data_ptr(), d_t.data_ptr(), out.data_ptr(), st.data_ptr() if with_starts else 0,
                               self.stream)
            err = None
        except _lib.B200SAError as ex:
            err = ex
        torch.cuda.synchronize()
        o, s = out.cpu().numpy(), _host32(st)
        if err is not None or not with_starts:
            assert np.all(s == MARK32)
        if err is not None:
            assert np.all(o == MARK8)                                          # nothing at all on an error
            return err
        assert np.all(o[n:] == MARK8) and np.all(s[k:] == MARK32)
        return o[:n].tobytes(), s[:k].tolist()


def _docs_of(text, starts):
    ends = list(starts[1:]) + [len(text)]
    return [text[a:b] for a, b in zip(starts, ends)]


def _families_bwt(rng):
    sets = _families(rng)
    sets += [[b"", b"", b"ab", b"b"], [b"ab", b"", b"", b"b"], [b"ab", b"ba", b"", b""],   # empty first, middle, last
             [b"", b"", b"", b"x"], [b"x", b"", b"", b""], [b"", b"", b""] + [b"a"] * 3]  # starts at one offset
    return sets


def test_forward_and_inverse_equal_model_on_families():
    rng = np.random.default_rng(141)
    sets = _families_bwt(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    for docs in sets:
        docs = [bytes(d) for d in docs]
        text, starts = model_docs.concat(docs)
        want_b, want_t, _, want_r = mb.brute(docs)
        g, _ = model_docs.brute(docs)
        if docs:
            assert abi.bwt(text, g, starts) == (want_b, want_t, want_r), docs
            got_text, got_starts = abi.unbwt(want_b, want_t)
            assert got_text == text and got_starts == starts.tolist(), docs
            _, rec = mb.inverse(want_b, want_t)
            assert ctx.stats()["doubling_rounds"] == rec["rounds"], docs
        st = DocumentSuffixTable(docs)
        b, t = st.bwt()
        assert b == want_b and t.tolist() == want_t and st.bwt_runs() == want_r, docs
        if docs:
            assert inverse_bwt_documents(b, t) == docs
        if len(docs) == 1:                                                # one document is the single text
            s1 = SuffixTable(docs[0])
            assert s1.bwt() == (want_b, want_t[0]) and s1.bwt_runs() == want_r
            assert inverse_bwt(want_b, want_t[0]) == docs[0]
            assert abi.bwt(text, g) == abi.bwt(text, g, starts)
    ctx.close()


@pytest.mark.parametrize("text", [b"banana", b"abracadabra"])
def test_known_answers(text):
    from tests.test_bwt_model import KNOWN
    want = KNOWN[(text,)]
    st = SuffixTable(text)
    assert st.bwt() == (want[0], want[1][0]) and st.bwt_runs() == want[3]
    assert inverse_bwt(*st.bwt()) == text


def test_known_answer_documents():
    from tests.test_bwt_model import KNOWN
    want = KNOWN[(b"ab", b"", b"b")]
    st = DocumentSuffixTable([b"ab", b"", b"b"])
    b, t = st.bwt()
    assert (b, t.tolist(), st.bwt_runs()) == (want[0], want[1], want[3])
    assert inverse_bwt_documents(b, t) == [b"ab", b"", b"b"]


def test_tiny_inputs_and_phases():
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    assert abi.bwt(b"", []) == (b"", [0], 1)                               # n = 0: the term row alone
    assert abi.bwt(b"", [], np.zeros(3, np.uint32)) == (b"", [0, 1, 2], 3)
    assert abi.bwt(b"x", [0]) == (b"x", [1], 2)                            # n = 1: rows $x, x$
    assert abi.unbwt(b"", [0]) == (b"", [0]) and abi.unbwt(b"x", [1]) == (b"x", [0])
    assert abi.unbwt(b"", [0, 1, 2])[1] == [0, 0, 0]
    assert SuffixTable(b"").bwt() == (b"", 0) and SuffixTable(b"").bwt_runs() == 1
    assert inverse_bwt(b"", 0) == b""
    e = DocumentSuffixTable([])
    assert e.bwt()[0] == b"" and len(e.bwt()[1]) == 0 and e.bwt_runs() == 0
    ctx.set_timing(True)
    sa = SuffixTable(b"mississippi").table()
    abi.bwt(b"mississippi", sa)
    assert [x for x, _ in ctx.phase_times()] == ["bwt_gather", "bwt_compact"]
    abi.bwt(b"mississippi", sa, np.zeros(1, np.uint32))
    assert [x for x, _ in ctx.phase_times()] == ["bwt_check", "bwt_gather", "bwt_compact"]
    b, t = SuffixTable(b"mississippi").bwt()
    abi.unbwt(b, [t])
    assert [x for x, _ in ctx.phase_times()] == ["unbwt_sort", "unbwt_walk", "unbwt_rank", "unbwt_emit"]
    ctx.close()


def _scale_texts(n):
    return {"dna": _u8(gen.dna(n)), "bytes": _u8(gen.rand_bytes(n)), "english": _u8(gen.english(n))}


@pytest.mark.parametrize("n", [1_000_000, 10_000_000])
def test_round_trip_at_scale(n):
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    for name, text in _scale_texts(n).items():
        st = SuffixTable(text)
        b, primary = st.bwt()
        assert inverse_bwt(b, primary) == text, name
        if n >= 10_000_000:                                                # the serial statement at 10^7
            wb, wt, wr = bwt_check.forward(text, st.table())
            assert (b, primary, st.bwt_runs()) == (wb, int(wt[0]), wr), name
            assert bwt_check.inverse(b, [primary])[0] == text, name
        else:
            assert abi.unbwt(b, [primary]) == (text, [0]), name
    docs = _planted_docs(n, 142)
    st = DocumentSuffixTable(docs)
    b, t = st.bwt()
    assert inverse_bwt_documents(b, t) == docs
    if n >= 10_000_000:
        wb, wt, wr = bwt_check.forward(st.text(), st.table(), st.doc_starts())
        assert b == wb and np.array_equal(t, wt) and st.bwt_runs() == wr
        text, starts = bwt_check.inverse(b, t)
        assert text == st.text() and np.array_equal(starts, st.doc_starts())
    ctx.close()


@pytest.mark.parametrize("name", ["AP009048_10000.fasta", "AP009048_100000.fasta"])
def test_round_trip_fixtures(name):
    text = gen.fixture(name).tobytes()
    st = SuffixTable(text)
    b, primary = st.bwt()
    wb, wt, wr = bwt_check.forward(text, st.table())
    assert (b, primary, st.bwt_runs()) == (wb, int(wt[0]), wr)
    assert inverse_bwt(b, primary) == text


def test_round_trip_repetitive():
    a = b"a" * 1_000_000
    st = SuffixTable(a)
    b, primary = st.bwt()
    assert b == a and primary == 1_000_000 and st.bwt_runs() == 2            # L = a^n $ ... : rows $a^n first
    assert inverse_bwt(b, primary) == a
    docs = [b"ACGT"] * 100_000
    st = DocumentSuffixTable(docs)
    b, t = st.bwt()
    wb, wt, wr = bwt_check.forward(st.text(), st.table(), st.doc_starts())
    assert b == wb and np.array_equal(t, wt) and st.bwt_runs() == wr
    assert inverse_bwt_documents(b, t) == docs


def test_ruler_spacing_changes_no_output():
    rng = np.random.default_rng(143)
    cases = [[_u8(gen.dna(3000))], [_u8(gen.english(2000))], [b"a" * 500], _planted_docs(20_000, 144),
             [b"", b"ab", b"", b"ba", b""], [bytes(rng.integers(0, 256, 700, dtype=np.uint8))]]
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    for docs in cases:
        st = DocumentSuffixTable(docs)
        b, t = st.bwt()
        n = len(b)
        for s in (1, 2, 3, 64, n + 1, 1 << 31):
            with _ruler(s):
                got = abi.unbwt(b, t)
                assert got[0] == st.text() and np.array_equal(got[1], st.doc_starts()), s
                _, rec = mb.inverse(b, t, s)
                assert ctx.stats()["doubling_rounds"] == rec["rounds"], s
                if s > n:                                                  # the terminator rows alone
                    assert rec["rulers"] == len(docs)
    ctx.close()


def test_invalid_inputs_match_the_model():
    """Random (bwt, term_rows): BAD_ARG exactly where the model rejects; where the call succeeds, the
    transform of the decoded documents is the input."""
    rng = np.random.default_rng(145)
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    accepted = rejected = 0
    for it in range(600):
        n, k = int(rng.integers(0, 12)), int(rng.integers(1, 5))
        bwt = bytes(rng.choice(list(b"ab"), n).tolist())
        term_rows = rng.choice(n + k, k, replace=False).tolist() if it % 5 else \
            rng.integers(0, n + k + 2, k).tolist()
        want = mb.inverse_by_definition(bwt, term_rows)
        for s in (1, 3, 64):
            with _ruler(s):
                got = abi.unbwt(bwt, term_rows)
                assert mb.inverse(bwt, term_rows, s)[0] == want
            if want is None:
                assert isinstance(got, _lib.B200SAError) and got.code == BAD_ARG, (bwt, term_rows)
            else:
                assert _docs_of(*got) == want
                assert mb.brute(want)[:2] == (bwt, list(term_rows))
        if want is None:
            rejected += 1
            with pytest.raises(_lib.B200SAError):
                inverse_bwt_documents(bwt, term_rows)
        else:
            accepted += 1
            st = DocumentSuffixTable(want)
            b, t = st.bwt()
            assert b == bwt and t.tolist() == list(term_rows)
    assert accepted > 50 and rejected > 50
    ctx.close()


def test_abi_errors():
    ctx = _lib.Context(0)
    abi = _Abi(ctx)
    for term_rows in ([5], [0, 0], [1, 1, 2], [0, 9]):                      # out of range or repeated
        err = abi.unbwt(b"ab" if len(term_rows) == 1 else b"a", term_rows)
        assert isinstance(err, _lib.B200SAError) and err.code == BAD_ARG and "term_rows" in str(err)
    err = abi.unbwt(b"ab", [0])                                             # a cycle without the terminator
    assert err.code == BAD_ARG and "not the transform" in str(err)
    with pytest.raises(_lib.B200SAError):
        inverse_bwt(b"ab", 3)
    with pytest.raises(_lib.B200SAError):
        inverse_bwt(b"ab", -1)
    d = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = d.data_ptr()
    for kk in (1, 2, 5, 6):                                                 # (n, text, sa, starts, ndocs, bwt, term)
        args = [8, p, p, 0, 0, p, p]
        args[kk] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.bwt_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), kk
    with pytest.raises(_lib.B200SAError) as ex:                             # ndocs > 0 without doc_starts
        ctx.bwt_dev(8, p, p, 0, 2, p, p)
    assert ex.value.code == BAD_ARG
    with pytest.raises(_lib.B200SAError) as ex:                             # doc_starts with ndocs = 0, n > 0
        ctx.bwt_dev(8, p, p, p, 0, p, p)
    assert ex.value.code == BAD_ARG and "ndocs == 0" in str(ex.value)
    bad_starts = _dev32([1, 3])                                             # doc_starts[0] != 0, checked on the device
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.bwt_dev(8, p, p, bad_starts.data_ptr(), 2, p, p)
    assert ex.value.code == BAD_ARG and "doc_starts rejected" in str(ex.value)
    for kk in (2, 3, 4):                                                    # (n, ndocs, bwt, term, text)
        args = [8, 1, p, p, p]
        args[kk] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.unbwt_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), kk
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.unbwt_dev(8, 0, p, p, p)
    assert ex.value.code == BAD_ARG and "ndocs" in str(ex.value)
    # n + k above B200SA_MAX_N: before any launch and without allocating
    ws = ctx.stats()["workspace_bytes"]
    for call in (lambda: ctx.bwt_dev(0xFFFFF000, p, p, 0, 0, p, p),
                 lambda: ctx.bwt_dev(0xFFFFEFFF, p, p, p, 2, p, p),
                 lambda: ctx.unbwt_dev(0xFFFFF000, 1, p, p, p),
                 lambda: ctx.unbwt_dev(1 << 33, 1, p, p, p)):
        with pytest.raises(_lib.B200SAError) as ex:
            call()
        assert ex.value.code == TOO_LARGE
    assert ctx.stats()["workspace_bytes"] == ws
    ctx.close()


def test_concurrent_transforms_with_suffix_table_builds():
    docs = _planted_docs(2_000_000, 146)
    st = DocumentSuffixTable(docs)
    g, starts, text = st.table(), st.doc_starts(), st.text()
    want_b, want_t, want_r = bwt_check.forward(text, g, starts)
    etext = _u8(gen.english(300_000))
    want_sa = SuffixTable(etext).table()
    errors = []

    def run(fn):
        try:
            for _ in range(3):
                fn()
        except Exception as ex:
            errors.append(ex)

    def transform():                                                         # a context of its own per thread
        ctx = _lib.Context(0)
        abi = _Abi(ctx)
        assert abi.bwt(text, g, starts) == (want_b, want_t.tolist(), want_r)
        got = abi.unbwt(want_b, want_t)
        assert got[0] == text and np.array_equal(got[1], starts)
        ctx.close()

    def classes():                                                           # the shared default context
        assert st.bwt_runs() == want_r and inverse_bwt_documents(want_b, want_t) == docs

    def build():
        assert np.array_equal(SuffixTable(etext).table(), want_sa)

    th = [threading.Thread(target=run, args=(f,)) for f in (transform, transform, classes, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
