"""Approximate positions (b200sa_approx_positions_dev, b200sa_docs_approx_positions_dev, and the approximate_*
methods of SuffixTable and DocumentSuffixTable) against the definition of tests/model_approx.py on small
sets and the serial C statement of tests/approx_check.c on large ones."""
import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import approx_check, model_approx, model_docs
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG = -1
MARK = 0xA5A5A5A5
MARK64 = 0xA5A5A5A5A5A5A5A5


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a).view(dtype).copy()).cuda()


def _shifted(blob, k):
    """The bytes on the device at an address that is k past an aligned one (at least one byte allocated)."""
    buf = torch.zeros(len(blob) + k + 1, dtype=torch.uint8, device="cuda")
    if len(blob):
        buf[k:k + len(blob)] = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
    return buf, buf.data_ptr() + k


def _offsets(qs):
    off = np.zeros(len(qs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(q) for q in qs])
    return off


def _abi(ctx, text, table, qs, k, cap, starts=None, with_mis=True, shift=(0, 0), off=None, buf=None):
    """The C-ABI on host inputs: (total, offsets, pos, mis) with offsets pre-filled with MARK64 and pos / mis
    buffers of max(buf or cap, 1) entries pre-filled with MARK (mis None without with_mis)."""
    text, blob = bytes(text), b"".join(qs)
    off = _offsets(qs) if off is None else np.asarray(off, dtype=np.uint64)
    n, nq = len(text), len(off) - 1
    keep_t, d_t = _shifted(text, shift[0])
    keep_q, d_q = _shifted(blob, shift[1])
    d_r = _dev(np.asarray(table, np.uint32) if n else np.zeros(1, np.uint32), np.int32)
    d_off = _dev(off, np.int64)
    d_o = torch.full((nq + 1,), MARK64 - (1 << 64), dtype=torch.int64, device="cuda")
    size = max(cap if buf is None else buf, 1)
    d_p = torch.full((size,), MARK - (1 << 32), dtype=torch.int32, device="cuda")
    d_m = torch.full((size,), MARK - (1 << 32), dtype=torch.int32, device="cuda")
    mp = d_m.data_ptr() if with_mis else 0
    stream = torch.cuda.current_stream().cuda_stream
    if starts is None:
        total = ctx.approx_positions_dev(d_t, n, d_r.data_ptr(), d_q, d_off.data_ptr(), nq, k, d_o.data_ptr(),
                                         d_p.data_ptr(), mp, cap, stream)
    else:
        d_s = _dev(np.asarray(starts, np.uint32) if len(starts) else np.zeros(1, np.uint32), np.int32)
        total = ctx.docs_approx_positions_dev(d_t, n, d_r.data_ptr(), d_s.data_ptr(), len(starts), d_q,
                                              d_off.data_ptr(), nq, k, d_o.data_ptr(), d_p.data_ptr(), mp, cap, stream)
    torch.cuda.synchronize()
    return (total, d_o.cpu().numpy().view(np.uint64), d_p.cpu().numpy().view(np.uint32),
            d_m.cpu().numpy().view(np.uint32) if with_mis else None)


def _fetch(ctx, text, table, qs, k, starts=None, **kw):
    """(offsets, pos, mis) of the count call then the fetch call."""
    total, _, _, _ = _abi(ctx, text, table, qs, k, 0, starts)
    tot, off, pos, mis = _abi(ctx, text, table, qs, k, total, starts, **kw)
    assert tot == total
    return off, pos[:total], (mis[:total] if mis is not None else None)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _queries(rng, docs, k):
    """Substrings with substitutions, m = 0, m <= k, m = k + 1, longer than the text, absent bytes, and windows
    that end at a document end."""
    text = b"".join(docs)
    alpha = sorted(set(text)) or [97]
    rand = lambda m: bytes(int(alpha[int(x)]) for x in rng.integers(0, len(alpha), m))
    qs = [b"", rand(1), rand(max(k, 1)), rand(k + 1), rand(k + 3), text + b"a", b"\x01z"]
    nonempty = [d for d in docs if d]
    for _ in range(6):
        if not nonempty:
            break
        d = nonempty[int(rng.integers(0, len(nonempty)))]
        m = int(rng.integers(1, len(d) + 1))
        a = int(rng.integers(0, len(d) - m + 1))
        q = bytearray(d[a:a + m])
        for _ in range(int(rng.integers(0, k + 2))):
            q[int(rng.integers(0, m))] ^= int(rng.integers(1, 256))
        qs += [bytes(q), d[len(d) - m:]]
    return qs


FAMILY_KS = [0, 1, 2, 3, 4, 6, 31]


def test_abi_and_classes_equal_model_on_families():
    rng = np.random.default_rng(41)
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = FAMILY_KS[i % len(FAMILY_KS)]
        qs = _queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_approx.brute(docs, qs, k)
        assert _same(_fetch(ctx, text, g, qs, k, starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        assert _same(st.approximate_positions_batch(qs, k), want), (docs, k)
        assert np.array_equal(st.approximate_counts(qs, k), np.diff(want[0].astype(np.int64))), (docs, k)
        if len(docs) == 1:                                     # one document is the single text
            sa = ctx.build(np.frombuffer(text, dtype=np.uint8)) if text else np.zeros(0, np.uint32)
            assert _same(_fetch(ctx, text, sa, qs, k), want), (docs, k)
            t1 = SuffixTable(text)
            assert _same(t1.approximate_positions_batch(qs, k), want), (docs, k)
            p, e = t1.approximate_positions(qs[-1], k)
            a, b = int(want[0][-2]), int(want[0][-1])
            assert np.array_equal(p, want[1][a:b]) and np.array_equal(e, want[2][a:b])
    ctx.close()


def test_k0_equals_sorted_positions():
    rng = np.random.default_rng(42)
    for docs in _families(rng)[::3]:
        qs = _queries(rng, docs, 0)
        st = DocumentSuffixTable(docs)
        off, pos, mis = st.approximate_positions_batch(qs, 0)
        assert not mis.any()
        for q, a, b in zip(qs, off[:-1], off[1:]):
            rows = st.positions(q)
            want = np.sort(st.doc_starts()[rows[:, 0]].astype(np.int64) + rows[:, 1]) if len(rows) else []
            assert np.array_equal(pos[int(a):int(b)], want), (docs, q)
        if len(docs) == 1:
            t1 = SuffixTable(docs[0])
            for q in qs:
                p, _ = t1.approximate_positions(q, 0)
                assert np.array_equal(p, np.sort(t1.positions(q))), (docs, q)


def test_cap_protocol_and_null_mismatches():
    rng = np.random.default_rng(43)
    text = _u8(gen.dna(3000))
    sa = SuffixTable(text).table()
    qs = [text[a:a + 12] for a in rng.integers(0, 2980, 30)] + [b"ACGT", b"", b"AC"]
    ctx = _lib.Context(0)
    want = model_approx.brute([text], qs, 2)
    total = int(want[0][-1])
    assert total > 1
    tot, off, pos, mis = _abi(ctx, text, sa, qs, 2, 0, buf=total + 5)           # counts only
    assert tot == total and np.array_equal(off, want[0])
    assert (pos == MARK).all() and (mis == MARK).all()
    tot, off, pos, mis = _abi(ctx, text, sa, qs, 2, total - 1, buf=total + 5)   # too small: offsets only
    assert tot == total and np.array_equal(off, want[0])
    assert (pos == MARK).all() and (mis == MARK).all()
    tot, off, pos, mis = _abi(ctx, text, sa, qs, 2, total, buf=total + 5)       # fits: nothing past total
    assert tot == total and np.array_equal(off, want[0])
    assert np.array_equal(pos[:total], want[1]) and np.array_equal(mis[:total], want[2])
    assert (pos[total:] == MARK).all() and (mis[total:] == MARK).all()
    tot, off, pos, mis = _abi(ctx, text, sa, qs, 2, total, with_mis=False, buf=total + 5)
    assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all() and mis is None
    ctx.close()


@pytest.mark.parametrize("shift", [(1, 3), (3, 2), (2, 1)])
def test_unaligned_buffers_and_all_byte_values(shift):
    rng = np.random.default_rng(44)
    text = bytes(rng.integers(0, 256, 700, dtype=np.uint8)) + bytes(range(256)) + b"\x00\x00\xff\xff" * 5
    sa = SuffixTable(text).table()
    qs = []
    for m in (1, 2, 3, 5, 9, 17, 33):
        for a in rng.integers(0, len(text) - m, 6):
            q = bytearray(text[a:a + m])
            q[int(rng.integers(0, m))] ^= 0x80
            qs.append(bytes(q))
    qs += [text[-m:] for m in range(1, 12)] + [bytes([255, 255])]
    ctx = _lib.Context(0)
    for k in (0, 1, 3):
        want = model_approx.brute([text], qs, k)
        assert _same(_fetch(ctx, text, sa, qs, k, shift=shift), want), k
        starts = np.array([0, 300, 300, 956], dtype=np.uint32)
        g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
        docs = [text[0:300], b"", text[300:956], text[956:]]
        assert _same(_fetch(ctx, text, g, qs, k, starts, shift=shift), model_approx.brute(docs, qs, k)), k
    ctx.close()


def test_repetitive_texts_span_many_items():
    ctx = _lib.Context(0)
    for text, qs in ((b"a" * 5000, [b"a" * m for m in (1, 4, 9, 30)] + [b"ab" * 7, b"b" * 9]),
                     (b"ACGT" * 1500, [b"ACGT" * 3, b"CGTACGTT", b"GGGGGGGG", b"ACGTACGTAC" * 2])):
        sa = SuffixTable(text).table()
        for k in (0, 1, 3, 8):
            want = model_approx.brute([text], qs, k)
            assert _same(_fetch(ctx, text, sa, qs, k), want), k
        docs = [text[:2000], b"", text[2000:4100], text[4100:]]
        st = DocumentSuffixTable(docs)
        for k in (0, 2, 5):
            assert _same(st.approximate_positions_batch(qs, k), model_approx.brute(docs, qs, k)), k
    ctx.close()


def test_short_queries_on_documents_with_empty_documents():
    docs = [b"", b"abcab", b"", b"", b"b", b"cc", b""]
    st = DocumentSuffixTable(docs)
    qs = [b"x", b"zz", b"zzz", b"bcabz", b"", b"cc"]
    for k in (1, 2, 3, 5, 31):
        assert _same(st.approximate_positions_batch(qs, k), model_approx.brute(docs, qs, k)), k
    empty = DocumentSuffixTable([b"", b""])
    off, pos, mis = empty.approximate_positions_batch(qs, 3)
    assert not off.any() and len(pos) == 0 and len(mis) == 0
    off, pos, mis = SuffixTable(b"").approximate_positions_batch(qs, 3)
    assert not off.any() and len(pos) == 0
    assert len(st.approximate_positions_batch([], 2)[0]) == 1


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"abracadabra"
    sa = SuffixTable(text).table()
    with pytest.raises(_lib.B200SAError) as e:
        _abi(ctx, text, sa, [b"abc"], 32, 0)
    assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value)
    for off in ([1, 3], [0, 3, 2, 4], [0, 5, 3]):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abca"], 1, 0, off=off)
        assert e.value.code == BAD_ARG and "q_off rejected" in str(e.value)
    for starts in ([1, 5], [0, 7, 3], [0, 20]):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abc"], 1, 0, starts=np.asarray(starts, np.uint32))
        assert e.value.code == BAD_ARG and "doc_starts rejected" in str(e.value)
    with pytest.raises(ValueError):
        SuffixTable(text).approximate_positions(b"abc", 32)
    assert _same(_fetch(ctx, text, sa, [b"abc"], 31), model_approx.brute([text], [b"abc"], 31))
    ctx.close()


def test_repeated_calls_are_identical():
    rng = np.random.default_rng(45)
    text = _u8(gen.dna(200_000))
    st = SuffixTable(text)
    qs = [text[a:a + 30] for a in rng.integers(0, len(text) - 30, 300)] + [b"ACGTACGT"]
    a = st.approximate_positions_batch(qs, 3)
    b = st.approximate_positions_batch(qs, 3)
    assert _same(a, b)
    want = approx_check.approx(text, None, qs, 3)
    assert _same(a, want)


def _mutate(a, rng, rate):
    alpha = np.frombuffer(b"ACGT", dtype=np.uint8)
    sub = rng.random(a.shape) < rate
    a[sub] = rng.choice(alpha, int(sub.sum()))
    return a


def test_scale_reads_and_20mers_against_c_statement():
    rng = np.random.default_rng(46)
    t = gen.dna(10_000_000)
    text = _u8(t)
    at = rng.integers(0, len(t) - 150, 10_000)
    reads = _mutate(t[at[:, None] + np.arange(150)[None, :]].copy(), rng, 0.01)
    at20 = rng.integers(0, len(t) - 20, 500)
    mers = t[at20[:, None] + np.arange(20)[None, :]].copy()
    cuts = np.unique(rng.integers(1, len(t), 9000))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for table, st in (("text", SuffixTable(text)), ("docs", DocumentSuffixTable(docs))):
        for blob, m, k in ((reads, 150, 4), (mers, 20, 3)):
            nq = len(blob)
            qs = [bytes(r) for r in blob]
            off, pos, mis = st.approximate_positions_batch(qs, k)
            assert int(off[-1]) == len(pos) and len(pos) >= (nq if m == 20 else nq // 2)
            sample = rng.choice(nq, 12, replace=False)
            for q in sample.tolist():
                want = approx_check.approx(text, None if table == "text" else starts, [qs[q]], k)
                a, b = int(off[q]), int(off[q + 1])
                assert np.array_equal(pos[a:b], want[1]) and np.array_equal(mis[a:b], want[2]), (table, m, q)
