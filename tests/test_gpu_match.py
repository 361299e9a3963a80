"""Matching statistics and SMEMs (b200sa_match_stats_dev, b200sa_docs_match_stats_dev, b200sa_smems_dev,
SuffixTable / DocumentSuffixTable .matching_statistics and .smems) against the pure-Python model of
tests/model_match.py on small sets and the serial C statement of tests/match_check.c on large ones."""
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import match_check, model_docs, model_match
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_docs_list import _scale_docs

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
MARK = 0xA5A5A5A5


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a).view(dtype).copy()).cuda()


def _shifted(blob, k):
    """The bytes on the device at an address that is k past an aligned one (at least one byte allocated)."""
    buf = torch.zeros(len(blob) + k + 1, dtype=torch.uint8, device="cuda")
    if len(blob):
        buf[k:k + len(blob)] = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
    return buf, buf.data_ptr() + k


def _abi(ctx, text, sa, lcp, qs, starts=None, ranges=True, with_lcp=True, shift=(0, 0), off=None, q_bytes=None):
    """The C-ABI on host inputs: (len, start, end) pre-filled with MARK (start / end None without ranges)."""
    text, blob = bytes(text), b"".join(qs)
    off = model_match.offsets(qs) if off is None else np.asarray(off, dtype=np.uint64)
    q_bytes = len(blob) if q_bytes is None else q_bytes
    n, nq = len(text), len(off) - 1
    keep_t, d_t = _shifted(text, shift[0])
    keep_q, d_q = _shifted(blob, shift[1])
    d_sa, d_lcp, d_off = _dev(sa, np.int32), _dev(lcp, np.int32), _dev(off, np.int64)
    out = [torch.full((max(len(blob), 1),), MARK - (1 << 32), dtype=torch.int32, device="cuda") for _ in range(3)]
    ptrs = [o.data_ptr() for o in out]
    if not ranges:
        ptrs[1] = ptrs[2] = 0
    stream = torch.cuda.current_stream().cuda_stream
    lcp_ptr = d_lcp.data_ptr() if with_lcp else 0
    if starts is None:
        ctx.match_stats_dev(d_t, n, d_sa.data_ptr(), lcp_ptr, d_q, d_off.data_ptr(), nq, q_bytes, *ptrs, stream)
    else:
        d_s = _dev(np.asarray(starts, np.uint32), np.int32)
        ctx.docs_match_stats_dev(d_t, n, d_sa.data_ptr(), lcp_ptr, d_s.data_ptr(), len(starts), d_q, d_off.data_ptr(),
                                 nq, q_bytes, *ptrs, stream)
    torch.cuda.synchronize()
    res = [o.cpu().numpy().view(np.uint32)[:len(blob)] for o in out]
    return res[0], (res[1] if ranges else None), (res[2] if ranges else None)


def _smems_abi(ctx, off, ln, min_len, cap):
    """(total, offsets, qpos buffer of max(cap, 1) entries pre-filled with MARK)."""
    nq, qb = len(off) - 1, int(off[-1])
    d_off, d_len = _dev(off, np.int64), _dev(ln if len(ln) else np.zeros(1, np.uint32), np.int32)
    d_so = torch.full((nq + 1,), -1, dtype=torch.int64, device="cuda")
    d_qp = torch.full((max(cap, 1),), MARK - (1 << 32), dtype=torch.int32, device="cuda")
    total = ctx.smems_dev(d_off.data_ptr(), nq, qb, d_len.data_ptr(), min_len, d_so.data_ptr(),
                          d_qp.data_ptr() if cap else 0, cap, torch.cuda.current_stream().cuda_stream)
    return total, d_so.cpu().numpy().view(np.uint64), d_qp.cpu().numpy().view(np.uint32)


def _queries(rng, docs):
    text = b"".join(docs)
    qs = {x[a:a + m] for x in docs for m in range(1, 5) for a in range(len(x) - m + 1)}
    qs |= {b"", b"z", b"\x01", b"zz\x02z", text, text + b"a", text + text}     # absent bytes, longer than the text
    for _ in range(8):
        if text:
            a = int(rng.integers(0, len(text)))
            q = bytearray(text[a:a + int(rng.integers(1, 12))] + text[:int(rng.integers(0, 5))])
            q[int(rng.integers(0, len(q)))] ^= int(rng.integers(1, 256))        # a substitution
            qs.add(bytes(q))
    return sorted(qs)


def _same(got, want):
    return all(np.array_equal(a, b) for a, b in zip(got, want))


def test_abi_and_classes_equal_model_on_families():
    rng = np.random.default_rng(31)
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for docs in sets:
        qs = _queries(rng, docs)
        g, glcp = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_match.model(docs, g, glcp, qs)
        if len(docs):
            assert _same(_abi(ctx, text, g, glcp, qs, starts), want[1:]), docs
        st = DocumentSuffixTable(docs)
        assert _same(st.matching_statistics(qs), want), docs
        for m in (1, 3):
            so, qpos = model_match.smems(want[0], want[1], m)
            at = np.repeat(want[0][:-1], np.diff(so.astype(np.int64))).astype(np.int64) + qpos
            assert _same(st.smems(qs, m), (so, qpos, want[1][at], want[2][at], want[3][at])), (docs, m)
        if len(docs) == 1:                                     # one document is the single text
            sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
            assert np.array_equal(sa, g) and np.array_equal(lcp, glcp)
            assert _same(_abi(ctx, text, sa, lcp, qs), want[1:]), docs
            t1 = SuffixTable(text)
            assert _same(t1.matching_statistics(qs), want), docs
            assert _same(t1.smems(qs, 2), st.smems(qs, 2)), docs
    ctx.close()


def _edge_queries(text, rng):
    """Per length L in 0..40, text offset and query offset mod 8: junk, text[p:p + L], a byte that differs from
    text[p + L], filler to a multiple of 8 bytes -- so the match starts at every pair of alignments."""
    qs = []
    for L in range(41):
        for to in range(8):
            for qo in range(8):
                p = 8 * int(rng.integers(0, (len(text) - 64) // 8)) + to
                q = bytes(rng.integers(0, 256, qo, dtype=np.uint8)) + text[p:p + L] + bytes([text[p + L] ^ 0x80])
                qs.append(q + bytes(rng.integers(0, 256, -len(q) % 8, dtype=np.uint8)))
    return qs


@pytest.mark.parametrize("shift", [(0, 0), (1, 3), (3, 2), (2, 1)])
def test_compare_path_every_alignment_and_all_byte_values(shift):
    rng = np.random.default_rng(32)
    text = bytes(rng.integers(0, 256, 900, dtype=np.uint8)) + bytes(range(256)) + b"\x00\x00\xff\xff" * 5
    ctx = _lib.Context(0)
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    qs = _edge_queries(text, rng)
    # matches that end exactly at n and at the query's end, at every alignment of the tail
    qs += [text[-k:] for k in range(1, 42)] + [text[-k:] + b"\x07" for k in range(1, 42)]
    qs += [text[a:a + k] for a in range(8) for k in range(1, 42)]
    off = model_match.offsets(qs)
    blob = np.frombuffer(b"".join(qs), dtype=np.uint8)
    want = match_check.stats(text, None, sa, blob, off)
    assert _same(_abi(ctx, text, sa, lcp, qs, shift=shift), want)
    # documents: the same text cut at every residue, so that matches end exactly at a document end
    cuts = np.unique(np.r_[rng.integers(1, len(text), 60), [len(text) - 1, len(text) - 9]])
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(text)])]
    docs.insert(3, b"")
    g, glcp = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), model_docs.concat(docs)[1])
    starts = model_docs.concat(docs)[1]
    qs2 = qs + [d[-k:] + b"\x07" for d in docs for k in (1, 5, 9) if len(d) >= k] + [d for d in docs if d]
    off2 = model_match.offsets(qs2)
    want2 = match_check.stats(text, starts, g, np.frombuffer(b"".join(qs2), dtype=np.uint8), off2)
    assert _same(_abi(ctx, text, g, glcp, qs2, starts, shift=shift), want2)
    ctx.close()


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1023, 1024, 1025, 32768, 32769])
def test_runs_and_level_edges(n):
    ctx = _lib.Context(0)
    # a^n queried with a^m: m < n, = n, > n
    text = b"a" * n
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    qs = [b"a" * m for m in sorted({1, max(1, n // 2), max(1, n - 1), n, n + 1, n + 9})]
    ln, st, en = _abi(ctx, text, sa, lcp, qs)
    off = model_match.offsets(qs)
    for k, q in enumerate(qs):
        want = np.minimum(np.arange(len(q), 0, -1), n)
        a = int(off[k])
        assert np.array_equal(ln[a:a + len(q)], want)
        # shorter suffixes sort first: a^l starts the suffixes of l bytes or more, ranks [l - 1, n)
        assert np.array_equal(st[a:a + len(q)], want - 1) and (en[a:a + len(q)] == n).all()
    # a binary text of the same length: ranges across the block-minima boundaries
    rng = np.random.default_rng(n)
    text = bytes(rng.choice(list(b"ab"), n))
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    qs = [bytes(rng.choice(list(b"ab"), int(rng.integers(1, 24)))) for _ in range(300)] + [text[:1500], text[-1500:], b"c", b"a", b"b"]
    qs += [text[int(sa[r]):][:50] + b"c" for r in (0, n // 2, n - 1)]   # witnesses at the first and the last rank
    off = model_match.offsets(qs)
    want = match_check.stats(text, None, sa, np.frombuffer(b"".join(qs), dtype=np.uint8), off)
    assert _same(_abi(ctx, text, sa, lcp, qs), want)
    ctx.close()


def test_lengths_only_call_equals_full_call():
    rng = np.random.default_rng(33)
    ctx = _lib.Context(0)
    docs = [bytes(rng.choice(list(b"ACGT"), int(rng.integers(0, 400)))) for _ in range(30)]
    text, starts = model_docs.concat(docs)
    g, glcp = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts)
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    qs = [bytes(rng.choice(list(b"ACGT"), int(rng.integers(1, 60)))) for _ in range(200)] + [docs[1], b""]
    for args in ((text, sa, lcp, qs), (text, g, glcp, qs, starts)):
        full = _abi(ctx, *args)
        ln, st, en = _abi(ctx, *args, ranges=False, with_lcp=False)
        assert st is None and np.array_equal(ln, full[0])
    ctx.close()


def _reads(t, rng, count, length, rate):
    """Half reads sampled from t with substitutions at `rate`, half random strings over t's alphabet."""
    t = np.frombuffer(t, dtype=np.uint8)
    a = rng.integers(0, len(t) - length, count // 2)
    reads = t[a[:, None] + np.arange(length)[None, :]].copy()
    sub = rng.random(reads.shape) < rate
    reads[sub] = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), int(sub.sum()))
    rnd = rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), (count - count // 2, length))
    return [r.tobytes() for r in reads] + [r.tobytes() for r in rnd]


def test_scale_against_the_serial_checker():
    t, docs = _scale_docs()
    rng = np.random.default_rng(34)
    qs = _reads(t, rng, 50_000, 100, 0.02)                         # 5 M pattern positions
    off = model_match.offsets(qs)
    blob = np.frombuffer(b"".join(qs), dtype=np.uint8)
    win = (0, 400_000), (len(blob) - 400_000, len(blob))           # the ranges are checked on two windows
    for st, starts in ((DocumentSuffixTable(docs), True), (SuffixTable(t), False)):
        s = st.doc_starts() if starts else None
        got = st.matching_statistics(qs)
        assert np.array_equal(got[0], off)
        assert np.array_equal(got[1], match_check.stats(st.text(), s, st.table(), blob, off, ranges=False)[0])
        for x0, x1 in win:
            want = match_check.stats(st.text(), s, st.table(), blob, off, x0, x1)
            assert _same([g[x0:x1] for g in got[1:]], want)
        # every SMEM string's positions range is its (start, end)
        so, qpos, ln, a, b = st.smems(qs[:3000] + qs[-3000:], 20)
        sub = qs[:3000] + qs[-3000:]
        qid = np.repeat(np.arange(len(sub)), np.diff(so.astype(np.int64)))
        strings = [sub[q][p:p + l] for q, p, l in zip(qid.tolist(), qpos.tolist(), ln.tolist())]
        assert len(strings) > 3000 and min(ln) >= 20
        if starts:
            ps, pe = st.positions_batch(strings)
            assert np.array_equal(ps, a) and np.array_equal(pe, b)
        else:
            for k in range(0, len(strings), 97):
                hits = st.positions(strings[k])
                assert np.array_equal(hits, st.table()[a[k]:b[k]])


def test_fixture_100k():
    t = gen.fixture("AP009048_100000.fasta").tobytes()
    st = SuffixTable(t)
    rng = np.random.default_rng(35)
    qs = _reads(t, rng, 2000, 80, 0.03) + [t[:5000], t[-300:] + b"N"]
    off = model_match.offsets(qs)
    want = match_check.stats(t, None, st.table(), np.frombuffer(b"".join(qs), dtype=np.uint8), off)
    assert _same(st.matching_statistics(qs)[1:], want)
    # from_parts tables work: lcp comes from lcp_lens()
    again = SuffixTable.from_parts(t, st.table())
    assert _same(again.matching_statistics(qs[:50]), st.matching_statistics(qs[:50]))


def test_smem_ranges_feed_listing_and_topk():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:1500])
    rng = np.random.default_rng(36)
    qs = _reads(b"".join(docs[:1500]), rng, 600, 120, 0.02)
    so, qpos, ln, a, b = st.smems(qs, 16)
    qid = np.repeat(np.arange(len(qs)), np.diff(so.astype(np.int64)))
    strings = [qs[q][p:p + l] for q, p, l in zip(qid.tolist(), qpos.tolist(), ln.tolist())]
    assert len(strings) > 300
    assert _same(st.documents_for_ranges(a, b), st.documents_batch(strings))
    assert _same(st.top_documents_for_ranges(a, b, 3), st.top_documents_batch(strings, 3))
    # ranges of positions_batch, empty ones included
    qs2 = [b"ACG", b"T", b"", b"GGGGGGGGGGGGGGGGGGGGGG", b"CA"]
    ps, pe = st.positions_batch(qs2)
    assert _same(st.documents_for_ranges(ps, pe), st.documents_batch(qs2))
    assert _same(st.top_documents_for_ranges(ps, pe, 10), st.top_documents_batch(qs2, 10))
    assert st.documents_for_ranges([], [])[0].tolist() == [0]
    with pytest.raises(ValueError):
        st.top_documents_for_ranges(ps, pe, 0)
    with pytest.raises(ValueError):
        st.documents_for_ranges([1, 2], [3])
    with pytest.raises(_lib.B200SAError):
        st.documents_for_ranges([5], [4])


def test_smem_protocol():
    t = gen.fixture("AP009048_10000.fasta").tobytes()
    st = SuffixTable(t)
    rng = np.random.default_rng(37)
    qs = _reads(t, rng, 300, 90, 0.03) + [b"", t[100:160]]
    off, ln, _, _ = st.matching_statistics(qs)
    ctx = _lib.Context(0)
    for m in (1, 20):
        want_off, want_qpos = model_match.smems(off, ln, m)
        total = len(want_qpos)
        assert total > 0
        for cap in (0, total - 1):                                 # too small: offsets and total only
            tot, so, qp = _smems_abi(ctx, off, ln, m, cap)
            assert tot == total and np.array_equal(so, want_off) and (qp == MARK).all()
        tot, so, qp = _smems_abi(ctx, off, ln, m, total)
        assert tot == total and np.array_equal(so, want_off) and np.array_equal(qp, want_qpos)
        tot, so, qp = _smems_abi(ctx, off, ln, m, total + 5)
        assert np.array_equal(qp[:total], want_qpos) and (qp[total:] == MARK).all()
    tot, so, qp = _smems_abi(ctx, off, ln, int(ln.max()) + 1, 8)   # longer than every match
    assert tot == 0 and not so.any() and (qp == MARK).all()
    ctx.set_timing(True)
    _smems_abi(ctx, off, ln, 20, 1 << 16)
    names = [p for p, _ in ctx.phase_times()]
    for p in ("match_check", "smem_flag", "smem_scan", "smem_emit"):
        assert p in names, names
    ctx.close()
    assert st.smems(qs, 1000)[0].tolist() == [0] * (len(qs) + 1)
    with pytest.raises(ValueError):
        st.smems(qs, 0)


def test_abi_errors_and_empty_inputs():
    ctx = _lib.Context(0)
    text = b"abracadabra"
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    qs = [b"abra", b"cad"]
    good = _abi(ctx, text, sa, lcp, qs)
    # q_off: not starting at 0, not ascending, not ending at q_bytes
    for off, qb in (([1, 4, 7], 7), ([0, 5, 3, 7], 7), ([0, 4, 7], 6), ([0, 4, 6], 7)):
        with pytest.raises(_lib.B200SAError) as ex:
            _abi(ctx, text, sa, lcp, qs, off=off, q_bytes=qb)
        assert ex.value.code == BAD_ARG and "q_off" in str(ex.value)
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.smems_dev(_dev(np.asarray(off, np.uint64), np.int64).data_ptr(), len(off) - 1, qb,
                          _dev(good[0], np.int32).data_ptr(), 1, torch.zeros(8, dtype=torch.int64, device="cuda").data_ptr(),
                          0, 0, 0)
        assert ex.value.code == BAD_ARG and "q_off" in str(ex.value)
    assert _same(_abi(ctx, text, sa, lcp, qs), good)               # the context still works
    # each required pointer, and start without end
    d = torch.zeros(64, dtype=torch.int64, device="cuda")
    p = d.data_ptr()
    base = [p, 11, p, p, p, p, 2, 7, p, p, p]
    for k in (0, 2, 3, 4, 5, 8, 9, 10):
        args = list(base)
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.match_stats_dev(*args)
        assert ex.value.code == BAD_ARG, k
    dbase = [p, 11, p, p, p, 1, p, p, 2, 7, p, p, p]
    for k in (0, 2, 3, 4, 6, 7, 10, 11, 12):
        args = list(dbase)
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.docs_match_stats_dev(*args)
        assert ex.value.code == BAD_ARG, k
    with pytest.raises(_lib.B200SAError) as ex:                    # ndocs = 0 with n > 0
        ctx.docs_match_stats_dev(p, 11, p, p, p, 0, p, p, 2, 7, p, p, p)
    assert ex.value.code == BAD_ARG
    with pytest.raises(_lib.B200SAError) as ex:                    # doc_starts is checked on the device
        _abi(ctx, text, sa, lcp, qs, starts=[0, 7, 5])
    assert ex.value.code == BAD_ARG and "doc_starts" in str(ex.value)
    for args in ([p, 1 << 33, p, p, p, p, 2, 7, p, p, p], [p, 11, p, p, p, p, 2, 1 << 33, p, p, p]):
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.match_stats_dev(*args)
        assert ex.value.code == TOO_LARGE
    sbase = [p, 2, 7, p, 1, p, p, 4]
    for k in (0, 3, 5, 6):
        args = list(sbase)
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.smems_dev(*args)
        assert ex.value.code == BAD_ARG, k
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.smems_dev(p, 2, 7, p, 0, p, p, 4)                      # min_len = 0
    assert ex.value.code == BAD_ARG and "min_len" in str(ex.value)
    with pytest.raises(_lib.B200SAError) as ex:
        ctx.smems_dev(p, 2, 1 << 33, p, 1, p, p, 4)
    assert ex.value.code == TOO_LARGE
    # nq = 0 and q_bytes = 0 write nothing; smems writes offsets[0] = 0
    ln, st, en = _abi(ctx, text, sa, lcp, [])
    assert len(ln) == 0
    ln, st, en = _abi(ctx, text, sa, lcp, [b"", b""])
    assert len(ln) == 0
    tot, so, _ = _smems_abi(ctx, np.zeros(1, np.uint64), np.zeros(0, np.uint32), 1, 4)
    assert tot == 0 and so.tolist() == [0]
    tot, so, _ = _smems_abi(ctx, np.zeros(3, np.uint64), np.zeros(0, np.uint32), 1, 4)
    assert tot == 0 and so.tolist() == [0, 0, 0]
    # n = 0: nothing occurs
    z = np.zeros(0, np.uint32)
    for starts in (None, [0, 0]):
        ln, st, en = _abi(ctx, b"", z, z, qs, starts)
        assert not ln.any() and not st.any() and not en.any()
    # phases
    ctx.set_timing(True)
    _abi(ctx, text, sa, lcp, qs)
    names = [p for p, _ in ctx.phase_times()]
    assert names == ["match_check", "match_levels", "match_search"], names
    _abi(ctx, text, sa, lcp, qs, ranges=False)
    assert [p for p, _ in ctx.phase_times()] == ["match_check", "match_search"]
    ctx.close()
    # the classes on empty tables and empty batches
    for e in (DocumentSuffixTable([]), DocumentSuffixTable([b"", b""]), SuffixTable(b"")):
        off, ln, st, en = e.matching_statistics([b"ab", b"", b"c"])
        assert off.tolist() == [0, 2, 2, 3] and not ln.any() and not st.any() and not en.any()
        assert e.smems([b"ab", b"c"])[0].tolist() == [0, 0, 0]
        assert e.matching_statistics([])[0].tolist() == [0] and e.smems([])[0].tolist() == [0]
    one = SuffixTable(b"banana")
    assert one.matching_statistics([])[0].tolist() == [0]
    so, qpos, ln, a, b = one.smems([b"nanaba", b""], 2)
    assert so.tolist() == [0, 2, 2] and qpos.tolist() == [0, 4] and ln.tolist() == [4, 2]
    assert [sorted(one.table()[x:y].tolist()) for x, y in zip(a, b)] == [[2], [0]]


def test_concurrent_matching_statistics_with_suffix_table_builds():
    t, docs = _scale_docs()
    st = DocumentSuffixTable(docs[:800])
    text = b"".join(docs[:800])
    rng = np.random.default_rng(38)
    qs = _reads(text, rng, 2000, 100, 0.02)
    want = st.matching_statistics(qs)
    g, glcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    etext = _u8(gen.english(300_000))
    want_t = SuffixTable(etext).table()
    errors = []

    def run(fn):
        try:
            for _ in range(4):
                fn()
        except Exception as ex:
            errors.append(ex)

    def stats():                                                   # a context of its own per thread
        ctx = _lib.Context(0)
        assert _same(_abi(ctx, text, g, glcp, qs, starts), want[1:])
        ctx.close()

    def build():
        assert np.array_equal(SuffixTable(etext).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (stats, stats, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
