"""The edit metric of approximate positions (B200SA_APPROX_EDIT on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev, metric="edit" on the approximate_* methods of SuffixTable and
DocumentSuffixTable) against the definition of tests/model_edit.py on small sets and the serial C statement of
tests/edit_check.c on large ones."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import edit_check, model_approx, model_docs, model_edit
from tests.test_edit_model import edited
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT


def _queries(rng, docs, k):
    """Substrings with substitutions and indels, m = 0, m <= k, m = k + 1, longer than the text, absent bytes,
    and substrings that end at a document end."""
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
        qs += [edited(rng, d[a:a + m], int(rng.integers(0, k + 2)), alpha), d[len(d) - m:]]
    return qs


FAMILY_KS = [0, 1, 2, 3, 4, 6, 31]


def test_abi_and_classes_equal_model_on_families():
    rng = np.random.default_rng(51)
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = FAMILY_KS[i % len(FAMILY_KS)]
        qs = _queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_edit.brute(docs, qs, k)
        assert _same(_fetch(ctx, text, g, qs, k | EDIT, starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        assert _same(st.approximate_positions_batch(qs, k, metric="edit"), want), (docs, k)
        assert np.array_equal(st.approximate_counts(qs, k, metric="edit"), np.diff(want[0].astype(np.int64)))
        if len(docs) == 1:                                     # one document is the single text
            sa = ctx.build(np.frombuffer(text, dtype=np.uint8)) if text else np.zeros(0, np.uint32)
            assert _same(_fetch(ctx, text, sa, qs, k | EDIT), want), (docs, k)
            t1 = SuffixTable(text)
            assert _same(t1.approximate_positions_batch(qs, k, metric="edit"), want), (docs, k)
            p, e = t1.approximate_positions(qs[-1], k, metric="edit")
            a, b = int(want[0][-2]), int(want[0][-1])
            assert np.array_equal(p, want[1][a:b]) and np.array_equal(e, want[2][a:b])
    ctx.close()


def test_k0_equals_sorted_positions():
    rng = np.random.default_rng(52)
    for docs in _families(rng)[::3]:
        qs = _queries(rng, docs, 0)
        st = DocumentSuffixTable(docs)
        off, pos, dist = st.approximate_positions_batch(qs, 0, metric="edit")
        assert not dist.any()
        for q, a, b in zip(qs, off[:-1], off[1:]):
            rows = st.positions(q)
            want = np.sort(st.doc_starts()[rows[:, 0]].astype(np.int64) + rows[:, 1]) if len(rows) else []
            assert np.array_equal(pos[int(a):int(b)], want), (docs, q)
        if len(docs) == 1:
            t1 = SuffixTable(docs[0])
            for q in qs:
                p, _ = t1.approximate_positions(q, 0, metric="edit")
                assert np.array_equal(p, np.sort(t1.positions(q))), (docs, q)


def test_hamming_occurrences_are_edit_occurrences():
    rng = np.random.default_rng(53)
    text = _u8(gen.dna(20_000))
    docs = [text[:7000], b"", text[7000:15000], text[15000:]]
    qs = [edited(rng, text[a:a + 24], 2, b"ACGT") for a in rng.integers(0, len(text) - 24, 60)] + [b"ACGTAC"]
    for st in (SuffixTable(text), DocumentSuffixTable(docs)):
        for k in (1, 3, 6):
            ho, hp, hm = st.approximate_positions_batch(qs, k)
            eo, ep, ed = st.approximate_positions_batch(qs, k, metric="edit")
            for q in range(len(qs)):
                e = dict(zip(ep[int(eo[q]):int(eo[q + 1])].tolist(), ed[int(eo[q]):int(eo[q + 1])].tolist()))
                for p, mis in zip(hp[int(ho[q]):int(ho[q + 1])].tolist(), hm[int(ho[q]):int(ho[q + 1])].tolist()):
                    assert p in e and e[p] <= mis, (k, q, p)


def test_cap_protocol_and_null_distances():
    rng = np.random.default_rng(54)
    text = _u8(gen.dna(3000))
    sa = SuffixTable(text).table()
    qs = [edited(rng, text[a:a + 12], 1, b"ACGT") for a in rng.integers(0, 2980, 30)] + [b"ACGT", b"", b"AC"]
    ctx = _lib.Context(0)
    want = model_edit.brute([text], qs, 2)
    total = int(want[0][-1])
    assert total > 1
    kf = 2 | EDIT
    tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, 0, buf=total + 5)           # counts only
    assert tot == total and np.array_equal(off, want[0])
    assert (pos == MARK).all() and (dist == MARK).all()
    tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total - 1, buf=total + 5)   # too small: offsets only
    assert tot == total and np.array_equal(off, want[0])
    assert (pos == MARK).all() and (dist == MARK).all()
    tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, buf=total + 5)       # fits: nothing past total
    assert tot == total and np.array_equal(off, want[0])
    assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
    assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
    tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, with_mis=False, buf=total + 5)
    assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all() and dist is None
    ctx.close()


@pytest.mark.parametrize("shift", [(1, 3), (3, 2), (2, 1)])
def test_unaligned_buffers_and_all_byte_values(shift):
    rng = np.random.default_rng(55)
    text = bytes(rng.integers(0, 256, 700, dtype=np.uint8)) + bytes(range(256)) + b"\x00\x00\xff\xff" * 5
    sa = SuffixTable(text).table()
    alpha = list(range(256))
    qs = [edited(rng, text[a:a + m], 1, alpha) for m in (1, 2, 3, 5, 9, 17, 33)
          for a in rng.integers(0, len(text) - m, 6)]
    qs += [text[-m:] for m in range(1, 12)] + [bytes([255, 255]), text[:5]]
    ctx = _lib.Context(0)
    starts = np.array([0, 300, 300, 956], dtype=np.uint32)
    g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
    docs = [text[0:300], b"", text[300:956], text[956:]]
    for k in (0, 1, 3):
        assert _same(_fetch(ctx, text, sa, qs, k | EDIT, shift=shift), model_edit.brute([text], qs, k)), k
        assert _same(_fetch(ctx, text, g, qs, k | EDIT, starts, shift=shift), model_edit.brute(docs, qs, k)), k
    ctx.close()


def test_repetitive_texts_put_many_windows_on_the_reporter_rule():
    ctx = _lib.Context(0)
    for text, qs in ((b"a" * 3000, [b"a" * m for m in (1, 4, 9, 30)] + [b"ab" * 7, b"b" * 9, b"a" * 20 + b"b"]),
                     (b"ACGT" * 800, [b"ACGT" * 3, b"CGTACGTT", b"GGGGGGGG", b"ACGTACGTAC" * 2, b"ACGACGT" * 3])):
        sa = SuffixTable(text).table()
        for k in (0, 1, 3, 8):
            assert _same(_fetch(ctx, text, sa, qs, k | EDIT), model_edit.brute([text], qs, k)), k
        docs = [text[:1000], b"", text[1000:2100], text[2100:]]
        st = DocumentSuffixTable(docs)
        for k in (0, 2, 5):
            assert _same(st.approximate_positions_batch(qs, k, metric="edit"), model_edit.brute(docs, qs, k)), k
    ctx.close()


def test_long_queries():
    rng = np.random.default_rng(56)
    text = _u8(gen.dna(30_000))
    docs = [text[:12_000], text[12_000:12_000], text[12_000:]]
    qs = []
    for m in (1000, 5000):
        for a in rng.integers(0, len(text) - m, 3):
            qs.append(edited(rng, text[a:a + m], int(rng.integers(0, 12)), b"ACGT"))
    qs.append(text[12_000 - 1000:12_000])                      # ends at a document end
    for st, starts in ((SuffixTable(text), None), (DocumentSuffixTable(docs), np.array([0, 12_000, 12_000]))):
        for k in (4, 10, 31):
            want = edit_check.edit(text, starts, qs, k)
            assert _same(st.approximate_positions_batch(qs, k, metric="edit"), want), k
    assert int(want[0][-1]) >= 3


def test_short_queries_on_documents_with_empty_documents():
    docs = [b"", b"abcab", b"", b"", b"b", b"cc", b""]
    st = DocumentSuffixTable(docs)
    qs = [b"x", b"zz", b"zzz", b"bcabz", b"", b"cc", b"ab"]
    for k in (1, 2, 3, 5, 31):
        assert _same(st.approximate_positions_batch(qs, k, metric="edit"), model_edit.brute(docs, qs, k)), k
    empty = DocumentSuffixTable([b"", b""])
    off, pos, dist = empty.approximate_positions_batch(qs, 3, metric="edit")
    assert not off.any() and len(pos) == 0 and len(dist) == 0
    off, pos, dist = SuffixTable(b"").approximate_positions_batch(qs, 3, metric="edit")
    assert not off.any() and len(pos) == 0
    assert len(st.approximate_positions_batch([], 2, metric="edit")[0]) == 1


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"abracadabra"
    sa = SuffixTable(text).table()
    for k in (0x20000, EDIT | 0x40000, 1 << 31, 0x10000 | 0x8000000 | 3):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abc"], k, 0)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value), hex(k)
    for k in (32 | EDIT, 0xFFFF | EDIT, 32, 99):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abc"], k, 0)
        assert e.value.code == BAD_ARG and "k above B200SA_APPROX_MAX_K" in str(e.value), hex(k)
    for metric in ("levenshtein", "Edit", None):
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_positions(b"abc", 1, metric=metric)
    with pytest.raises(ValueError):
        SuffixTable(text).approximate_counts([b"abc"], 32, metric="edit")
    assert _same(_fetch(ctx, text, sa, [b"abc"], 31 | EDIT), model_edit.brute([text], [b"abc"], 31))
    assert _same(_fetch(ctx, text, sa, [b"abc"], 1), model_approx.brute([text], [b"abc"], 1))
    ctx.close()


def test_repeated_calls_are_identical():
    rng = np.random.default_rng(57)
    text = _u8(gen.dna(200_000))
    st = SuffixTable(text)
    qs = [edited(rng, text[a:a + 30], 2, b"ACGT") for a in rng.integers(0, len(text) - 30, 300)] + [b"ACGTACGT"]
    a = st.approximate_positions_batch(qs, 3, metric="edit")
    b = st.approximate_positions_batch(qs, 3, metric="edit")
    assert _same(a, b)
    assert _same(a, edit_check.edit(text, None, qs, 3))


def _reads(t, rng, count, m, sub, indel):
    """count reads of m bytes sampled from t, with substitutions at rate sub and insertions or deletions at rate
    indel, then cut or padded from the text back to m bytes."""
    out = []
    for a in rng.integers(0, len(t) - 2 * m, count).tolist():
        r = bytearray(t[a:a + m].tobytes())
        for x in np.flatnonzero(rng.random(m) < sub).tolist():
            r[x] = b"ACGT"[int(rng.integers(0, 4))]
        for x in sorted(np.flatnonzero(rng.random(m) < indel).tolist(), reverse=True):
            if rng.random() < 0.5:
                del r[x]
            else:
                r.insert(x, b"ACGT"[int(rng.integers(0, 4))])
        out.append(bytes(r[:m]) if len(r) >= m else bytes(r) + t[a + len(r):a + m].tobytes())
    return out


def test_scale_reads_with_indels_against_c_statement():
    rng = np.random.default_rng(58)
    t = gen.dna(10_000_000)
    text = _u8(t)
    reads = _reads(t, rng, 10_000, 150, 0.01, 0.005)
    cuts = np.unique(rng.integers(1, len(t), 9000))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for table, st in (("text", SuffixTable(text)), ("docs", DocumentSuffixTable(docs))):
        for k in (4, 8):
            off, pos, dist = st.approximate_positions_batch(reads, k, metric="edit")
            assert int(off[-1]) == len(pos) and len(pos) >= len(reads) // 2 and (dist <= k).all()
            for q in rng.choice(len(reads), 8, replace=False).tolist():
                want = edit_check.edit(text, None if table == "text" else starts, [reads[q]], k)
                a, b = int(off[q]), int(off[q + 1])
                assert np.array_equal(pos[a:b], want[1]) and np.array_equal(dist[a:b], want[2]), (table, k, q)
