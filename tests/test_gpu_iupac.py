"""IUPAC queries in approximate positions (B200SA_APPROX_IUPAC on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev, iupac=True on the approximate_* methods of SuffixTable and DocumentSuffixTable)
against the definition of tests/model_iupac.py on small sets and the serial C statement of tests/iupac_check.c
on large ones, and against the call without the flag where the two must agree."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import iupac_check, model_approx, model_docs, model_iupac
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
METRIC = {"hamming": 0, "edit": EDIT}
CODES = b"ACGTURYSWKMBDHVN"
VALID = set(CODES + CODES.lower())


def _masked_dna(rng, n):
    """DNA with soft-masked runs and N, U bytes."""
    t = bytearray(_u8(gen.dna(n)))
    for a in rng.integers(0, max(n - 8, 1), n // 40):
        t[a:a + 8] = bytes(t[a:a + 8]).lower()
    for a in rng.integers(0, max(n, 1), n // 60):
        t[a] = int(b"NU"[int(rng.integers(0, 2))])
    return bytes(t)


def _degenerate(rng, q, rate):
    q = bytearray(q)
    for x in range(len(q)):
        if rng.random() < rate:
            q[x] = int(CODES[int(rng.integers(4, len(CODES)))])
    return bytes(q)


def _queries(rng, docs, k):
    """IUPAC queries: m = 0, short and all-degenerate ones, fewer than k + 1 concrete symbols, and substrings of
    the documents (bytes that are no code turned into N) with degenerate positions and either case."""
    qs = [b"", b"N", b"n" * (k + 2), b"NGG", b"ACGT", bytes(int(x) for x in rng.choice(list(CODES), 6))]
    qs.append(b"N" * (k + 1) + b"A" * min(k, 3) + b"N")
    for d in [d for d in docs if d][:6]:
        m = int(rng.integers(1, len(d) + 1))
        a = int(rng.integers(0, len(d) - m + 1))
        src = bytes(b if b in VALID else ord("N") for b in d[a:a + m])
        q = _degenerate(rng, src.upper(), 0.2)
        qs += [q, q.lower()]
    return qs


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_families_equal_model(metric):
    rng = np.random.default_rng(91 if metric == "hamming" else 92)
    sets = _families(rng)[::2] + [[_masked_dna(rng, int(rng.integers(1, 200))) for _ in range(3)] for _ in range(20)]
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = [0, 1, 2, 3, 4, 31][i % 6]
        qs = _queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_iupac.brute(docs, qs, k, metric)
        assert _same(_fetch(ctx, text, g, qs, k | METRIC[metric] | IUPAC, starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        assert _same(st.approximate_positions_batch(qs, k, metric=metric, iupac=True), want), (docs, k)
        assert np.array_equal(st.approximate_counts(qs, k, metric=metric, iupac=True),
                              np.diff(want[0].astype(np.int64)))
        if len(docs) == 1:
            t1 = SuffixTable(text)
            assert _same(t1.approximate_positions_batch(qs, k, metric=metric, iupac=True), want), (docs, k)
            p, d = t1.approximate_positions(qs[-1], k, metric=metric, iupac=True)
            a, b = int(want[0][-2]), int(want[0][-1])
            assert np.array_equal(p, want[1][a:b]) and np.array_equal(d, want[2][a:b])
    ctx.close()


def test_concrete_uppercase_queries_equal_the_plain_call():
    rng = np.random.default_rng(93)
    text = _masked_dna(rng, 30_000)
    docs = [text[:9000], b"", text[9000:20000], text[20000:]]
    up = text.upper()
    qs = [_u8(up[a:a + int(m)]) for a, m in zip(rng.integers(0, len(text) - 40, 80), rng.integers(1, 40, 80))]
    qs = [bytes(b if b in b"ACGT" else ord("A") for b in q) for q in qs] + [b"", b"A", b"ACGTACGTTT"]
    for st in (SuffixTable(text), DocumentSuffixTable(docs)):
        for metric in ("hamming", "edit"):
            for k, best in ((0, None), (2, None), (5, None), (3, 0), (4, 2)):
                plain = st.approximate_positions_batch(qs, k, metric=metric, best=best)
                flagged = st.approximate_positions_batch(qs, k, metric=metric, best=best, iupac=True)
                assert _same(plain, flagged), (metric, k, best)


def test_lowercase_and_u_queries():
    rng = np.random.default_rng(94)
    text = _masked_dna(rng, 20_000)
    up = text.upper()
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else ord("N") for b in up[a:a + 24]), 0.15)
          for a in rng.integers(0, len(text) - 24, 60)]
    st = SuffixTable(text)
    for metric, k in (("hamming", 3), ("edit", 2)):
        want = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
        for other in ([q.lower() for q in qs], [q.replace(b"T", b"U") for q in qs],
                      [q.lower().replace(b"t", b"u") for q in qs]):
            assert _same(st.approximate_positions_batch(other, k, metric=metric, iupac=True), want), metric


def test_k0_is_the_union_of_the_expansions():
    rng = np.random.default_rng(95)
    text = _masked_dna(rng, 50_000)
    docs = [text[:20000], b"", text[20000:]]
    up = text.upper()
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else ord("A") for b in up[a:a + 9]), 0.3)
          for a in rng.integers(0, len(text) - 9, 40)] + [b"NGG", b"RYN", b"ACGTN"]
    qs = [q for q in qs if len(model_iupac.expansions(q)) <= 256]
    st, dt = SuffixTable(text), DocumentSuffixTable(docs)
    off, pos, mis = st.approximate_positions_batch(qs, 0, iupac=True)
    doff, dpos, _ = dt.approximate_positions_batch(qs, 0, iupac=True)
    assert not mis.any()
    for q in range(len(qs)):
        exp = model_iupac.expansions(qs[q])
        union = np.unique(np.concatenate([st.positions(e).astype(np.int64) for e in exp] + [np.zeros(0, np.int64)]))
        assert np.array_equal(pos[int(off[q]):int(off[q + 1])], union), qs[q]
        rows = [dt.positions(e) for e in exp]
        flat = np.concatenate([dt.doc_starts()[r[:, 0]].astype(np.int64) + r[:, 1] for r in rows if len(r)]
                              + [np.zeros(0, np.int64)])
        assert np.array_equal(dpos[int(doff[q]):int(doff[q + 1])], np.unique(flat)), qs[q]


def test_whole_table_queries():
    rng = np.random.default_rng(96)
    text = _masked_dna(rng, 3000)
    docs = [text[:1000], b"", text[1000:2500], text[2500:]]
    qs = [b"N" * 6, b"NNANN", b"NANGN", b"N" * 21 + b"GG", b"n", b"RYKM"]
    for metric in ("hamming", "edit"):
        for k in (1, 3):
            for d in ([text], docs):
                st = SuffixTable(text) if len(d) == 1 else DocumentSuffixTable(d)
                got = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
                assert _same(got, model_iupac.brute(d, qs, k, metric)), (metric, k, len(d))


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_best_equals_the_flagged_call_at_its_threshold(metric):
    rng = np.random.default_rng(97)
    text = _masked_dna(rng, 40_000)
    docs = [text[:15000], text[15000:]]
    up = text.upper()
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else ord("N") for b in up[a:a + 20]), 0.1)
          for a in rng.integers(0, len(text) - 20, 60)]
    qs = [_degenerate(rng, q, 0.05) for q in qs] + [b"ACGTNNACGTNNACGTNNAC", b"N" * 4, b""]
    for st in (SuffixTable(text), DocumentSuffixTable(docs)):
        for k, s in ((3, 0), (4, 1), (2, 2)):
            off, pos, dist = st.approximate_positions_batch(qs, k, metric=metric, best=s, iupac=True)
            full = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
            for q in range(len(qs)):
                d = full[2][int(full[0][q]):int(full[0][q + 1])]
                if len(d) == 0:
                    assert off[q] == off[q + 1]
                    continue
                t = min(k, int(d.min()) + s)
                at = st.approximate_positions_batch([qs[q]], t, metric=metric, iupac=True)
                a, b = int(off[q]), int(off[q + 1])
                assert np.array_equal(pos[a:b], at[1]) and np.array_equal(dist[a:b], at[2]), (k, s, q)


def test_cap_protocol_and_null_distances():
    rng = np.random.default_rng(98)
    text = _masked_dna(rng, 3000)
    sa = SuffixTable(text).table()
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else 65 for b in text.upper()[a:a + 12]), 0.2)
          for a in rng.integers(0, 2980, 30)] + [b"NGG", b"", b"AN"]
    ctx = _lib.Context(0)
    for metric in ("hamming", "edit"):
        kf = 2 | METRIC[metric] | IUPAC
        want = model_iupac.brute([text], qs, 2, metric)
        total = int(want[0][-1])
        assert total > 1
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, 0, buf=total + 5)           # counts only
        assert tot == total and np.array_equal(off, want[0])
        assert (pos == MARK).all() and (dist == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total - 1, buf=total + 5)   # too small: offsets only
        assert tot == total and np.array_equal(off, want[0])
        assert (pos == MARK).all() and (dist == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, buf=total + 5)       # fits: nothing past total
        assert tot == total and np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, with_mis=False, buf=total + 5)
        assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all()
    ctx.close()


@pytest.mark.parametrize("shift", [(1, 3), (3, 2)])
def test_unaligned_buffers(shift):
    rng = np.random.default_rng(99)
    text = _masked_dna(rng, 900) + bytes(range(256))
    sa = SuffixTable(text).table()
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else 67 for b in text.upper()[a:a + m]), 0.2)
          for m in (1, 3, 9, 17) for a in rng.integers(0, 880, 5)] + [b"NNN"]
    ctx = _lib.Context(0)
    starts = np.array([0, 300, 300, 900], dtype=np.uint32)
    g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
    docs = [text[0:300], b"", text[300:900], text[900:]]
    for metric, k in (("hamming", 0), ("hamming", 2), ("edit", 1)):
        kf = k | METRIC[metric] | IUPAC
        assert _same(_fetch(ctx, text, sa, qs, kf, shift=shift), model_iupac.brute([text], qs, k, metric)), k
        assert _same(_fetch(ctx, text, g, qs, kf, starts, shift=shift), model_iupac.brute(docs, qs, k, metric)), k
    ctx.close()


def test_empty_documents():
    docs = [b"", b"ACGTA", b"", b"", b"T", b"cc", b""]
    st = DocumentSuffixTable(docs)
    qs = [b"N", b"NN", b"RYN", b"ACGTN", b"", b"CC", b"cc"]
    for metric in ("hamming", "edit"):
        for k in (0, 1, 2, 5, 31):
            got = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
            assert _same(got, model_iupac.brute(docs, qs, k, metric)), (metric, k)
    off, pos, _ = DocumentSuffixTable([b"", b""]).approximate_positions_batch(qs, 3, iupac=True)
    assert not off.any() and len(pos) == 0
    off, pos, _ = SuffixTable(b"").approximate_positions_batch(qs, 3, metric="edit", iupac=True)
    assert not off.any() and len(pos) == 0
    assert len(st.approximate_positions_batch([], 2, iupac=True)[0]) == 1


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"ACGTACGTNNacgt"
    sa = SuffixTable(text).table()
    for q, off, byte in ((b"AC-G", 2, 0x2D), (b"A.", 1, 0x2E), (b"ACGX", 3, 0x58), (b"\x00", 0, 0)):
        for kf in (1 | IUPAC, 1 | EDIT | IUPAC, 1 | BEST | IUPAC):
            with pytest.raises(_lib.B200SAError) as e:
                _abi(ctx, text, sa, [b"ACGT", q], kf, 0)
            msg = str(e.value)
            assert e.value.code == BAD_ARG and ("0x%02x" % byte) in msg and ("offset %d" % (4 + off)) in msg, msg
    for kf in (1 | IUPAC | 0x20000, 1 | IUPAC | 0x2000000, 1 | IUPAC | BEST | 0x40000, 1 | IUPAC | (1 << 31)):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"ACG"], kf, 0)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value), hex(kf)
    for bad in (1, 0, None, "yes", np.int64(1)):
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_positions(b"ACG", 1, iupac=bad)
        with pytest.raises(ValueError):
            DocumentSuffixTable([text]).approximate_counts([b"ACG"], 1, metric="edit", iupac=bad)
    assert _same(_fetch(ctx, text, sa, [b"NNG"], 31 | IUPAC), model_iupac.brute([text], [b"NNG"], 31))
    ctx.close()


def test_repeated_calls_are_identical():
    rng = np.random.default_rng(100)
    text = _masked_dna(rng, 200_000)
    st = SuffixTable(text)
    qs = [_degenerate(rng, bytes(b if b in b"ACGT" else 71 for b in text.upper()[a:a + 23]), 0.1)
          for a in rng.integers(0, len(text) - 23, 300)] + [b"ACGTNNNN"]
    for metric, k in (("hamming", 3), ("edit", 2)):
        a = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
        b = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
        assert _same(a, b)
        want = iupac_check.iupac(text, None, qs, k, metric)
        assert _same(a, want), metric


def _guides(t, rng, count):
    """20-nt guides + NGG from the text, with a few substitutions, and degenerate 20-mers."""
    bases = np.frombuffer(b"ACGT", dtype=np.uint8)
    out = []
    for a in rng.integers(0, len(t) - 23, count):
        g = t[a:a + 20].copy()
        sub = rng.random(20) < 0.05
        g[sub] = rng.choice(bases, int(sub.sum()))
        out.append(g.tobytes() + b"NGG")
    for a in rng.integers(0, len(t) - 20, count):
        q = bytearray(t[a:a + 20].tobytes())
        for x in rng.choice(20, 3, replace=False):
            q[int(x)] = int(b"RYSWKMBDHV"[int(rng.integers(0, 10))])
        out.append(bytes(q))
    return out


@pytest.mark.parametrize("metric,k", [("hamming", 3), ("edit", 2)])
def test_scale_guides_against_c_statement(metric, k):
    rng = np.random.default_rng(101)
    t = gen.dna(10_000_000)
    text = _u8(t)
    qs = _guides(t, rng, 500)
    cuts = np.unique(rng.integers(1, len(t), 9000))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for name, st in (("text", SuffixTable(text)), ("docs", DocumentSuffixTable(docs))):
        off, pos, dist = st.approximate_positions_batch(qs, k, metric=metric, iupac=True)
        assert int(off[-1]) == len(pos) and len(pos) >= len(qs) // 2 and (dist <= k).all()
        for q in rng.choice(len(qs), 8, replace=False).tolist():
            want = iupac_check.iupac(text, None if name == "text" else starts, [qs[q]], k, metric)
            a, b = int(off[q]), int(off[q + 1])
            assert np.array_equal(pos[a:b], want[1]) and np.array_equal(dist[a:b], want[2]), (name, q)
