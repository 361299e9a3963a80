"""Best hits of approximate positions (B200SA_APPROX_BEST on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev, best= on the approximate_* methods of SuffixTable and DocumentSuffixTable), for
both metrics: every query's list against the plain GPU call at t(q) = min(k, best(q) + s), against
tests/model_best.py on small sets, and against best(q) from the serial C statements on large ones."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import approx_check, edit_check, model_approx, model_best, model_docs
from tests.test_edit_model import edited
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_edit import _queries, _reads

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
METRIC = {"hamming": 0, "edit": EDIT}
FAMILY_KS = [0, 1, 2, 3, 5, 31]


def slack(s):
    return s << 8                               # B200SA_APPROX_SLACK(s)


def _at_thresholds(fetch, plain_k, k, s):
    """The BEST lists as the plain calls build them: best(q) from the plain lists at k, then q's plain list at
    t(q); fetch(t) is the plain call at t."""
    bests = [min(d for _, d in h) if h else None for h in model_best.lists(plain_k)]
    ts = [model_best.threshold(b, k, s) for b in bests]
    at = {t: model_best.lists(fetch(t)) for t in set(ts) if t is not None}
    return model_approx._pack([at[t][q] if t is not None else [] for q, t in enumerate(ts)]), bests


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_families_equal_plain_call_at_each_threshold_and_model(metric):
    rng = np.random.default_rng(71 + len(metric))
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = FAMILY_KS[i % len(FAMILY_KS)]
        s = [0, 1, 2, k][(i // len(FAMILY_KS)) % 4]
        qs = _queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        tables = [(g, starts)]
        if len(docs) == 1:                                     # one document is the single text
            tables.append((ctx.build(np.frombuffer(text, dtype=np.uint8)) if text else np.zeros(0, np.uint32), None))
        for table, st in tables:
            kf = k | METRIC[metric]
            plain = _fetch(ctx, text, table, qs, kf, st)
            got = _fetch(ctx, text, table, qs, kf | slack(s) | BEST, st)
            want, bests = _at_thresholds(lambda t: _fetch(ctx, text, table, qs, t | METRIC[metric], st), plain, k, s)
            assert _same(got, want), (docs, k, s)
            if s == 0:
                assert all(d == b for h, b in zip(model_best.lists(got), bests) for _, d in h)
            if s >= k:
                assert _same(got, plain), (docs, k, s)
            if len(text) <= 200 and sum(len(q) for q in qs) <= 600:
                assert _same(got, model_best.select(docs, qs, k, s, metric)), (docs, k, s)
        dst = DocumentSuffixTable(docs)
        off, pos, dist = dst.approximate_positions_batch(qs, k, metric=metric, best=s)
        assert _same((off, pos, dist), got), (docs, k, s)
        assert np.array_equal(dst.approximate_counts(qs, k, metric=metric, best=s), np.diff(off.astype(np.int64)))
        if len(docs) == 1:
            t1 = SuffixTable(text)
            assert _same(t1.approximate_positions_batch(qs, k, metric=metric, best=s), got), (docs, k, s)
            p, d = t1.approximate_positions(qs[-1], k, metric=metric, best=s)
            a, b = int(off[-2]), int(off[-1])
            assert np.array_equal(p, pos[a:b]) and np.array_equal(d, dist[a:b])
    ctx.close()


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_slack_k_is_the_plain_call_and_slack_0_the_best_stratum(metric):
    rng = np.random.default_rng(72)
    text = _u8(gen.dna(50_000))
    docs = [text[:20_000], b"", text[20_000:]]
    qs = [edited(rng, text[a:a + 40], int(rng.integers(0, 6)), b"ACGT") for a in rng.integers(0, 49_000, 200)]
    qs += [b"ACGTACGTAC", b"A", b"", b"NNNNNNNNNNNNNNNNNNNNNNNN"]
    for st in (SuffixTable(text), DocumentSuffixTable(docs)):
        for k in (0, 3, 6):
            plain = st.approximate_positions_batch(qs, k, metric=metric)
            for s in (k, k + 1, 31):
                assert _same(st.approximate_positions_batch(qs, k, metric=metric, best=s), plain), (k, s)
            off, pos, dist = st.approximate_positions_batch(qs, k, metric=metric, best=0)
            for q, h in enumerate(model_best.lists(plain)):
                low = min(d for _, d in h) if h else None
                a, b = int(off[q]), int(off[q + 1])
                assert pos[a:b].tolist() == [p for p, d in h if d == low], (k, q)
                assert (dist[a:b] == low).all()
            assert np.array_equal(st.approximate_counts(qs, k, metric=metric, best=0), np.diff(off.astype(np.int64)))


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_cap_protocol_and_null_distances(metric):
    rng = np.random.default_rng(73)
    text = _u8(gen.dna(3000))
    sa = SuffixTable(text).table()
    qs = [edited(rng, text[a:a + 12], int(rng.integers(0, 3)), b"ACGT") for a in rng.integers(0, 2980, 30)]
    qs += [b"ACGT", b"", b"AC", b"TTTTTTTTTTTTTTTTTTTTT"]
    ctx = _lib.Context(0)
    kf = 3 | METRIC[metric] | slack(1) | BEST
    want = model_best.select([text], qs, 3, 1, metric)
    total = int(want[0][-1])
    assert total > 1
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


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_edge_cases(metric):
    docs = [b"", b"abcab", b"", b"", b"b", b"cc", b""]
    qs = [b"x", b"zz", b"zzz", b"bcabz", b"", b"cc", b"ab", b"zzzzzzzzzz"]     # no hit, m = 0, 0 < m <= k
    st = DocumentSuffixTable(docs)
    for k in (0, 1, 2, 3, 5, 31):
        for s in (0, 1, 2, k):
            assert _same(st.approximate_positions_batch(qs, k, metric=metric, best=s),
                         model_best.select(docs, qs, k, s, metric)), (k, s)
    t1 = SuffixTable(b"abcab")
    for k, s in ((2, 0), (3, 1), (5, 5)):
        assert _same(t1.approximate_positions_batch(qs, k, metric=metric, best=s),
                     model_best.select([b"abcab"], qs, k, s, metric)), (k, s)
    for table in (DocumentSuffixTable([b"", b""]), SuffixTable(b"")):
        off, pos, dist = table.approximate_positions_batch(qs, 3, metric=metric, best=0)
        assert not off.any() and len(pos) == 0 and len(dist) == 0
    off, pos, _ = st.approximate_positions_batch([b"", b"zzzz"], 2, metric=metric, best=0)
    assert not off.any() and len(pos) == 0
    assert len(st.approximate_positions_batch([], 2, metric=metric, best=1)[0]) == 1


@pytest.mark.parametrize("shift", [(1, 3), (3, 2)])
def test_unaligned_buffers(shift):
    rng = np.random.default_rng(74)
    text = bytes(rng.integers(0, 256, 700, dtype=np.uint8)) + bytes(range(256)) + b"\x00\x00\xff\xff" * 5
    sa = SuffixTable(text).table()
    alpha = list(range(256))
    qs = [edited(rng, text[a:a + m], 1, alpha) for m in (1, 2, 3, 5, 9, 17, 33) for a in rng.integers(0, len(text) - m, 6)]
    qs += [text[-m:] for m in range(1, 12)] + [bytes([255, 255]), text[:5]]
    ctx = _lib.Context(0)
    starts = np.array([0, 300, 300, 956], dtype=np.uint32)
    g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
    docs = [text[0:300], b"", text[300:956], text[956:]]
    for metric in ("hamming", "edit"):
        for k, s in ((0, 0), (1, 0), (3, 1)):
            kf = k | METRIC[metric] | slack(s) | BEST
            assert _same(_fetch(ctx, text, sa, qs, kf, shift=shift), model_best.select([text], qs, k, s, metric))
            assert _same(_fetch(ctx, text, g, qs, kf, starts, shift=shift), model_best.select(docs, qs, k, s, metric))
    ctx.close()


def test_repeated_calls_are_identical_and_count_rounds():
    rng = np.random.default_rng(75)
    text = _u8(gen.dna(200_000))
    st = SuffixTable(text)
    qs = [edited(rng, text[a:a + 30], int(rng.integers(0, 4)), b"ACGT") for a in rng.integers(0, len(text) - 30, 300)]
    for metric in ("hamming", "edit"):
        a = st.approximate_positions_batch(qs, 5, metric=metric, best=1)
        b = st.approximate_positions_batch(qs, 5, metric=metric, best=1)
        assert _same(a, b)
    ctx = _lib.Context(0)
    sa = st.table()
    bests = [min(d for _, d in h) if h else None for h in model_best.lists(st.approximate_positions_batch(qs[:40], 5))]
    _fetch(ctx, text, sa, qs[:40], 5 | slack(0) | BEST)
    want = max(5 if b is None else b for b in bests) + 1
    assert ctx.stats()["doubling_rounds"] == want
    ctx.close()


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"abracadabra"
    sa = SuffixTable(text).table()
    for k in (3 | slack(1), 3 | slack(1) | EDIT):                  # slack bits without BEST: a threshold above 31
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abc"], k, 0)
        assert e.value.code == BAD_ARG and "k above B200SA_APPROX_MAX_K" in str(e.value), hex(k)
    for k in (32 | BEST, 3 | slack(32) | BEST, 32 | slack(32) | BEST | EDIT, 0xFF | BEST, 3 | slack(255) | BEST,
              3 | BEST | 0x20000, 3 | BEST | 0x40000, 3 | BEST | (1 << 31), 3 | BEST | 0x200000):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"abc"], k, 0)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value), hex(k)
    assert _same(_fetch(ctx, text, sa, [b"abc"], 31 | slack(31) | BEST | EDIT),
                 model_best.select([text], [b"abc"], 31, 31, "edit"))
    for bad in (True, -1, 32, 1.5, "0"):
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_positions(b"abc", 1, best=bad)
        with pytest.raises(ValueError):
            DocumentSuffixTable([text]).approximate_counts([b"abc"], 1, metric="edit", best=bad)
    ctx.close()


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_scale_reads_against_c_statement(metric):
    rng = np.random.default_rng(76)
    t = gen.dna(10_000_000)
    text = _u8(t)
    reads = _reads(t, rng, 10_000, 150, 0.01, 0.005)
    cuts = np.unique(rng.integers(1, len(t), 9000))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    check = approx_check.approx if metric == "hamming" else edit_check.edit
    for table, st in (("text", SuffixTable(text)), ("docs", DocumentSuffixTable(docs))):
        for k, s in ((4, 0), (8, 1)):
            off, pos, dist = st.approximate_positions_batch(reads, k, metric=metric, best=s)
            assert int(off[-1]) == len(pos) and len(pos) >= len(reads) // 4 and (dist <= k).all()
            for q in rng.choice(len(reads), 8, replace=False).tolist():
                full = check(text, None if table == "text" else starts, [reads[q]], k)
                d = full[2]
                keep = d <= (min(k, int(d.min()) + s) if len(d) else -1)
                a, b = int(off[q]), int(off[q + 1])
                assert np.array_equal(pos[a:b], full[1][keep]) and np.array_equal(dist[a:b], d[keep]), (table, k, q)
