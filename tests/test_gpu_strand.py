"""Approximate positions on both DNA strands (B200SA_APPROX_BOTH_STRANDS on b200sa_approx_positions_dev and
b200sa_docs_approx_positions_dev, strands="both" on the approximate_* methods of SuffixTable and
DocumentSuffixTable), for every mix of the edit metric, IUPAC queries and best hits: against tests/model_strand.py
on small sets, each strand's sublist against the call without the flag on q and on a host-built rc(q), and the
serial C statements run on q and rc(q) on large sets."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import approx_check, edit_check, iupac_check, model_best, model_docs, model_strand
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_approx import _queries as _plain_queries
from tests.test_gpu_docs import _families, _u8
from tests.test_gpu_edit import _reads
from tests.test_gpu_iupac import _degenerate, _guides, _masked_dna
from tests.test_gpu_iupac import _queries as _iupac_queries

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
MINUS = model_strand.MINUS
METRIC = {"hamming": 0, "edit": EDIT}
COMBOS = [(metric, iupac, best) for metric in ("hamming", "edit") for iupac in (False, True) for best in (None, 1)]


def _kf(k, metric, iupac, best):
    return k | METRIC[metric] | (IUPAC if iupac else 0) | (0 if best is None else (best << 8) | BEST) | BOTH


def _packed(res):
    """(offsets, pos, d | MINUS) of the four arrays strands="both" returns."""
    off, pos, dist, minus = res
    assert dist.dtype == np.uint32 and minus.dtype == bool and not (dist & MINUS).any()
    return off, pos, dist | np.where(minus, np.uint32(MINUS), np.uint32(0))


def _dna_queries(rng, docs, k):
    """DNA-like queries with a palindrome, m = 0, 0 < m <= k, and document substrings with their reverse
    complements."""
    qs = [b"", b"A", b"ACGT", b"GAATTC", b"AC" * (k + 1)]
    for d in [d for d in docs if d][:4]:
        m = int(rng.integers(1, len(d) + 1))
        a = int(rng.integers(0, len(d) - m + 1))
        qs += [d[a:a + m], model_strand.revcomp(d[a:a + m])]
    return qs


@pytest.mark.parametrize("metric,iupac,best", COMBOS)
def test_families_equal_model(metric, iupac, best):
    rng = np.random.default_rng(200 + COMBOS.index((metric, iupac, best)))
    sets = _families(rng)[::4] + [[_masked_dna(rng, int(rng.integers(1, 120))) for _ in range(3)] for _ in range(8)]
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = [0, 1, 2, 3, 4, 31][i % 6]
        if iupac:
            qs = _iupac_queries(rng, docs, k)
        else:
            qs = (_plain_queries(rng, docs, k) if i % 2 else _dna_queries(rng, docs, k))
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = model_strand.brute(docs, qs, k, metric, iupac, best)
        assert _same(_fetch(ctx, text, g, qs, _kf(k, metric, iupac, best), starts), want), (docs, k)
        st = DocumentSuffixTable(docs)
        kw = dict(metric=metric, iupac=iupac, best=best, strands="both")
        assert _same(_packed(st.approximate_positions_batch(qs, k, **kw)), want), (docs, k)
        assert np.array_equal(st.approximate_counts(qs, k, **kw), np.diff(want[0].astype(np.int64)))
        if len(docs) == 1:
            t1 = SuffixTable(text)
            assert _same(_fetch(ctx, text, g, qs, _kf(k, metric, iupac, best)), want), (docs, k)
            p, d, mi = t1.approximate_positions(qs[-1], k, **kw)
            a, b = int(want[0][-2]), int(want[0][-1])
            assert np.array_equal(p, want[1][a:b]) and np.array_equal(d | (mi.astype(np.uint32) << 31), want[2][a:b])
    ctx.close()


def _flagless(st, qs, k, metric, iupac, best):
    """Per query the (plus, minus) lists the call without the flag builds: the plain lists of q and of the
    host-built rc(q) at k, cut to d <= t(q) with best(q) over both when best is set."""
    plus = model_best.lists(st.approximate_positions_batch(qs, k, metric=metric, iupac=iupac))
    rcs = [model_strand.revcomp(q, iupac) for q in qs]
    minus = model_best.lists(st.approximate_positions_batch(rcs, k, metric=metric, iupac=iupac))
    out = []
    for hp, hm in zip(plus, minus):
        if best is not None:
            ds = [d for _, d in hp + hm]
            t = min(k, min(ds) + best) if ds else -1
            hp, hm = [h for h in hp if h[1] <= t], [h for h in hm if h[1] <= t]
        out.append((hp, hm))
    return out


@pytest.mark.parametrize("metric,iupac,best", COMBOS)
def test_sublists_equal_the_flagless_call(metric, iupac, best):
    rng = np.random.default_rng(300 + COMBOS.index((metric, iupac, best)))
    text = _masked_dna(rng, 4000)
    docs = [text[:1500], b"", text[1500:]]
    up = text.upper()
    qs = [bytes(b if b in b"ACGT" else ord("A") for b in up[a:a + int(m)])
          for a, m in zip(rng.integers(0, len(text) - 30, 20), rng.integers(1, 30, 20))]
    if iupac:
        qs = [_degenerate(rng, q, 0.1) for q in qs]
    qs = qs + [model_strand.revcomp(q, iupac) for q in qs[:5]] + [b"", b"ACGT", b"GAATTC"]
    for st in (SuffixTable(text), DocumentSuffixTable(docs)):
        for k in (0, 1, 2, 3, 4, 31):
            got = st.approximate_positions_batch(qs, k, metric=metric, iupac=iupac, best=best, strands="both")
            want = _flagless(st, qs, k, metric, iupac, best)
            assert model_strand.strand_lists(_packed(got)) == want, (k, type(st).__name__)
            assert all(h == model_strand.merge(hp, hm) for h, (hp, hm) in zip(model_best.lists(_packed(got)), want))


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_palindromes_empty_short_and_long_queries(metric):
    rng = np.random.default_rng(310)
    t = gen.dna(30_000)
    text = _u8(t)
    long_qs = [_reads(t[:12000], rng, 1, 1000, 0.001, 0.001)[0],                  # inside either table's documents
               model_strand.revcomp(_reads(t[13000:], rng, 1, 5000, 0.0002, 0.0002)[0])]
    for st in (SuffixTable(text), DocumentSuffixTable([text[:12000], text[12000:]])):
        k = 3
        off, pos, dist, minus = st.approximate_positions_batch([b"ACGT", b"GAATTC", b"", b"AC", b"G"], k,
                                                               metric=metric, strands="both")
        for q in range(2):                                                  # palindromes: every hit twice
            a, b = int(off[q]), int(off[q + 1])
            assert b > a and np.array_equal(pos[a:b:2], pos[a + 1:b:2]) and not minus[a:b:2].any()
            assert minus[a + 1:b:2].all() and np.array_equal(dist[a:b:2], dist[a + 1:b:2])
        assert off[2] == off[3]                                             # m = 0
        for q in (3, 4):                                                    # 0 < m <= k: every window twice
            a, b = int(off[q]), int(off[q + 1])
            one = st.approximate_positions_batch([[b"AC", b"G"][q - 3]], k, metric=metric)[1]
            assert np.array_equal(pos[a:b], np.repeat(one, 2))
        if metric == "hamming":
            continue
        for best in (None, 0):
            got = st.approximate_positions_batch(long_qs, 8, metric=metric, best=best, strands="both")
            want = _flagless(st, long_qs, 8, metric, False, best)
            assert model_strand.strand_lists(_packed(got)) == want, best
            assert got[3][int(got[0][1]):].sum() > 0                        # the 5000-byte query's minus hit


def test_only_the_minus_strand_holds_the_best_hit():
    t = gen.dna(20_000)
    text = bytearray(_u8(t))
    q = bytes(text[5000:5030])
    text[5007] = ord("A") if text[5007] != ord("A") else ord("C")          # the plus locus: one substitution
    text[12000:12030] = model_strand.revcomp(q)                            # the minus locus: exact
    text = bytes(text)
    for metric in ("hamming", "edit"):
        for st in (SuffixTable(text), DocumentSuffixTable([text[:9000], text[9000:]])):
            off, pos, dist, minus = st.approximate_positions_batch([q], 4, metric=metric, strands="both")
            assert (5000 in pos[~minus].tolist()) and 12000 in pos[minus].tolist()
            off, pos, dist, minus = st.approximate_positions_batch([q], 4, metric=metric, best=0, strands="both")
            assert pos.tolist() == [12000] and minus.tolist() == [True] and dist.tolist() == [0], metric
            assert st.approximate_counts([q], 4, metric=metric, best=0, strands="both").tolist() == [1]


def test_cap_protocol_null_distances_and_counts():
    rng = np.random.default_rng(330)
    text = _masked_dna(rng, 3000)
    sa = SuffixTable(text).table()
    up = text.upper()
    qs = [bytes(b if b in b"ACGT" else 65 for b in up[a:a + 12]) for a in rng.integers(0, 2980, 20)]
    qs = qs + [model_strand.revcomp(q) for q in qs[:4]] + [b"GAATTC", b"", b"AN"]
    ctx = _lib.Context(0)
    for metric, iupac, best in COMBOS:
        kf = _kf(2, metric, iupac, best)
        want = model_strand.brute([text], qs, 2, metric, iupac, best)
        total = int(want[0][-1])
        assert total > 1
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, 0, buf=total + 5)             # counts only
        assert tot == total and np.array_equal(off, want[0])
        assert (pos == MARK).all() and (dist == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total - 1, buf=total + 5)     # too small: offsets only
        assert tot == total and np.array_equal(off, want[0])
        assert (pos == MARK).all() and (dist == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, buf=total + 5)         # fits: nothing past total
        assert tot == total and np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
        tot, off, pos, dist = _abi(ctx, text, sa, qs, kf, total, with_mis=False, buf=total + 5)
        assert tot == total and np.array_equal(pos[:total], want[1]) and (pos[total:] == MARK).all()
        st = SuffixTable(text)
        kw = dict(metric=metric, iupac=iupac, best=best, strands="both")
        res = st.approximate_positions_batch(qs, 2, **kw)
        assert np.array_equal(st.approximate_counts(qs, 2, **kw), np.diff(res[0].astype(np.int64)))
        assert all(len(x) == total for x in res[1:])
    ctx.close()


@pytest.mark.parametrize("shift", [(1, 3), (3, 2)])
def test_unaligned_buffers(shift):
    rng = np.random.default_rng(340)
    text = _masked_dna(rng, 900) + bytes(range(256))
    sa = SuffixTable(text).table()
    qs = [bytes(b if b in b"ACGT" else 67 for b in text.upper()[a:a + m])
          for m in (1, 3, 9, 17) for a in rng.integers(0, 880, 5)] + [b"NNN", b"GAATTC"]
    ctx = _lib.Context(0)
    starts = np.array([0, 300, 300, 900], dtype=np.uint32)
    g, _ = ctx.docs_build(np.frombuffer(text, dtype=np.uint8), starts, with_lcp=False)
    docs = [text[0:300], b"", text[300:900], text[900:]]
    for metric, k, iupac, best in (("hamming", 0, False, None), ("hamming", 2, True, None), ("edit", 1, False, 0),
                                   ("edit", 2, True, 1)):
        kf = _kf(k, metric, iupac, best)
        assert _same(_fetch(ctx, text, sa, qs, kf, shift=shift),
                     model_strand.brute([text], qs, k, metric, iupac, best)), k
        assert _same(_fetch(ctx, text, g, qs, kf, starts, shift=shift),
                     model_strand.brute(docs, qs, k, metric, iupac, best)), k
    ctx.close()


def test_repeated_calls_are_identical():
    rng = np.random.default_rng(350)
    t = gen.dna(200_000)
    st = SuffixTable(_u8(t))
    qs = _reads(t, rng, 300, 40, 0.02, 0.01)
    qs = qs[:150] + [model_strand.revcomp(q) for q in qs[150:]]
    for metric, k, best in (("hamming", 3, None), ("edit", 2, None), ("edit", 3, 0)):
        a = st.approximate_positions_batch(qs, k, metric=metric, best=best, strands="both")
        b = st.approximate_positions_batch(qs, k, metric=metric, best=best, strands="both")
        assert _same(a, b) and int(a[0][-1]) > 0


def test_bad_arguments():
    ctx = _lib.Context(0)
    text = b"ACGTACGTNNacgtGAATTC"
    sa = SuffixTable(text).table()
    for extra in (0, EDIT, IUPAC, EDIT | IUPAC, BEST | (1 << 8), BEST | EDIT, BEST | IUPAC | (2 << 8),
                  BEST | EDIT | IUPAC):
        kf = 1 | extra | BOTH                                              # bit 28 is accepted in every mix
        assert _same(_fetch(ctx, text, sa, [b"ACG", b"GAATTC"], kf),
                     model_strand.brute([text], [b"ACG", b"GAATTC"], 1, "edit" if extra & EDIT else "hamming",
                                        bool(extra & IUPAC), (extra >> 8) & 0xFF if extra & BEST else None)), hex(kf)
    for bit in (19, 22, 23, 26, 29, 30):
        for kf in (1 | BOTH | (1 << bit), 1 | BEST | BOTH | (1 << bit), 1 | (1 << bit)):
            with pytest.raises(_lib.B200SAError) as e:
                _abi(ctx, text, sa, [b"ACG"], kf, 0)
            assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in str(e.value), hex(kf)
    for kf in (32 | BOTH, 32 | EDIT | BOTH):
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"ACG"], kf, 0)
        assert e.value.code == BAD_ARG and "k above B200SA_APPROX_MAX_K" in str(e.value), hex(kf)
    for kf in (1 | IUPAC | BOTH, 1 | EDIT | IUPAC | BOTH, 1 | BEST | IUPAC | BOTH):   # the caller's offset
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"ACGT", b"AC-G"], kf, 0)
        msg = str(e.value)
        assert e.value.code == BAD_ARG and "0x2d" in msg and "offset 6" in msg, msg
    for kf in (1 | BOTH, 1 | BEST | BOTH, 1 | IUPAC | BOTH):              # q_off[nq] above B200SA_MAX_N / 2
        with pytest.raises(_lib.B200SAError) as e:
            _abi(ctx, text, sa, [b"ACGT"], kf, 0, off=[0, 2 ** 31 + 1])
        assert e.value.code == TOO_LARGE, hex(kf)
    for bad in ("Both", "reverse", None, True, 1):
        with pytest.raises(ValueError):
            SuffixTable(text).approximate_positions(b"ACG", 1, strands=bad)
        with pytest.raises(ValueError):
            DocumentSuffixTable([text]).approximate_counts([b"ACG"], 1, metric="edit", strands=bad)
    assert _same(_fetch(ctx, text, sa, [b"ACG"], 1 | BOTH), model_strand.brute([text], [b"ACG"], 1))
    ctx.close()


def _check_sample(st, text, starts, qs, k, metric, iupac, off, pos, dist, minus, picks):
    """Queries `picks` against the serial C statement run on q and on rc(q), merged on the host."""
    for q in picks:
        rc = model_strand.revcomp(qs[q], iupac)
        if iupac:
            fw, rv = (iupac_check.iupac(text, starts, [x], k, metric) for x in (qs[q], rc))
        else:
            check = approx_check.approx if metric == "hamming" else edit_check.edit
            fw, rv = (check(text, starts, [x], k) for x in (qs[q], rc))
        want = model_strand.merge(model_best.lists(fw)[0], model_best.lists(rv)[0])
        a, b = int(off[q]), int(off[q + 1])
        got = [(p, d | (MINUS if m else 0)) for p, d, m in zip(pos[a:b].tolist(), dist[a:b].tolist(),
                                                               minus[a:b].tolist())]
        assert got == want, q


@pytest.mark.parametrize("metric", ["hamming", "edit"])
def test_scale_reads_and_guides_against_c_statements(metric):
    rng = np.random.default_rng(360)
    t = gen.dna(10_000_000)
    text = _u8(t)
    reads = _reads(t, rng, 10_000, 150, 0.01, 0.005 if metric == "edit" else 0)
    reads = [model_strand.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
    guides = [g for g in _guides(t, rng, 1000) if g.endswith(b"NGG")]
    guides = [model_strand.revcomp(g, True) if i % 2 else g for i, g in enumerate(guides)]
    cuts = np.unique(rng.integers(1, len(t), 9000))
    starts = np.r_[0, cuts].astype(np.uint32)
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    for name, st in (("text", SuffixTable(text)), ("docs", DocumentSuffixTable(docs))):
        s = None if name == "text" else starts
        k = 4
        off, pos, dist, minus = st.approximate_positions_batch(reads, k, metric=metric, strands="both")
        assert int(off[-1]) == len(pos) and (dist <= k).all()
        hit = np.diff(off.astype(np.int64)) > 0
        assert hit.sum() >= len(reads) * 3 // 4
        has_minus = np.array([minus[int(off[q]):int(off[q + 1])].any() for q in range(len(reads))])
        assert has_minus[1::2].sum() >= len(reads) // 4 and has_minus[::2].sum() < len(reads) // 8
        _check_sample(st, text, s, reads, k, metric, False, off, pos, dist, minus,
                      rng.choice(len(reads), 4, replace=False).tolist())
        kg = 3 if metric == "hamming" else 2
        off, pos, dist, minus = st.approximate_positions_batch(guides, kg, metric=metric, iupac=True, strands="both")
        assert int(off[-1]) == len(pos) and (dist <= kg).all() and minus.any() and (~minus).any()
        _check_sample(st, text, s, guides, kg, metric, True, off, pos, dist, minus,
                      rng.choice(len(guides), 6, replace=False).tolist())
