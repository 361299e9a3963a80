"""Fixed symbols in IUPAC queries (B200SA_APPROX_FIXED on b200sa_docs_approx_positions_dev, fixed=True on the
approximate_positions* and approximate_counts methods): bit for bit against tests/model_fixed.py on small
collections for every mix of metric, best, strands, documents and align; the stated invariants on the device; a
few MB of DNA with CRISPR guides against the serial C statement on a sample; and the argument checks and listing
protocol."""
import numpy as np
import pytest

from suffix_b200 import DocumentSuffixTable, SuffixTable, _approx, _lib, gen
from tests import fixed_check, model_docs, model_fixed, model_iupac, model_strand
from tests.test_fixed_model import _queries, _text
from tests.test_gpu_approx import MARK, _abi, _fetch, _same
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG = -1
EDIT = 0x10000                                  # B200SA_APPROX_EDIT
BEST = 0x100000                                 # B200SA_APPROX_BEST
IUPAC = 0x1000000                               # B200SA_APPROX_IUPAC
FIXED = 0x2000000                               # B200SA_APPROX_FIXED
ALIGN = 0x8000000                               # B200SA_APPROX_ALIGN
BOTH = 0x10000000                               # B200SA_APPROX_BOTH_STRANDS
DOCS = 0x20000000                               # B200SA_APPROX_DOCUMENTS
MINUS = model_strand.MINUS
METRIC = {"hamming": 0, "edit": EDIT}
MIXES = [(metric, best, strands, mode) for metric in ("hamming", "edit") for best in (None, 0, 1)
         for strands in ("forward", "both") for mode in ("hits", "documents", "align")]


def _kf(k, metric, best, strands, mode="hits", fixed=True):
    return (k | METRIC[metric] | IUPAC | (FIXED if fixed else 0) | (0 if best is None else (best << 8) | BEST) |
            (BOTH if strands == "both" else 0) | {"hits": 0, "documents": DOCS, "align": ALIGN}[mode])


def _want(docs, qs, k, metric, best, strands, mode):
    return model_fixed.listing(docs, qs, k, metric, best, strands, documents=mode == "documents",
                               align_ops=mode == "align")


def _method(st, mode, batch=True):
    """The method of a mode: approximate_positions*, and for the listings the functions behind
    approximate_documents* and approximate_alignments*, which keep their keyword lists."""
    if mode == "hits":
        return getattr(st, "approximate_positions" + ("_batch" if batch else ""))
    f = {"documents": _approx.documents, "align": _approx.alignments}[mode]
    f = {"documents": _approx.documents_batch, "align": _approx.alignments_batch}[mode] if batch else f
    return lambda q, k, **kw: f(st, q, k, **kw)


def _fixed_queries(rng, docs, k):
    """_queries plus a PAM suffix of each class (ngg, nrg) and m <= k."""
    qs = _queries(rng, docs, k)
    text = b"".join(docs).upper()
    src = bytes(b if b in b"ACGT" else ord("A") for b in text)
    if len(src) >= 6:
        a = int(rng.integers(0, len(src) - 5))
        qs += [src[a:a + 3] + b"ngg", src[a:a + 3] + b"nrg", src[a:a + 3].lower() + src[a + 3:a + 6]]
    return qs + [b"acgt"[:max(k, 1)], b"N" * max(k, 1)]


@pytest.mark.parametrize("metric,best,strands,mode", MIXES)
def test_families_equal_model(metric, best, strands, mode):
    rng = np.random.default_rng(700 + MIXES.index((metric, best, strands, mode)))
    sets = _families(rng)[::12] + [[_text(rng, int(rng.integers(1, 60))) for _ in range(3)] for _ in range(6)]
    sets += [[b"", _text(rng, 50), b"", b"ACGT"]]
    ctx = _lib.Context(0)
    for i, docs in enumerate(sets):
        k = 31 if i == len(sets) - 1 else [0, 1, 2, 3][i % 4]
        if mode == "align" and k == 31:
            k = 3
        qs = _fixed_queries(rng, docs, k)
        g, _ = model_docs.brute(docs)
        text, starts = model_docs.concat(docs)
        want = _want(docs, qs, k, metric, best, strands, mode)
        assert _same(_fetch(ctx, text, g, qs, _kf(k, metric, best, strands, mode), starts), want), (docs, k)
        if len(docs) == 1 and mode == "hits":                      # a single text through the documents entry
            kw = dict(metric=metric, best=best, strands=strands, iupac=True, fixed=True)
            a = SuffixTable(text).approximate_positions_batch(qs, k, **kw)
            b = DocumentSuffixTable(docs).approximate_positions_batch(qs, k, **kw)
            assert _same(a, b), (docs, k)
    ctx.close()


def test_methods_equal_the_abi():
    rng = np.random.default_rng(710)
    docs = [_text(rng, 300).upper(), _text(rng, 200).upper()]
    st = DocumentSuffixTable(docs)
    qs = _fixed_queries(rng, docs, 2)
    for metric, best, strands, mode in MIXES[::5]:
        kw = dict(metric=metric, best=best, strands=strands, iupac=True, fixed=True)
        off = _method(st, mode)(qs, 2, **kw)[0]                    # hits, or listed documents
        assert np.array_equal(off, _want(docs, qs, 2, metric, best, strands, "hits" if mode == "align" else mode)[0])
        one = _method(st, mode, False)(qs[-3], 2, **kw)
        assert _same(one, _method(st, mode)([qs[-3]], 2, **kw)[1:])
    counts = st.approximate_counts(qs, 2, iupac=True, fixed=True, strands="both")
    assert np.array_equal(counts, np.diff(_want(docs, qs, 2, "hamming", None, "both", "hits")[0].astype(np.int64)))
    for kw in (dict(fixed=True), dict(fixed=1, iupac=True), dict(fixed=None, iupac=True)):
        with pytest.raises(ValueError):
            st.approximate_positions(b"ACGTngg", 1, **kw)


def test_invariants_on_the_device():
    rng = np.random.default_rng(720)
    t = gen.dna(200_000)
    text = _u8(t)
    cuts = np.unique(rng.integers(1, len(t), 40))
    docs = [text[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(t)])]
    starts = np.r_[0, cuts].astype(np.uint32)
    g = DocumentSuffixTable(docs).table()
    ctx = _lib.Context(0)
    guides = []
    for a in rng.integers(0, len(t) - 23, 60):
        s = bytearray(t[a:a + 20].tobytes())
        for x in rng.choice(20, int(rng.integers(0, 3)), replace=False):
            s[int(x)] = int(b"ACGT"[int(rng.integers(0, 4))])
        guides.append(bytes(s))
    upper = [s + b"NGG" for s in guides]
    pam = [s + b"ngg" for s in guides]
    for metric, best, strands, mode in MIXES:                      # 1: no lowercase is the call without the flag
        k = 2 if metric == "edit" else 3
        a = _fetch(ctx, text, g, upper, _kf(k, metric, best, strands, mode), starts)
        b = _fetch(ctx, text, g, upper, _kf(k, metric, best, strands, mode, fixed=False), starts)
        assert _same(a, b) and int(a[0][-1]) > 0, (metric, best, strands, mode)
    for strands in ("forward", "both"):                            # 2: Hamming filters, distances unchanged
        off0, pos0, d0 = _fetch(ctx, text, g, pam, _kf(3, "hamming", None, strands, fixed=False), starts)
        off1, pos1, d1 = _fetch(ctx, text, g, pam, _kf(3, "hamming", None, strands), starts)
        keep = np.zeros(len(pos0), dtype=bool)
        for q in range(len(pam)):
            for i in range(int(off0[q]), int(off0[q + 1])):
                minus = d0[i] >= MINUS
                Q = model_strand.revcomp(pam[q], True) if minus else pam[q]
                w, cls, fx = text[int(pos0[i]):int(pos0[i]) + len(Q)], model_iupac.classes(Q), model_fixed.marks(Q)
                keep[i] = all(w[x] in cls[x] for x in range(len(Q)) if fx[x])
        q_of = np.repeat(np.arange(len(pam)), np.diff(off0.astype(np.int64)))
        assert np.array_equal(pos1, pos0[keep]) and np.array_equal(d1, d0[keep])
        assert np.array_equal(off1[1:], np.cumsum(np.bincount(q_of[keep], minlength=len(pam))))
        assert len(pos1) < len(pos0)
    low = [s.lower() for s in guides[:20]] + [b"acgtn", b"nrg"]     # 3: all fixed is exact Hamming at 0
    exact = _fetch(ctx, text, g, low, _kf(0, "hamming", None, "forward", fixed=False), starts)
    assert int(exact[0][-1]) > 0 and not exact[2].any()
    for metric in ("hamming", "edit"):
        for k in (0, 1, 3):
            assert _same(_fetch(ctx, text, g, low, _kf(k, metric, None, "forward"), starts), exact), (metric, k)
    for metric in ("hamming", "edit"):                             # 4: the operations keep fixed symbols whole
        off, pos, words = _fetch(ctx, text, g, pam, _kf(2, metric, None, "both", "align"), starts)
        assert int(off[-1]) > 0
        q_of = np.repeat(np.arange(len(pam)), np.diff(off.astype(np.int64)))
        prev = None
        for i in range(len(pos)):
            key = (q_of[i], int(pos[i]), int(words[i]) >= MINUS)
            if key != prev:
                Q = model_strand.revcomp(pam[key[0]], True) if key[2] else pam[key[0]]
                fx, x, prev = model_fixed.marks(Q), 0, key
            code, n = int(words[i]) & 15, (int(words[i]) & (MINUS - 1)) >> 4
            for _ in range(n):
                if code in (1, 8):
                    assert not fx[x]
                if code == 2:
                    assert not fx[x] and not (x > 0 and fx[x - 1])
                else:
                    x += 1
    ctx.close()


def test_scale_against_the_c_statement():
    rng = np.random.default_rng(730)
    t = gen.dna(3_000_000)
    text = _u8(t)
    st = SuffixTable(text)
    sites = np.flatnonzero((t[21:-2] == ord("G")) & (t[22:-1] == ord("G")))      # 20 nt, then an intact NGG
    guides = []
    for a in rng.choice(sites, 200, replace=False):
        s = bytearray(t[a:a + 20].tobytes())
        for x in rng.choice(20, int(rng.integers(0, 3)), replace=False):
            s[int(x)] = int(b"ACGT"[int(rng.integers(0, 4))])
        guides.append(bytes(s) + b"ngg")
    sample = rng.choice(len(guides), 6, replace=False).tolist()
    for metric, k in (("hamming", 3), ("edit", 2)):
        off, pos, dist, minus = st.approximate_positions_batch(guides, k, metric=metric, iupac=True, fixed=True,
                                                               strands="both")
        assert (np.diff(off.astype(np.int64)) > 0).all()                    # each guide finds its own site
        for q in sample:
            a, b = int(off[q]), int(off[q + 1])
            for strand, Q in ((False, guides[q]), (True, model_strand.revcomp(guides[q], True))):
                _, wp, wd = fixed_check.fixed(text, None, [Q], k, metric)
                sel = minus[a:b] == strand
                assert np.array_equal(pos[a:b][sel], wp) and np.array_equal(dist[a:b][sel], wd), (metric, q, strand)


def test_argument_checks_and_protocol():
    ctx = _lib.Context(0)
    text = b"ACGTACGTNNacgtGAATTCGG"
    sa = SuffixTable(text).table()
    starts = np.array([0, 8, 8], dtype=np.uint32)
    docs = [text[:8], b"", text[8:]]
    g = DocumentSuffixTable(docs).table()
    for extra in (0, EDIT, BEST | (1 << 8), BOTH, BEST | EDIT | BOTH):
        with pytest.raises(_lib.B200SAError) as e:                             # bit 25 on the single-text entry
            _abi(ctx, text, sa, [b"ACg"], 1 | extra | IUPAC | FIXED, 0)
        msg = str(e.value)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_MAX_K" in msg and "FIXED" not in msg, hex(extra)
        with pytest.raises(_lib.B200SAError) as e:                             # without B200SA_APPROX_IUPAC
            _abi(ctx, text, g, [b"ACg"], 1 | extra | FIXED, 0, starts)
        msg = str(e.value)
        assert e.value.code == BAD_ARG and "B200SA_APPROX_FIXED" in msg and "B200SA_APPROX_IUPAC" in msg
        for bit in (19, 22, 23, 26, 30):                                       # an unknown bit with the flag
            with pytest.raises(_lib.B200SAError) as e:
                _abi(ctx, text, g, [b"ACg"], 1 | extra | IUPAC | FIXED | (1 << bit), 0, starts)
            msg = str(e.value)
            assert e.value.code == BAD_ARG and all(
                w in msg for w in ("B200SA_APPROX_MAX_K", "B200SA_APPROX_DOCUMENTS", "B200SA_APPROX_ALIGN")), bit
    qs = [b"ACGt", b"gaat", b"ACGTn", b"", b"N", b"CGg", b"cc"]
    for metric, best, strands, mode in MIXES[::2]:
        kf = _kf(1, metric, best, strands, mode)
        want = _want(docs, qs, 1, metric, best, strands, mode)
        total = int(want[0][-1])
        assert total > 1, (metric, best, strands, mode)
        for cap in (0, 1, total - 1):                                          # offsets and total only
            tot, off, pos, dist = _abi(ctx, text, g, qs, kf, cap, starts, buf=total + 5)
            assert tot == total and np.array_equal(off, want[0])
            assert (pos == MARK).all() and (dist == MARK).all(), cap
        tot, off, pos, dist = _abi(ctx, text, g, qs, kf, total, starts, buf=total + 5)   # nothing past total
        assert tot == total and np.array_equal(off, want[0])
        assert np.array_equal(pos[:total], want[1]) and np.array_equal(dist[:total], want[2])
        assert (pos[total:] == MARK).all() and (dist[total:] == MARK).all()
        tot, off, _, _ = _abi(ctx, text, g, [], kf, 0, starts)                 # nq = 0
        assert tot == 0 and off.tolist() == [0]
        tot, off, pos, _ = _abi(ctx, b"", [], [b"Ag", b"", b"g"], kf, 4, np.array([0], np.uint32))   # n = 0
        assert tot == 0 and off.tolist() == [0, 0, 0, 0] and (pos == MARK).all()
        tot, off, pos, _ = _abi(ctx, text, g, [b"", b""], kf, 4, starts)      # m = 0
        assert tot == 0 and off.tolist() == [0, 0, 0] and (pos == MARK).all()
    with pytest.raises(_lib.B200SAError) as e:                                 # the byte check names the offset
        _abi(ctx, text, g, [b"ACGT", b"ac-g"], 1 | IUPAC | FIXED, 0, starts)
    assert e.value.code == BAD_ARG and "offset 6" in str(e.value)
    ctx.close()
