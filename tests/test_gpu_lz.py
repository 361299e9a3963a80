"""Longest previous factors and the LZ77 factorization (b200sa_lpf_dev, b200sa_lz77_dev, SuffixTable /
DocumentSuffixTable .longest_previous_factors, .lz77_factors, .lz77_count) against the numpy model of
tests/model_lz.py and, at scale, the serial C statement of tests/lz_check.c; the factors must decode back
to the text."""
import math
import threading

import numpy as np
import pytest
import torch

from suffix_b200 import DocumentSuffixTable, SuffixTable, _lib, gen
from tests import lz_check, model_docs, model_lz as mz
from tests.test_gpu_docs import _families, _u8

pytestmark = pytest.mark.gpu

BAD_ARG, TOO_LARGE = -1, -2
MARK = 0xA5A5A5A5
LIT = mz.LITERAL


def _dev(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return torch.from_numpy((a if len(a) else np.zeros(1, np.uint32)).view(np.int32).copy()).cuda()


def _marked(k):
    return torch.full((max(k, 1),), MARK - (1 << 32), dtype=torch.int32, device="cuda")


def _host(t):
    return t.cpu().numpy().view(np.uint32)


class _Abi:
    """The C-ABI on host arrays: the table and its LCP array go to the device once."""

    def __init__(self, ctx, g, lcp):
        self.ctx, self.n = ctx, len(g)
        self.g, self.lcp = _dev(g), _dev(lcp)
        self.stream = torch.cuda.current_stream().cuda_stream
        torch.cuda.synchronize()

    def lpf(self, with_src=True):
        lpf, src = _marked(self.n), _marked(self.n)
        torch.cuda.synchronize()
        self.ctx.lpf_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), lpf.data_ptr(),
                         src.data_ptr() if with_src else 0, self.stream)
        torch.cuda.synchronize()
        return _host(lpf)[:self.n], _host(src)[:self.n]

    def lz77(self, cap=None):
        """(z, start, length, source): buffers of max(cap, 1) entries pre-filled with MARK; cap = None counts
        first and fetches into buffers of exactly that size."""
        if cap is None:
            cap = self.ctx.lz77_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), stream=self.stream)
        out = [_marked(cap) for _ in range(3)]
        torch.cuda.synchronize()
        z = self.ctx.lz77_dev(self.n, self.g.data_ptr(), self.lcp.data_ptr(), *(o.data_ptr() if cap else 0 for o in out),
                              cap, self.stream)
        return (z,) + tuple(_host(o) for o in out)


def _check_abi(abi, g, lcp, want=None):
    """Both entry points against the model (or want = (lpf, src, start, length, source))."""
    if want is None:
        lpf, src = mz.lpf_src(g, lcp)
        start, length, source, rounds = mz.factors(g, lcp)
        want = (lpf, src, start, length, source)
    got_lpf, got_src = abi.lpf()
    assert np.array_equal(got_lpf, want[0]) and np.array_equal(got_src, want[1])
    assert np.array_equal(abi.lpf(with_src=False)[0], want[0])
    z, start, length, source = abi.lz77()
    assert z == len(want[2])
    assert np.array_equal(start, want[2]) and np.array_equal(length, want[3]) and np.array_equal(source, want[4])
    assert abi.ctx.stats()["doubling_rounds"] == (math.ceil(math.log2(z)) if z else 0)
    return want


def _check_class(st, text, want):
    lpf, src = st.longest_previous_factors()
    assert np.array_equal(lpf, want[0]) and np.array_equal(src, want[1])
    f = st.lz77_factors()
    assert all(np.array_equal(a, b) for a, b in zip(f, want[2:]))
    assert st.lz77_count() == len(want[2])
    if len(text):
        assert lz_check.decode(_u8(text), *f).tobytes() == _u8(text)


def test_abi_and_classes_equal_model_on_families():
    rng = np.random.default_rng(121)
    sets = _families(rng)
    assert len(sets) >= 300
    ctx = _lib.Context(0)
    for docs in sets:
        text, starts = model_docs.concat(docs)
        st = DocumentSuffixTable(docs)
        if not text:
            assert st.lz77_count() == 0 and [len(x) for x in st.lz77_factors()] == [0, 0, 0]
            assert [len(x) for x in st.longest_previous_factors()] == [0, 0]
            continue
        g, glcp = model_docs.brute(docs)
        want = _check_abi(_Abi(ctx, g, glcp), g, glcp)
        _check_class(st, text, want)
        nonempty = {int(starts[d]) for d in range(len(docs)) if len(docs[d])}
        assert nonempty <= set(want[2].tolist())                     # every non-empty document starts a factor
        if len(docs) == 1:                                           # one document is the single text
            _check_class(SuffixTable(text), text, want)
    ctx.close()


def test_definition_on_a_sample_of_the_families():
    rng = np.random.default_rng(122)
    for docs in [d for d in _families(rng) if 0 < sum(map(len, d)) <= 40][::3]:
        st = DocumentSuffixTable(docs)
        lpf, src = st.longest_previous_factors()
        assert np.array_equal(lpf, mz.brute_lpf(docs)), docs
        text = st.text()
        start, length, source = st.lz77_factors()
        s0, l0 = mz.serial_parse(lpf)
        assert np.array_equal(start, s0) and np.array_equal(length, l0)
        for s, l, q in zip(start.tolist(), length.tolist(), source.tolist()):
            assert (q == LIT and l == 1 and lpf[s] == 0) or (q < s and text[q:q + l] == text[s:s + l]), docs
        at = st.locate(start)                                        # positions map to documents
        assert np.all(at[:, 1] + length <= np.array([len(docs[d]) for d in at[:, 0]]))


@pytest.mark.parametrize("text", [b"aaaaaaaa", b"abababab", b"banana", b"mississippi", b"abaababaabaab"])
def test_known_answers(text):
    from tests.test_lz_model import KNOWN
    want_lpf, want_f = KNOWN[text]
    t = SuffixTable(text)
    assert t.longest_previous_factors()[0].tolist() == want_lpf
    assert [(int(s), int(l), None if q == LIT else int(q)) for s, l, q in zip(*t.lz77_factors())] == want_f
    assert t.lz77_count() == len(want_f)


def _texts(n):
    return {"dna": _u8(gen.dna(n)), "bytes": _u8(gen.rand_bytes(n)), "ab": (b"ab" * (n // 2 + 1))[:n],
            "english": _u8(gen.english(n))}


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769])
def test_level_edges(n):
    """n around the 32^k sizes where the block minima gain a level, against the model (small n) or the C
    statement."""
    ctx = _lib.Context(0)
    for name, text in _texts(n).items():
        t = SuffixTable(text)
        sa, lcp = t.table(), t.lcp_lens()
        want = None if n <= 1100 else lz_check.lz(sa, lcp)
        want = _check_abi(_Abi(ctx, sa, lcp), sa, lcp, want)
        _check_class(t, text, want)
    ctx.close()


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 6, 7, 8])
def test_z_at_powers_of_two(k):
    """z = 2^k - 1, 2^k, 2^k + 1 (where that many factors fit distinct bytes and one copy): the parse takes
    exactly ceil(log2 z) rounds."""
    ctx = _lib.Context(0)
    for z in (2 ** k - 1, 2 ** k, 2 ** k + 1):
        if z < 2 or z > 257:
            continue
        t = bytes(range(z - 1)) + bytes(range(z - 1))[:5] if z >= 3 else bytes(range(z))
        sa, lcp = ctx.build_lcp(np.frombuffer(t, dtype=np.uint8))
        _check_abi(_Abi(ctx, sa, lcp), sa, lcp)
        assert SuffixTable(t).lz77_count() == z
    ctx.close()


def _planted_docs(n, seed):
    """~1 kB documents of DNA, one in ten overwritten by a copy of an earlier one with a few substitutions."""
    rng = np.random.default_rng(seed)
    t = gen.dna(n)
    cuts = np.arange(0, n, 1000)[1:]
    docs = [t[a:b].copy() for a, b in zip(np.r_[0, cuts], np.r_[cuts, n])]
    for i in range(1, len(docs)):
        if rng.random() < 0.1:
            j = int(rng.integers(0, i))
            d = docs[j][:len(docs[i])].copy()
            d[rng.integers(0, len(d), 3)] = ord("T")
            docs[i][:len(d)] = d
    docs.insert(3, np.zeros(0, np.uint8))
    return [_u8(d) for d in docs]


@pytest.mark.parametrize("n", [1_000_000, 10_000_000])
def test_scale_against_the_serial_checker(n):
    ctx = _lib.Context(0)
    texts = {"dna": _u8(gen.dna(n)), "bytes": _u8(gen.rand_bytes(n)), "english": _u8(gen.english(n)),
             "AP009048_tiled": _u8(gen.tiled(gen.fixture("AP009048_100000.fasta"), n))}
    for name, text in texts.items():
        t = SuffixTable(text)
        sa, lcp = t.table(), t.lcp_lens()
        want = lz_check.lz(sa, lcp)
        _check_abi(_Abi(ctx, sa, lcp), sa, lcp, want)
        f = t.lz77_factors()
        assert all(np.array_equal(a, b) for a, b in zip(f, want[2:])), name
        assert lz_check.decode(text, *f).tobytes() == text, name
    docs = _planted_docs(n, 123)
    st = DocumentSuffixTable(docs)
    g, glcp, starts = st.table(), st.lcp_lens(), st.doc_starts()
    want = lz_check.lz(g, glcp)
    _check_abi(_Abi(ctx, g, glcp), g, glcp, want)
    f = st.lz77_factors()
    assert all(np.array_equal(a, b) for a, b in zip(f, want[2:]))
    assert lz_check.decode(st.text(), *f).tobytes() == st.text()
    nonempty = starts[np.array([len(d) > 0 for d in docs])]
    assert np.all(np.isin(nonempty, f[0]))
    at = st.locate(f[0])
    lens = np.array([len(d) for d in docs], dtype=np.int64)
    assert np.all(at[:, 1].astype(np.int64) + f[1] <= lens[at[:, 0]])   # no factor crosses a document end
    # the planted copies are long factors from earlier documents
    assert int((f[1] >= 200).sum()) > 0.05 * len(docs)
    ctx.close()


def test_cap_protocol_and_the_capacity_guess():
    ctx = _lib.Context(0)
    text = _u8(gen.dna(5000))
    sa, lcp = ctx.build_lcp(np.frombuffer(text, dtype=np.uint8))
    abi = _Abi(ctx, sa, lcp)
    _, _, start, length, source = want = lz_check.lz(sa, lcp)
    z = len(start)
    assert z > 10
    for cap in (0, 1, z - 1):                                  # too small: z and nothing else
        got = abi.lz77(cap)
        assert got[0] == z and all(np.all(a == MARK) for a in got[1:]), cap
    for cap in (z, z + 7):                                     # exact and larger: nothing past z
        got = abi.lz77(cap)
        assert got[0] == z
        assert all(np.array_equal(a[:z], b) and np.all(a[z:] == MARK) for a, b in zip(got[1:], want[2:])), cap
    t = SuffixTable(text)
    for guess in (0, 1, z - 1, z, 10 * z):                     # short guesses take the second call
        assert all(np.array_equal(a, b) for a, b in zip(t.lz77_factors(_cap_guess=guess), want[2:])), guess
    ctx.close()


def test_abi_errors_and_tiny_inputs():
    ctx = _lib.Context(0)
    d = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = d.data_ptr()
    for k in (1, 2, 3):                                        # (n, sa, lcp, lpf, src)
        args = [8, p, p, p, p]
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.lpf_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), k
    for k in (1, 2, 3, 4, 5):                                  # (n, sa, lcp, start, len, src, cap)
        args = [8, p, p, p, p, p, 4]
        args[k] = 0
        with pytest.raises(_lib.B200SAError) as ex:
            ctx.lz77_dev(*args)
        assert ex.value.code == BAD_ARG and "null" in str(ex.value), k
    assert _lib.lib().b200sa_lz77_dev(ctx._h, 8, p, p, None, None, None, 0, None, 0) == BAD_ARG   # total = NULL
    for call in (lambda: ctx.lpf_dev(1 << 33, p, p, p, p), lambda: ctx.lz77_dev(1 << 33, p, p, p, p, p, 4)):
        with pytest.raises(_lib.B200SAError) as ex:
            call()
        assert ex.value.code == TOO_LARGE
    # cap = 0 takes NULL arrays; n = 0 gives z = 0 without a launch; the phases have names of their own
    assert ctx.lz77_dev(0, 0, 0) == 0
    ctx.lpf_dev(0, 0, 0, 0)
    assert ctx.stats()["kernel_launches"] == 0
    abi = _Abi(ctx, [0], [0])                                  # n = 1: one literal, no parse round
    assert [x.tolist() if k else x for k, x in enumerate(abi.lz77())] == [1, [0], [1], [LIT]]
    assert ctx.stats()["doubling_rounds"] == 0
    assert [x.tolist() for x in abi.lpf()] == [[0], [LIT]]
    ctx.set_timing(True)
    abi.lpf()
    assert [x for x, _ in ctx.phase_times()] == ["lz_levels", "lz_lpf"]
    abi.lz77(0)
    assert [x for x, _ in ctx.phase_times()] == ["lz_levels", "lz_lpf", "lz_parse", "lz_count"]
    abi.lz77(1)
    assert [x for x, _ in ctx.phase_times()] == ["lz_levels", "lz_lpf", "lz_parse", "lz_count", "lz_emit"]
    ctx.close()
    for e in (SuffixTable(b""), DocumentSuffixTable([]), DocumentSuffixTable([b"", b""])):
        assert e.lz77_count() == 0 and [len(x) for x in e.lz77_factors()] == [0, 0, 0]
    one = SuffixTable(b"x")
    assert [x.tolist() for x in one.lz77_factors()] == [[0], [1], [LIT]]


def test_concurrent_factorizations_with_suffix_table_builds():
    docs = _planted_docs(2_000_000, 124)
    st = DocumentSuffixTable(docs)
    g, glcp = st.table(), st.lcp_lens()
    want = lz_check.lz(g, glcp)
    etext = _u8(gen.english(300_000))
    want_t = SuffixTable(etext).table()
    errors = []

    def run(fn):
        try:
            for _ in range(4):
                fn()
        except Exception as ex:
            errors.append(ex)

    def factorize():                                           # a context of its own per thread
        ctx = _lib.Context(0)
        abi = _Abi(ctx, g, glcp)
        z, start, length, source = abi.lz77()
        assert z == len(want[2]) and np.array_equal(start, want[2]) and np.array_equal(source, want[4])
        assert np.array_equal(abi.lpf()[0], want[0])
        ctx.close()

    def classes():                                             # the shared default context
        assert st.lz77_count() == len(want[2])

    def build():
        assert np.array_equal(SuffixTable(etext).table(), want_t)

    th = [threading.Thread(target=run, args=(f,)) for f in (factorize, factorize, classes, build)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
