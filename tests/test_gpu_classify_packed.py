"""Classification of 2-bit text from its packed words (k_classify_packed): type / LMS bitmaps, the
(byte, class) histogram, the LMS positions in descending order with their 16-character window keys and
the digit counts of key bits 16-31, against oracle.types and numpy; then SA + LCP of the same texts
against the oracle.  The packing is coded by the alphabet of the first 1 MiB; texts with bytes that first
occur later take the second packing (or, with a fifth byte, the byte classifier)."""
import ctypes
import itertools

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import _lib, gen

pytestmark = pytest.mark.gpu

TILE = 32768                      # characters per tile of the packed classifier


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _hook():
    L = _lib.lib()
    fn = L.b200sa_test_classify_packed
    vp, u64 = ctypes.c_void_p, ctypes.c_uint64
    fn.argtypes = [vp, vp, u64, vp, vp, vp, vp, vp, vp, u64, ctypes.POINTER(u64)]
    fn.restype = ctypes.c_int
    return fn


def _classify_packed(ctx, t):
    n = len(t)
    nw = (n + 31) // 32
    st = np.zeros(nw, np.uint32)
    lm = np.zeros(nw, np.uint32)
    hist = np.zeros(768, np.uint32)
    cap = n // 2 + 1
    pos = np.zeros(cap, np.uint32)
    keys = np.zeros(cap, np.uint32)
    dig = np.zeros(512, np.uint32)
    m = ctypes.c_uint64(0)
    rc = _hook()(ctx._h, t.ctypes.data, n, st.ctypes.data, lm.ctypes.data, hist.ctypes.data, pos.ctypes.data,
                 keys.ctypes.data, dig.ctypes.data, cap, ctypes.byref(m))
    assert rc == 0, _lib.lib().b200sa_last_error(ctx._h)
    bits = lambda w: np.unpackbits(w.view(np.uint8), bitorder="little")[:n]
    return bits(st), bits(lm), hist, pos[: m.value], keys[: m.value], dig


def _window_keys(t, pos):
    """lms_window<2>: the 16 dense codes from each position, first one most significant, zeros past n."""
    codes = np.searchsorted(np.unique(t), t).astype(np.uint64)
    padded = np.concatenate([codes, np.zeros(16, np.uint64)])
    key = np.zeros(len(pos), np.uint64)
    for i in range(16):
        key |= padded[pos.astype(np.int64) + i] << np.uint64(30 - 2 * i)
    return key.astype(np.uint32)


def _check_classify(ctx, t):
    t = np.ascontiguousarray(t, dtype=np.uint8)
    ty = oracle.types(t)                      # 0 S, 1 L, 2 Valley (reference semantics)
    sbit, lbit, hist, pos, keys, dig = _classify_packed(ctx, t)
    assert np.array_equal(sbit, (ty != 1).astype(np.uint8))
    assert np.array_equal(lbit, (ty == 2).astype(np.uint8))
    want_pos = np.flatnonzero(ty == 2)[::-1].astype(np.uint32)
    assert np.array_equal(pos, want_pos)
    want_hist = np.zeros(768, np.uint32)
    np.add.at(want_hist, t.astype(np.int64) + 256 * np.array([1, 0, 2])[ty], 1)
    assert np.array_equal(hist, want_hist)
    want_keys = _window_keys(t, want_pos)
    assert np.array_equal(keys, want_keys)
    want_dig = np.concatenate([np.bincount((want_keys >> 16) & 0xff, minlength=256),
                               np.bincount(want_keys >> 24, minlength=256)]).astype(np.uint32)
    assert np.array_equal(dig, want_dig)


def _u8(s):
    return np.frombuffer(s, np.uint8)


def _cases():
    rng = np.random.default_rng(11)
    out = []
    for sigma, alpha in ((1, b"G"), (2, b"AT"), (3, b"ACT"), (4, b"ACGT")):
        for n in (2, 3, 1000, 70_001):
            out.append(("sigma%d_n%d" % (sigma, n), _u8(alpha)[rng.integers(0, sigma, n)]))
    for n in (15, 16, 17, 31, 32, 33, 63, 64, 65, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1,
              3 * TILE - 1, 3 * TILE + 1):
        out.append(("n%d" % n, gen.dna(n, seed=n)))
    # LMS positions within 16 characters of the end
    for tail in (b"TATATATATATATATT", b"CAC", b"GACAGT", b"TACT"):
        out.append(("tail_" + tail.decode(), np.concatenate([gen.dna(TILE - 5), _u8(tail)])))
    out.append(("a^100k", np.full(100_000, ord("A"), np.uint8)))
    out.append(("a^300k c a^300k g", np.concatenate([np.full(300_000, ord("A"), np.uint8), _u8(b"C"),
                                                     np.full(300_000, ord("A"), np.uint8), _u8(b"G")])))
    out.append(("c a^200k", np.concatenate([_u8(b"C"), np.full(200_000, ord("A"), np.uint8)])))
    # bytes that first occur after the first 1 MiB: the alphabet of a sample no longer codes the text
    ac = _u8(b"AC")[rng.integers(0, 2, 1_200_000)]
    ac[-100_000:] = _u8(b"ACGT")[rng.integers(0, 4, 100_000)]
    out.append(("late_GT_1.2m", ac))
    late_c = np.full(1_100_000, ord("A"), np.uint8)
    late_c[::7] = ord("T")
    late_c[-3] = ord("C")
    out.append(("late_C_1.1m", late_c))
    out.append(("dna_1m", gen.dna(1_000_000)))
    out.append(("dna_5m", gen.dna(5_000_000)))
    return out


CASES = _cases()


@pytest.mark.parametrize("name,t", CASES, ids=[c[0] for c in CASES])
def test_classify_packed(ctx, name, t):
    _check_classify(ctx, t)


def test_classify_packed_every_short_dna(ctx):
    """Every text over {A,C,G,T} of length 2 to 8."""
    for n in range(2, 9):
        for tup in itertools.product(b"ACGT", repeat=n):
            _check_classify(ctx, np.array(tup, np.uint8))


# a fifth byte after the first 1 MiB: the byte classifier takes the text
SA_CASES = CASES + [("late_N_1.2m", np.concatenate([gen.dna(1_200_000), _u8(b"N"), gen.dna(1000, seed=3)]))]


@pytest.mark.parametrize("name,t", SA_CASES, ids=[c[0] for c in SA_CASES])
def test_sa_lcp(ctx, name, t):
    t = np.ascontiguousarray(t)
    sa, lcp = ctx.build_lcp(t)
    want = oracle.sais(t)
    assert np.array_equal(sa, want)
    assert np.array_equal(lcp, oracle.lcp_kasai(t, want))


def test_sa_lcp_every_short_dna(ctx):
    """Every text over {A,C,G,T} of length 2 to 6."""
    for n in range(2, 7):
        for tup in itertools.product(b"ACGT", repeat=n):
            t = np.array(tup, np.uint8)
            sa, lcp = ctx.build_lcp(t)
            want = oracle.sais(t)
            assert np.array_equal(sa, want), t.tobytes()
            assert np.array_equal(lcp, oracle.lcp_kasai(t, want)), t.tobytes()


@pytest.mark.parametrize("text,path", [(b"ACGTACGGTCA" * 50, "packed 2-bit words"),
                                       (b"ACGTNACGGTCA" * 50, "bytes"),
                                       (b"AC" * 600_000 + b"GT", "packed 2-bit words"),
                                       (b"ACGT" * 300_000 + b"N", "bytes")],
                         ids=["sigma4", "sigma5", "sigma4_late", "sigma5_late"])
def test_trace_names_the_classifier(ctx, text, path, monkeypatch, capfd):
    monkeypatch.setenv("B200SA_TRACE", "1")
    t = _u8(text).copy()
    assert np.array_equal(ctx.build(t), oracle.sais(t))
    assert "[b200sa] classify: sigma=%d, %s" % (len(set(text)), path) in capfd.readouterr().err


def test_classify_packed_rejects_a_larger_alphabet(ctx):
    t = _u8(b"ACGTN" * 20).copy()
    n = len(t)
    rc = _hook()(ctx._h, t.ctypes.data, n, None, None, None, None, None, None, 0, None)
    assert rc != 0
    assert b"at most 4 distinct bytes" in _lib.lib().b200sa_last_error(ctx._h)
