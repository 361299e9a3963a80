"""Device primitives (through the b200sa_test_* hooks of the C-ABI library)
against numpy / the oracle.  All need an H100."""
import ctypes

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import _lib, gen
from tests import families

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _check(c, rc):
    assert rc == 0, (rc, _lib.lib().b200sa_last_error(c._h))


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 100000, 1 << 20, (1 << 22) + 12345])
@pytest.mark.parametrize("op", [0, 1])
def test_scan(ctx, n, op):
    rng = np.random.default_rng(n + op)
    a = rng.integers(0, 1000 if op == 0 else 1 << 30, n, dtype=np.uint32)
    out = np.empty(n, dtype=np.uint32)
    tot = ctypes.c_uint32(0)
    _check(ctx, _lib.lib().b200sa_test_scan(ctx._h, a.ctypes.data, n, op, out.ctypes.data, ctypes.byref(tot)))
    if op == 0:
        inc = np.cumsum(a.astype(np.uint64))
        want = np.concatenate([[0], inc[:-1]]).astype(np.uint32)
        assert tot.value == int(inc[-1]) & 0xFFFFFFFF
    else:
        inc = np.maximum.accumulate(a)
        want = np.concatenate([[0], inc[:-1]]).astype(np.uint32)
        assert tot.value == int(inc[-1])
    assert np.array_equal(out, want)


@pytest.mark.parametrize("n", [1, 2, 100, 2047, 2048, 2049, 70000, 1 << 20, 3_000_001])
@pytest.mark.parametrize("bits", [1, 8, 13, 32])
def test_sort_pairs32(ctx, n, bits):
    rng = np.random.default_rng(n * 31 + bits)
    keys = rng.integers(0, 1 << bits, n, dtype=np.uint64).astype(np.uint32)
    vals = np.arange(n, dtype=np.uint32)
    k, v = keys.copy(), vals.copy()
    _check(ctx, _lib.lib().b200sa_test_sort_pairs32(ctx._h, k.ctypes.data, v.ctypes.data, n, bits))
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[order])
    assert np.array_equal(v, vals[order])           # stability


@pytest.mark.parametrize("n", [1, 5, 2049, 100000, 1 << 20])
@pytest.mark.parametrize("bits", [9, 40, 62])
def test_sort_pairs64(ctx, n, bits):
    rng = np.random.default_rng(n * 17 + bits)
    keys = rng.integers(0, 1 << bits, n, dtype=np.uint64)
    if n > 10:
        keys[: n // 2] = keys[n // 2: n // 2 + n // 2]   # force ties
    vals = np.arange(n, dtype=np.uint32)
    k, v = keys.copy(), vals.copy()
    _check(ctx, _lib.lib().b200sa_test_sort_pairs64(ctx._h, k.ctypes.data, v.ctypes.data, n, bits))
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[order])
    assert np.array_equal(v, vals[order])


def _classify(ctx, t):
    n = len(t)
    nw = (n + 31) // 32
    st = np.zeros(nw, dtype=np.uint32)
    lm = np.zeros(nw, dtype=np.uint32)
    hist = np.zeros(768, dtype=np.uint32)
    pos = np.zeros(max(1, n // 2 + 1), dtype=np.uint32)
    m = ctypes.c_uint64(0)
    _check(ctx, _lib.lib().b200sa_test_classify_fused(ctx._h, t.ctypes.data, n, st.ctypes.data, lm.ctypes.data,
                                                      hist.ctypes.data, pos.ctypes.data, len(pos), ctypes.byref(m)))
    bits = lambda w: np.unpackbits(w.view(np.uint8), bitorder="little")[:n]
    return bits(st), bits(lm), hist, pos[: m.value][::-1]      # the fused kernel lists positions from the end


def _classify_cases():
    out = [(name, np.frombuffer(data, dtype=np.uint8)) for name, data in families.adversarial() if len(data) >= 1]
    out += [("kat:" + repr(c["text"])[:12], np.frombuffer(c["text"].encode(), dtype=np.uint8))
            for c in families.kat()["kat"] if len(c["text"]) >= 1]
    out += [("dna_1m", gen.dna(1_000_003)), ("bytes_300k", gen.rand_bytes(300_001)),
            ("a^100k", np.full(100_000, 97, dtype=np.uint8)),
            ("a^8192 b", np.concatenate([np.full(8192 * 3, 97, dtype=np.uint8), np.array([98], dtype=np.uint8)])),
            ("b a^8192..", np.concatenate([np.array([98], dtype=np.uint8), np.full(8192 * 3 + 5, 97, dtype=np.uint8)])),
            ("a^300k b a^300k c", np.concatenate([np.full(300_000, 97, dtype=np.uint8), np.array([98], dtype=np.uint8),
                                                  np.full(300_000, 97, dtype=np.uint8), np.array([99], dtype=np.uint8)])),
            ("z^70k a z^70k", np.concatenate([np.full(70_000, 122, dtype=np.uint8), np.array([97], dtype=np.uint8),
                                              np.full(70_000, 122, dtype=np.uint8)])),
            ("english_200k", gen.english(200_003))]
    return out


@pytest.mark.parametrize("name,t", _classify_cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_classify(ctx, name, t):
    t = np.ascontiguousarray(t)
    ty = oracle.types(t)                      # 0 S, 1 L, 2 Valley (reference semantics)
    sbit, lbit, hist, pos = _classify(ctx, t)
    assert np.array_equal(sbit, (ty != 1).astype(np.uint8))
    assert np.array_equal(lbit, (ty == 2).astype(np.uint8))
    assert np.array_equal(pos, np.flatnonzero(ty == 2).astype(np.uint32))
    want = np.zeros(768, dtype=np.uint32)
    np.add.at(want, t.astype(np.int64) + 256 * np.array([1, 0, 2])[ty], 1)
    assert np.array_equal(hist, want)


def _naive_u32_sa(R):
    R = list(R)
    return sorted(range(len(R)), key=lambda i: R[i:])


@pytest.mark.parametrize("case", ["unique", "const", "binary", "period", "random_small", "zipf", "big"])
def test_reduced_sa(ctx, case):
    rng = np.random.default_rng(7)
    if case == "unique":
        R = rng.permutation(5000).astype(np.uint32)
    elif case == "const":
        R = np.zeros(3000, dtype=np.uint32)
    elif case == "binary":
        R = rng.integers(0, 2, 4000, dtype=np.uint32)
    elif case == "period":
        R = np.tile(np.array([3, 1, 2, 1], dtype=np.uint32), 1000)
    elif case == "random_small":
        R = rng.integers(0, 7, 37, dtype=np.uint32)
    elif case == "zipf":
        R = np.minimum(rng.zipf(1.3, 6000), 5000).astype(np.uint32)
    else:
        R = rng.integers(0, 50, 300000, dtype=np.uint32)
    m = len(R)
    names = int(R.max()) + 1
    out = np.empty(m, dtype=np.uint32)
    rounds = ctypes.c_uint32(0)
    _check(ctx, _lib.lib().b200sa_test_reduced_sa(ctx._h, R.ctypes.data, m, names, out.ctypes.data, ctypes.byref(rounds)))
    if m <= 6000:
        assert out.tolist() == _naive_u32_sa(R)
    else:
        # u32 symbols < 256 here: compare with the byte oracle
        assert np.array_equal(out, oracle.sais(R.astype(np.uint8)))
