"""The one-sweep radix sort at the inputs that stress its look-back and ranking, under every tile width the
width rule can pick (no switch, B200SA_SORT_NARROW=1, B200SA_SORT_ITEMS=8 and a wide B200SA_SORT_ITEMS), against
numpy's stable argsort bit for bit.  Every key equal gives the longest look-back chains (one digit per pass,
so every tile adds to the same counter) and full-warp peer groups; digits that repeat in runs of 5,000 keys
cross every tile boundary (tiles of 2,048, 4,096 and 8,192 keys)."""
import numpy as np
import pytest

from suffix_b200 import _lib

pytestmark = pytest.mark.gpu

N = (1 << 21) + 777              # wide tiles by default; the last tile is partial at every width
SWITCHES = [{}, {"B200SA_SORT_NARROW": "1"}, {"B200SA_SORT_ITEMS": "8"}, {"B200SA_SORT_ITEMS": "32"}]


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _keys(kind, width):
    dt = np.uint32 if width == 32 else np.uint64
    if kind == "equal":
        return np.full(N, 0x5A5A5A5A5A5A5A5A & ((1 << width) - 1), dtype=dt)
    # one random key per run of 5,000: every pass sees a new digit every 5,000 keys
    per_run = np.random.default_rng(width).integers(0, 1 << width, N // 5000 + 1, dtype=np.uint64)
    return per_run[np.arange(N) // 5000].astype(dt)


@pytest.mark.parametrize("env", SWITCHES, ids=["default", "narrow", "items8", "wide"])
@pytest.mark.parametrize("width", [32, 64])
@pytest.mark.parametrize("kind", ["equal", "runs"])
def test_onesweep_stable(ctx, monkeypatch, kind, width, env):
    monkeypatch.delenv("B200SA_SORT_NARROW", raising=False)
    monkeypatch.delenv("B200SA_SORT_ITEMS", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    keys = _keys(kind, width)
    vals = np.arange(N, dtype=np.uint32)
    k, v = keys.copy(), vals.copy()
    hook = _lib.lib().b200sa_test_sort_pairs32 if width == 32 else _lib.lib().b200sa_test_sort_pairs64
    rc = hook(ctx._h, k.ctypes.data, v.ctypes.data, N, width)
    assert rc == 0, (rc, _lib.lib().b200sa_last_error(ctx._h))
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[order])
    assert np.array_equal(v, vals[order])
