"""The numpy prefix-doubling suffix array of uint32 strings (tests/model_u32_sa.py), pinned against
the brute-force sort and the byte oracle before test_gpu_refine.py uses it at m ~ 2M."""
import itertools

import numpy as np
import pytest

from oracle import oracle
from tests.model_u32_sa import u32_sa
from tests.test_gpu_primitives import _naive_u32_sa


def _cases():
    rng = np.random.default_rng(5)
    out = [np.zeros(0, np.uint32), np.array([7], np.uint32), np.zeros(300, np.uint32),
           np.full(257, 0xFFFFFFFF, np.uint32),                                       # the largest symbol
           np.tile(np.array([3, 1, 2, 1], np.uint32), 100), np.tile(np.array([0, 1], np.uint32), 129),
           np.concatenate([rng.integers(0, 9, 200), np.full(300, 4), rng.integers(0, 9, 50)]).astype(np.uint32),
           np.concatenate([np.full(100, 2), np.full(100, 1), np.full(100, 2)]).astype(np.uint32),
           rng.permutation(1000).astype(np.uint32)]
    out += [rng.integers(0, k, int(rng.integers(1, 600)), dtype=np.uint32) for k in (2, 3, 50, 1 << 20, 1 << 32)
            for _ in range(8)]
    return out


@pytest.mark.parametrize("R", _cases(), ids=lambda R: "m%d" % len(R))
def test_against_brute_force(R):
    assert u32_sa(R).tolist() == _naive_u32_sa(R)


def test_every_string_over_three_symbols_up_to_8():
    for m in range(1, 9):
        for tup in itertools.product((0, 1, 2), repeat=m):
            assert u32_sa(np.array(tup, np.uint32)).tolist() == _naive_u32_sa(tup), tup


@pytest.mark.parametrize("kind", ["random", "dna", "runs", "periodic"])
def test_against_byte_oracle(kind):
    rng = np.random.default_rng(9)
    if kind == "random":
        t = rng.integers(0, 256, 200_000, dtype=np.uint8)
    elif kind == "dna":
        t = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 200_000)]
    elif kind == "runs":
        t = np.repeat(rng.integers(0, 3, 3000).astype(np.uint8), rng.integers(1, 60, 3000))
    else:
        t = np.tile(np.frombuffer(b"abcab", np.uint8), 20_000)
    assert np.array_equal(u32_sa(t.astype(np.uint32)), oracle.sais(t))
