"""The LMS-suffix sort of 2-bit text: two one-sweep passes on the top 16 key bits, then
k_lms_bucket_sort (each top-16 bucket sorted by the low 16 bits in shared memory, round-1 ties and
group ids found in the same kernel).  SA and LCP are checked against the oracle and against the
four-pass sort (B200SA_LMS_SORT4=1), at the sizes where the kernel's 4096-slot windows and the
4096-member bucket limit matter."""
import itertools

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import _lib, gen

pytestmark = pytest.mark.gpu

BS_T = 4096            # slots per window of k_lms_bucket_sort
BS_CAP = 4096          # longest bucket it sorts; longer ones go back to the four-pass sort
PREFIX = b"ACGTACGT"   # one top-16 bucket: 8 characters, the first an S-type A after a T


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def lms_positions(t):
    """LMS positions of a text (the last character is L-type: a proper prefix sorts first)."""
    n = len(t)
    c = t.astype(np.int16)
    d = np.zeros(n, np.int8)
    d[:-1] = np.sign(c[1:] - c[:-1]).astype(np.int8)
    d[-1] = -1
    idx = np.where(d != 0, np.arange(n), n)
    nxt = np.minimum.accumulate(idx[::-1])[::-1]
    s = d[nxt] == 1
    lms = np.zeros(n, bool)
    lms[1:] = s[1:] & ~s[:-1]
    return np.nonzero(lms)[0]


def top16(t, p):
    """Top 16 key bits of the LMS suffixes at p: their first 8 characters as 2-bit codes, zero past the end."""
    alpha = np.unique(t)
    code = np.zeros(256, np.uint32)
    code[alpha] = np.arange(len(alpha))
    cc = np.concatenate([code[t], np.zeros(8, np.uint32)])
    key = np.zeros(len(p), np.uint32)
    for j in range(8):
        key = (key << 2) | cc[p + j]
    return key


def check(ctx, monkeypatch, t, old_too=True):
    sa, lcp = ctx.build_lcp(t)
    want = oracle.sais(t)
    assert np.array_equal(sa, want)
    assert np.array_equal(lcp, oracle.lcp_kasai(t, want))
    if old_too:
        monkeypatch.setenv("B200SA_LMS_SORT4", "1")
        sa4, lcp4 = ctx.build_lcp(t)
        monkeypatch.delenv("B200SA_LMS_SORT4")
        assert np.array_equal(sa4, sa) and np.array_equal(lcp4, lcp)


def test_every_text_up_to_8(ctx, monkeypatch):
    """Every text over {A,C,G,T} up to n = 8: all windows truncated, the span is the whole list."""
    for n in range(1, 9):
        for tup in itertools.product(b"ACGT", repeat=n):
            t = np.frombuffer(bytes(tup), np.uint8)
            sa, lcp = ctx.build_lcp(t)
            want = oracle.sais(t)
            assert np.array_equal(sa, want), bytes(tup)
            assert np.array_equal(lcp, oracle.lcp_kasai(t, want)), bytes(tup)


def test_random_short(ctx, monkeypatch):
    rng = np.random.default_rng(11)
    for n in range(9, 65):
        for _ in range(20):
            t = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)]
            check(ctx, monkeypatch, t, old_too=(n % 8 == 0))


def _text_with_m(target):
    """A prefix of G_dna whose LMS count is exactly `target`."""
    base = gen.dna(int(target * 3.6) + 1000, seed=gen.SEED_DNA + target)
    p = lms_positions(base)
    # a prefix that ends two characters after the target-th LMS position keeps exactly `target` of them
    # (the last character of a prefix is L-type, the character before it cannot become LMS)
    for end in range(int(p[target - 1]) + 2, int(p[target]) + 1):
        t = base[:end]
        if len(lms_positions(t)) == target:
            return t
    raise AssertionError("no prefix with m = %d" % target)


@pytest.mark.parametrize("m", [BS_T - 1, BS_T, BS_T + 1, 2 * BS_T - 1, 2 * BS_T, 2 * BS_T + 1])
def test_window_edges(ctx, monkeypatch, m):
    t = _text_with_m(m)
    check(ctx, monkeypatch, t)
    assert ctx.stats()["m"] == m


@pytest.mark.parametrize("n", [1_000_000, 5_000_000])
def test_dna(ctx, monkeypatch, n):
    check(ctx, monkeypatch, gen.dna(n))
    assert ctx.stats()["direct_sort"] == 1


def _bucket_text(members, seed, lead):
    """Random DNA with copies of 'T' + PREFIX so that the PREFIX bucket holds exactly `members` LMS
    suffixes (the background adds a few: counted, and the copies adjusted).  `lead` random characters
    before the copies move the bucket's slot range."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    head = acgt[rng.integers(0, 4, lead)]
    fill = acgt[rng.integers(0, 4, (members + 64, 7))]
    fill[:, 0] = ord("C")           # no copy of PREFIX runs on into the filler
    tail = acgt[rng.integers(0, 4, 20000)]
    ins = np.frombuffer(b"T" + PREFIX, np.uint8)
    key = top16(np.frombuffer(PREFIX, np.uint8), np.array([0]))[0]
    k = members
    for _ in range(12):
        body = np.concatenate([np.concatenate([ins, f]) for f in fill[:k]]) if k > 0 else np.zeros(0, np.uint8)
        t = np.concatenate([head, body, tail])
        p = lms_positions(t)
        keys = top16(t, p)
        have = int((keys == key).sum())
        if have == members:
            start = int((keys < key).sum())         # first slot of the bucket after the top-16 passes
            return t, start
        k += members - have
    raise AssertionError("could not hit %d members" % members)


@pytest.mark.parametrize("members", [BS_CAP - 1, BS_CAP, BS_CAP + 1])
def test_bucket_cap(ctx, monkeypatch, capfd, members):
    t, start = _bucket_text(members, seed=members, lead=30000)
    monkeypatch.setenv("B200SA_TRACE", "1")
    check(ctx, monkeypatch, t)
    monkeypatch.delenv("B200SA_TRACE")
    err = capfd.readouterr().err
    fell_back = "four-pass sort" in err
    assert fell_back == (members > BS_CAP), err[-2000:]
    assert "(bucket sort)" in err or members > BS_CAP


def test_bucket_straddles_window(ctx, monkeypatch, capfd):
    """A bucket of CAP members that starts well inside one 4096-slot window and ends in the next."""
    for lead in range(2000, 40000, 1500):
        t, start = _bucket_text(BS_CAP, seed=lead, lead=lead)
        if start % BS_T > BS_T // 4:
            break
    assert start % BS_T > BS_T // 4 and (start + BS_CAP) // BS_T == start // BS_T + 1
    monkeypatch.setenv("B200SA_TRACE", "1")
    check(ctx, monkeypatch, t)
    monkeypatch.delenv("B200SA_TRACE")
    assert "four-pass sort" not in capfd.readouterr().err
