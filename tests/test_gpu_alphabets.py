"""SA and LCP of every text packing, bit for bit against the oracle, at each alphabet size, LMS window
width and LCP path.

The library branches on the alphabet size sigma in three places:
* packing: 2 bits per character for sigma <= 4, 4 bits for sigma <= 16, bytes above that (and for every
  sigma under B200SA_NOPACK=1); past the end of the text the packed words hold zeros, which is also the
  code of the smallest symbol;
* the LMS windows: kc characters per window, as many as keep sigma^kc <= 2^32 (KC_TABLE);
* the LCP: a direct compare capped at CAP characters that falls back to the linear Phi/PLCP path when a
  pair reaches the cap; byte text longer than 32 MiB goes to the Phi path at once, and from 2^22
  characters on Phi is built by the partitioned scatter.

Every case is compared with oracle.sais (oracle.verify_sa above SAIS_MAX) and oracle.lcp_kasai, and
asserts the route it took: kc and the round-1 ties from the B200SA_TRACE line, direct_sort from the
stats, and lcp_direct / lcp_phi from the phase names, each predicted from the text and the oracle."""
import re

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import _lib
from tests.test_gpu_lms_sort import lms_positions

pytestmark = pytest.mark.gpu

CAP = 256                       # k_lcp_direct: a pair that reaches CAP characters sends the LCP to the Phi path
BYTE_DIRECT_MAX = 32 << 20      # byte text longer than this skips the direct compare
N_PHI = (1 << 22) + 777         # just above the size from which Phi is built by the partitioned scatter
SAIS_MAX = 5_000_000            # above this the SA is checked by oracle.verify_sa

# kc, the characters per LMS window (window_chars in b200sa.cu): 16 for 2-bit text, else as many as keep
# sigma^kc <= 2^32, at most 13 for 4-bit text and 8 for bytes.  Rows: (bits, lowest sigma, highest sigma, kc).
KC_TABLE = [(2, 1, 4, 16),
            (4, 5, 5, 13), (4, 6, 6, 12), (4, 7, 7, 11), (4, 8, 9, 10), (4, 10, 11, 9), (4, 12, 16, 8),
            (8, 1, 16, 8), (8, 17, 23, 7), (8, 24, 40, 6), (8, 41, 84, 5), (8, 85, 256, 4)]
# both ends of every row
SIGMAS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 15, 16, 17, 22, 23, 24, 40, 41, 84, 85, 215, 216, 255, 256]
NOPACK_SIGMAS = [1, 2, 3, 4, 16]
SHAPES = ["uniform", "skewed", "repeats"]
PATHS = ["build", "lcp", "robust"]     # build_lcp; stand-alone lcp (repacks the text); B200SA_NO_DIRECT=1

_KC_LINE = re.compile(r"direct LMS sort: kc=(\d+), round 1 leaves (\d+) of (\d+) tied")
_HAND = re.compile(r"direct LMS sort: hand over to the robust path: (\S+)")


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    c.set_timing(True)              # phase names
    yield c
    c.close()


@pytest.fixture(scope="module")
def cache():
    """(text, sa, lcp) by key, the oracle arrays computed once per text for all the path variants."""
    texts = {}

    def get(key, make):
        if key not in texts:
            t = make()
            sa = oracle.sais(t)
            texts[key] = (t, sa, oracle.lcp_kasai(t, sa))
        return texts[key]
    yield get
    texts.clear()


# ------------------------------------------------------------------ texts
def bits_of(sigma, nopack=False):
    return 8 if nopack or sigma > 16 else 2 if sigma <= 4 else 4


def window_chars(sigma, bits):
    kc, = [kc for b, lo, hi, kc in KC_TABLE if b == bits and lo <= sigma <= hi]
    return kc


def value_set(kind, sigma):
    """spread: evenly over 0..255 with 0x00 and 0xFF; contig: a run of byte values from 'A';
    sparse: 0x00, 0x07, 0x80, 0xFF and then seeded random values."""
    if kind == "spread":
        v = np.round(np.linspace(0, 255, sigma))
    elif kind == "contig":
        v = np.arange(sigma) + min(ord("A"), 256 - sigma)
    else:
        rest = np.setdiff1d(np.arange(256), [0x00, 0x07, 0x80, 0xFF])
        extra = np.random.default_rng(sigma).choice(rest, max(0, sigma - 4), replace=False)
        v = np.concatenate([[0x00, 0x07, 0x80, 0xFF][:sigma], extra])
    v = np.unique(v.astype(np.uint8))
    assert len(v) == sigma
    return v


def alpha_text(n, sigma, shape, seed, values=None):
    """n characters drawn from exactly sigma byte values (default: value_set("spread")).
    uniform: independent, equally likely;
    skewed: Zipf-like (p ~ rank^-1.2, the ranks in a random order of the values), so that windows tie
      and the refinement takes several rounds;
    repeats: the uniform text with planted copies of 300-5,000-character blocks of itself, each with 1-3
      substitutions, so that some adjacent suffixes share more than CAP characters."""
    values = value_set("spread", sigma) if values is None else values
    rng = np.random.default_rng(seed)
    if shape == "skewed":
        p = np.arange(1, sigma + 1) ** -1.2
        codes = rng.permutation(sigma)[rng.choice(sigma, n, p=p / p.sum())]
    else:
        codes = rng.integers(0, sigma, n)
    if shape == "repeats" and sigma > 1:
        for _ in range(min(400, max(8, n // 16384))):
            ln = int(rng.integers(300, 5001))
            src, dst = rng.integers(0, n - ln, 2)
            block = codes[src:src + ln].copy()
            at = rng.integers(0, ln, int(rng.integers(1, 4)))
            block[at] = (block[at] + rng.integers(1, sigma, len(at))) % sigma
            codes[dst:dst + ln] = block
    codes[rng.choice(n, sigma, replace=False)] = np.arange(sigma)      # every value occurs
    t = values[codes]
    assert len(np.unique(t)) == sigma
    return t


def ending_text(n, sigma, ending):
    """A uniform text of n characters, r = n % 16, that ends in
    run: a 12-character stem and 1 + r copies of the smallest symbol.  The stem also occurs earlier,
      followed by 41 + r of that symbol and then other characters: only the clamp to the characters
      left before the end tells the last suffixes from those earlier ones in a packed word;
    copy: the last CAP - 1 + r characters repeat an earlier stretch, so that the LCPs of the last
      suffixes run into the end of the text.  A pair whose LCP is its room (the characters left to the
      shorter suffix) is capped only from CAP + 1 on, and unlike a repeat inside the text it has no
      neighbour of LCP CAP - 1 with room to spare whose flag would send the LCP to the Phi path anyway."""
    values = value_set("spread", sigma)
    t = alpha_text(n, sigma, "uniform", seed=n * 1000 + sigma)
    r = n % 16
    if ending == "run":
        run = 1 + r
        t[100:112] = t[1000:1012]
        t[112:112 + run + 40] = values[0]
        t[n - run - 12:n - run] = t[1000:1012]
        t[n - run:] = values[0]
    else:
        c = CAP - 1 + r
        t[n - c:] = t[500:500 + c]
    assert len(np.unique(t)) == sigma
    return t


# ------------------------------------------------------------------ routes
def round1(t, kc):
    """(m, tied): the LMS suffixes, and those that round 1 of the direct sort leaves tied -- whose first
    kc characters lie inside the text and equal another such suffix's (a window that runs past the end
    is a group of its own)."""
    p = lms_positions(t)
    q = p[p + kc <= len(t)]
    vals = np.unique(t)
    codes = np.searchsorted(vals, t).astype(np.uint64)
    key = np.zeros(len(q), np.uint64)
    for i in range(kc):
        key = key * np.uint64(len(vals)) + codes[q + i]
    _, cnt = np.unique(key, return_counts=True)
    return len(p), int(cnt[cnt > 1].sum())


def lcp_route(sa, lcp, bits, env):
    """The LCP phases a call must take: the direct compare unless the text is bytes longer than
    BYTE_DIRECT_MAX or B200SA_LCP_LINEAR is set, and the Phi path when it is skipped or some pair
    reaches CAP with characters to spare (h == cap && room > cap in k_lcp_direct)."""
    n = len(sa)
    if "B200SA_LCP_LINEAR" in env or (bits == 8 and n > BYTE_DIRECT_MAX):
        return ["lcp_phi"]
    room = n - np.maximum(sa[1:], sa[:-1])
    capped = bool(np.any((lcp[1:] >= CAP) & (room > CAP)))
    return ["lcp_direct", "lcp_phi"] if capped else ["lcp_direct"]


def call(ctx, capfd, env, fn, *args):
    """fn(*args) with B200SA_TRACE=1 and env -> (result, trace, LCP phase names, stats)."""
    capfd.readouterr()
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200SA_TRACE", "1")
        for k, v in env.items():
            mp.setenv(k, v)
        out = fn(*args)
    err = capfd.readouterr().err
    phases = [name for name, _ in ctx.phase_times() if name in ("lcp_direct", "lcp_phi")]
    return out, err, phases, ctx.stats()


def same(got, want, what, sa, t):
    """Bit-exact, or the first differing rank with its two suffixes."""
    if np.array_equal(got, want):
        return
    r = int(np.flatnonzero(got != want)[0])
    a, b = (int(sa[r - 1]) if r else -1), int(sa[r])
    raise AssertionError("%s differs first at rank %d of %d: got %d, want %d; suffixes %d %r and %d %r"
                         % (what, r, len(want), got[r], want[r], a, bytes(t[a:a + 40]) if r else b"",
                            b, bytes(t[b:b + 40])))


def check(ctx, capfd, t, sa_w, lcp_w, bits, path, env=None, uniform=False):
    """One path on text t against the oracle arrays, with its route.  -> stats"""
    env = dict(env or {}) | ({"B200SA_NO_DIRECT": "1"} if path == "robust" else {})
    if path == "lcp":
        lcp, err, phases, st = call(ctx, capfd, env, ctx.lcp, t, sa_w)
    else:
        (sa, lcp), err, phases, st = call(ctx, capfd, env, ctx.build_lcp, t)
        same(sa, sa_w, "SA", sa_w, t)
    same(lcp, lcp_w, "LCP", sa_w, t)
    assert phases == lcp_route(sa_w, lcp_w, bits, env), (phases, err[-2000:])
    if path == "lcp":
        return st
    kc = window_chars(len(np.unique(t)), bits)
    m, tied = round1(t, kc)
    assert st["m"] == m
    line = _KC_LINE.findall(err)
    if path == "robust" or m == 0:
        assert not line and st["direct_sort"] == 0
        return st
    assert [tuple(map(int, x)) for x in line] == [(kc, tied, m)], err[-2000:]
    if uniform:         # random text settles in a few rounds unless round 1 ties (almost) everything
        handed = m > 64 and tied * 1000 > m * 999
        assert _HAND.findall(err) == (["round1-tied"] if handed else []), err[-2000:]
        assert st["direct_sort"] == (0 if handed else 1)
    return st


# ------------------------------------------------------------------ the alphabet sweep
def sweep_text(cache, sigma, shape, kind="spread"):
    n = 300_000 + 7 * sigma
    seed = 100 * sigma + SHAPES.index(shape)
    return cache(("sweep", sigma, shape, kind),
                 lambda: alpha_text(n, sigma, shape, seed, value_set(kind, sigma)))


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("sigma,nopack", [(s, False) for s in SIGMAS] + [(s, True) for s in NOPACK_SIGMAS],
                         ids=lambda x: ("nopack" if x else "packed") if isinstance(x, bool) else str(x))
def test_alphabet_sweep(ctx, capfd, cache, sigma, nopack, shape, path):
    t, sa, lcp = sweep_text(cache, sigma, shape)
    if shape == "repeats" or sigma == 1:
        assert lcp_route(sa, lcp, 8, {}) == ["lcp_direct", "lcp_phi"]       # the text does reach the cap
    env = {"B200SA_NOPACK": "1"} if nopack else {}
    check(ctx, capfd, t, sa, lcp, bits_of(sigma, nopack), path, env, uniform=shape == "uniform")


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("kind", ["contig", "sparse"])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_value_sets(ctx, capfd, cache, sigma, kind, path):
    """The byte -> code tables of the build and of the stand-alone LCP (which repacks) on byte sets
    other than the evenly spread one."""
    t, sa, lcp = sweep_text(cache, sigma, "uniform", kind)
    check(ctx, capfd, t, sa, lcp, bits_of(sigma), path, uniform=True)


# ------------------------------------------------------------------ text ends
ENDS = [("2bit", 4, False, 16), ("4bit", 6, False, 8), ("4bit", 16, False, 8), ("8bit", 41, False, 4),
        ("8bit", 256, False, 4), ("nopack", 4, True, 4)]          # (packing, sigma, nopack, characters per word)


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("ending", ["run", "copy"])
@pytest.mark.parametrize("packing,sigma,nopack,r",
                         [(p, s, nop, r) for p, s, nop, cpw in ENDS for r in range(cpw)],
                         ids=lambda x: str(x))
def test_text_end(ctx, capfd, cache, packing, sigma, nopack, r, ending, path):
    """Every length modulo the characters per packed word, ending in a run of the smallest symbol (the
    value of the padding) or in a copy of an earlier stretch."""
    n = 4096 + r
    t, sa, lcp = cache(("end", n, sigma, ending), lambda: ending_text(n, sigma, ending))
    env = {"B200SA_NOPACK": "1"} if nopack else {}
    check(ctx, capfd, t, sa, lcp, bits_of(sigma, nopack), path, env)


# ------------------------------------------------------------------ LCP thresholds
@pytest.mark.parametrize("sigma,nopack", [(4, False), (16, False), (41, False), (4, True), (16, True)],
                         ids=["2bit", "4bit", "8bit", "nopack4", "nopack16"])
def test_lcp_thresholds(ctx, capfd, cache, sigma, nopack):
    """A repeats text just above 2^22 characters with more than 2^20 LMS suffixes: the direct compare
    meets capped pairs and hands over to Phi built by the partitioned scatter; B200SA_LCP_LINEAR=1 takes
    that path at once, with B200SA_PHI_DIRECT=1 the plain Phi scatter."""
    t, sa, lcp = cache(("phi", sigma), lambda: alpha_text(N_PHI, sigma, "repeats", seed=sigma))
    assert lcp_route(sa, lcp, 8, {}) == ["lcp_direct", "lcp_phi"]
    bits = bits_of(sigma, nopack)
    base = {"B200SA_NOPACK": "1"} if nopack else {}
    variants = [{}, {"B200SA_LCP_LINEAR": "1"}, {"B200SA_LCP_LINEAR": "1", "B200SA_PHI_DIRECT": "1"}]
    for v in variants:
        st = check(ctx, capfd, t, sa, lcp, bits, "build", base | v)
        assert st["m"] >= 1 << 20
        check(ctx, capfd, t, sa, lcp, bits, "lcp", base | v)


@pytest.mark.parametrize("n,shape,route", [(BYTE_DIRECT_MAX, "uniform", ["lcp_direct"]),
                                           (BYTE_DIRECT_MAX + 1, "repeats", ["lcp_phi"])],
                         ids=["32MiB", "32MiB+1"])
def test_byte_text_at_32mib(ctx, capfd, n, shape, route):
    """Byte text up to 32 MiB takes the direct compare; one character more goes to the Phi path without
    trying it (the repeats there run the long matches of the PLCP kernels on byte text)."""
    t = alpha_text(n, 256, shape, seed=n)
    (sa, lcp), err, phases, _ = call(ctx, capfd, {}, ctx.build_lcp, t)
    assert oracle.verify_sa(t, sa) == 0
    want = oracle.lcp_kasai(t, sa)
    same(lcp, want, "LCP", sa, t)
    assert phases == route == lcp_route(sa, want, 8, {})


# ------------------------------------------------------------------ device entry points
@pytest.mark.parametrize("sigma,nopack", [(4, False), (16, False), (256, False), (4, True)],
                         ids=["2bit", "4bit", "8bit", "nopack"])
def test_device_entries_unaligned(ctx, cache, sigma, nopack):
    """build_lcp_dev and the stand-alone lcp_dev on a text pointer one byte past an aligned allocation
    give what the host calls give."""
    import torch
    t, sa_w, lcp_w = sweep_text(cache, sigma, "repeats")
    n = len(t)
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    with pytest.MonkeyPatch.context() as mp:
        if nopack:
            mp.setenv("B200SA_NOPACK", "1")
        sa, lcp = ctx.build_lcp(t)
        lcp2 = ctx.lcp(t, sa_w)
        d_t = torch.from_numpy(np.concatenate([[0], t]).astype(np.uint8)).to(dev)[1:]
        assert d_t.data_ptr() % 16 != 0
        d_sa = torch.zeros(n, dtype=torch.int32, device=dev)
        d_lcp = torch.zeros(n, dtype=torch.int32, device=dev)
        ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), stream)
        torch.cuda.synchronize()
        same(d_sa.cpu().numpy().view(np.uint32), sa, "SA (build_lcp_dev)", sa_w, t)
        same(d_lcp.cpu().numpy().view(np.uint32), lcp, "LCP (build_lcp_dev)", sa_w, t)
        d_lcp.zero_()
        ctx.lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), stream)
        torch.cuda.synchronize()
        same(d_lcp.cpu().numpy().view(np.uint32), lcp2, "LCP (lcp_dev)", sa_w, t)
    same(sa, sa_w, "SA", sa_w, t)
    same(lcp, lcp_w, "LCP", sa_w, t)
    same(lcp2, lcp_w, "LCP (lcp)", sa_w, t)
