"""The branches of the two refinement loops that order the LMS suffixes, each reached by an input
built for it and proved taken by its B200SA_TRACE line:

* the direct path's rounds >= 2 (lms_direct_sort_t): the local counting sort inside a group,
  its overflow on a group of more than GL_LIMIT steps (radix sort in the same round), the probe
  that prefers the radix sort when >= 2^20 suffixes are tied and large groups are common, and
  the three hand-overs to the robust path (round1-tied, no-convergence, round-limit);
* the robust path (reduced_sa / doubling_rounds): 32- and 64-bit round-0 keys, the k-gram or
  plain-pair first refinement, the probe, and a local-sort overflow that switches to radix
  sorting for good.

Every full build is compared with oracle.sais and oracle.lcp_kasai bit for bit; the reduced
string sort is compared with tests/model_u32_sa.py."""
import ctypes
import re

import numpy as np
import pytest

from oracle import oracle
from suffix_b200 import _lib, gen
from tests.model_u32_sa import u32_sa
from tests.test_gpu_lms_sort import lms_positions

pytestmark = pytest.mark.gpu

GL_LIMIT = 1024        # k_group_local_sort: steps from both ends; a group of GL_LIMIT + 2 members overflows
BS_CAP = 4096          # k_lms_bucket_sort: largest top-16 bucket of 2-bit text
KC = {"bytes": 4, "dna2": 16, "dna4": 13}           # window characters of each text kind
MAX_ROUNDS = {"bytes": 16, "dna2": 8, "dna4": 8}
ACGT = np.frombuffer(b"ACGT", np.uint8)

_ROUND = re.compile(r"direct LMS sort: round (\d+) \(h=\d+\): (\d+) -> (\d+) tied, (\S+)")
_HAND = re.compile(r"direct LMS sort: hand over to the robust path: (\S+)")
_DOUBLING = re.compile(r"doubling round (\d+): h=(\d+) -> active (\d+) of (\d+), (\S+)")
_ROUND0 = re.compile(r"reduced_sa: m=(\d+) names=(\d+) k0=(\d+) bw=(\d+): (\d+)-bit round-0 keys")


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


class Trace:
    def __init__(self, err):
        self.err = err
        self.rounds = {int(r): (int(a), int(b), how) for r, a, b, how in _ROUND.findall(err)}   # round -> (na, na_next, how)
        self.hand_over = _HAND.findall(err)
        self.doubling = [(int(r), int(h), int(a), how) for r, h, a, _, how in _DOUBLING.findall(err)]
        self.round0 = [(int(k0), int(bw), int(bits)) for _, _, k0, bw, bits in _ROUND0.findall(err)]

    def how(self, r):
        assert r in self.rounds, self.err[-3000:]
        return self.rounds[r][2]


def _set_env(monkeypatch, env):
    monkeypatch.setenv("B200SA_TRACE", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _clear_env(monkeypatch, env):
    for k in ("B200SA_TRACE",) + tuple(env):
        monkeypatch.delenv(k, raising=False)


def build(ctx, monkeypatch, capfd, t, **env):
    """Full build with B200SA_TRACE (and `env`); SA and LCP against the oracle.  -> (Trace, sa, direct_sort)"""
    capfd.readouterr()
    _set_env(monkeypatch, env)
    try:
        sa, lcp = ctx.build_lcp(t)
        direct = ctx.stats()["direct_sort"]
    finally:
        _clear_env(monkeypatch, env)
    tr = Trace(capfd.readouterr().err)
    want = oracle.sais(t)
    assert np.array_equal(sa, want), tr.err[-3000:]
    assert np.array_equal(lcp, oracle.lcp_kasai(t, want))
    return tr, sa, direct


def reduced(ctx, monkeypatch, capfd, R, names, **env):
    """b200sa_test_reduced_sa with B200SA_TRACE, against the numpy prefix-doubling reference."""
    m = len(R)
    out = np.empty(m, dtype=np.uint32)
    rounds = ctypes.c_uint32(0)
    capfd.readouterr()
    _set_env(monkeypatch, env)
    try:
        rc = _lib.lib().b200sa_test_reduced_sa(ctx._h, R.ctypes.data, m, names, out.ctypes.data, ctypes.byref(rounds))
    finally:
        _clear_env(monkeypatch, env)
    tr = Trace(capfd.readouterr().err)
    assert rc == 0, (rc, _lib.lib().b200sa_last_error(ctx._h))
    assert np.array_equal(out, u32_sa(R)), tr.err[-3000:]
    return tr, out


# ------------------------------------------------------------------ inputs of the direct path
def _background(kind, n, rng):
    if kind == "bytes":
        return rng.integers(0, 256, n, dtype=np.uint8)
    t = ACGT[rng.integers(0, 4, n)]
    if kind == "dna4":
        t[60::61] = ord("\n")                      # FASTA-like lines: sigma = 5, 4-bit packing
    return t


def _alphabet(kind):
    return np.arange(256, dtype=np.uint8) if kind == "bytes" else ACGT


# LMS at index 1 (an S-type character after an L-type one); the window from there lies inside the motif
MOTIF = {"bytes": np.frombuffer(b"\xff\x01\x02\x03\x04", np.uint8),
         "dna2": np.frombuffer(b"TA" + b"C" * 18, np.uint8),
         "dna4": np.frombuffer(b"TA" + b"C" * 18, np.uint8)}


def _group_size(t, kind, window):
    """LMS suffixes whose first window (kc characters, not truncated) equals `window`."""
    kc = KC[kind]
    p = lms_positions(t)
    p = p[p + kc <= len(t)]
    w = np.lib.stride_tricks.sliding_window_view(t, kc)[p]
    return int((w == window).all(axis=1).sum())


def motif_copies(kind, g, seed, tail=None, a_copy=False):
    """Random text of `kind` with one round-1 group of exactly g LMS suffixes: g copies of MOTIF, each
    followed by distinct random characters, so that round 2 sees one group of g members and splits it.
    tail = k: the last copy is followed by k 'A's and ends the text (k = 0: exactly at the end), and one
    more copy is followed by 40 'A's -- with 'A' = code 0 the padded windows of the truncated members
    equal its windows, and only the descending-position tie order puts them first."""
    rng = np.random.default_rng(seed)
    motif, kc = MOTIF[kind], KC[kind]
    alpha = _alphabet(kind)
    special = (tail is not None) + a_copy
    follow = alpha[rng.integers(0, len(alpha), (g - special, 16))]
    assert len(np.unique(follow[:, :kc], axis=0)) == g - special
    parts = [_background(kind, 30_000, rng)]
    parts += [np.concatenate([motif, f]) for f in follow]
    if a_copy:
        parts.append(np.concatenate([motif, np.full(40, ord("A"), np.uint8), np.frombuffer(b"C", np.uint8)]))
    parts.append(_background(kind, 30_000, rng))
    if tail is not None:
        parts.append(np.concatenate([motif, np.full(tail, ord("A"), np.uint8)]))
    t = np.concatenate(parts)
    assert _group_size(t, kind, motif[1:1 + kc]) == g
    return t


@pytest.mark.parametrize("kind", ["bytes", "dna2", "dna4"])
@pytest.mark.parametrize("g", [GL_LIMIT, GL_LIMIT + 1, GL_LIMIT + 2, 2000])
def test_local_sort_limit(ctx, monkeypatch, capfd, kind, g):
    """A group of g members in round 2: counted inside the group up to GL_LIMIT + 1 members, radix sorted
    after the overflow above that (the scan has already run on the overflowed buffers)."""
    t = motif_copies(kind, g, seed=g)
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 1 and not tr.hand_over
    assert tr.rounds[2][0] >= g
    assert tr.how(2) == ("local" if g <= GL_LIMIT + 1 else "radix(overflow)")
    assert all(how == "local" for r, (_, _, how) in tr.rounds.items() if r > 2)


@pytest.mark.parametrize("g", [2000, 5000])
def test_overflow_after_bucket_sort(ctx, monkeypatch, capfd, g):
    """2-bit text: the group ids of round 1 come from k_lms_bucket_sort (top-16 bucket <= BS_CAP) or from
    the four-pass sort and the max-scan (bucket > BS_CAP); either way round 2 overflows the local sort."""
    t = motif_copies("dna2", g, seed=7 * g)
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 1
    assert ("(bucket sort)" in tr.err) == (g <= BS_CAP) and ("four-pass sort" in tr.err) == (g > BS_CAP)
    assert tr.how(2) == "radix(overflow)"


@pytest.mark.parametrize("tail", [0, 5, 13])
@pytest.mark.parametrize("g", [1000, 2000])
def test_truncated_members(ctx, monkeypatch, capfd, g, tail):
    """Copies of the motif that end at the text end or `tail` characters before it sit in the big group
    with equal padded keys; they must stay in front of the copy that goes on (descending position) through
    the local sort (g = 1000) and the radix re-sort after an overflow (g = 2000)."""
    t = motif_copies("dna2", g, seed=g + tail, tail=tail, a_copy=True)
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 1
    assert tr.how(2) == ("local" if g <= GL_LIMIT + 1 else "radix(overflow)")
    assert all(how == "local" for r, (_, _, how) in tr.rounds.items() if r > 2)    # what round 2 left is small


def probe_text(copies, motifs, seed):
    """Random bytes with `motifs` distinct 5-byte motifs x `copies` copies, each followed by 4 random bytes:
    round 1 ties motifs x copies LMS suffixes in groups of `copies`, round 2 settles them."""
    rng = np.random.default_rng(seed)
    ids = rng.choice(253 ** 3, motifs, replace=False)
    mid = np.stack([ids // 253 ** 2, ids // 253 % 253, ids % 253], axis=1).astype(np.uint8) + 2
    rec = np.empty((motifs * copies, 9), np.uint8)
    rec[:, 0], rec[:, 1] = 0xFF, 0x01
    rec[:, 2:5] = np.repeat(mid, copies, axis=0)
    rec[:, 5:] = rng.integers(0, 256, (motifs * copies, 4), dtype=np.uint8)
    rec = rec[rng.permutation(len(rec))]
    return np.concatenate([rng.integers(0, 256, 100_000, dtype=np.uint8), rec.reshape(-1)])


@pytest.mark.parametrize("copies,motifs,how", [(150, 8000, "radix(probe)"), (4, 300_000, "local")],
                         ids=["big_groups", "small_groups"])
def test_probe(ctx, monkeypatch, capfd, copies, motifs, how):
    """>= 2^20 suffixes tied after round 1: the probe samples ~4096 of them and takes the radix sort when
    more than 5 % sit in groups of >= 128."""
    t = probe_text(copies, motifs, seed=copies)
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 1
    assert tr.rounds[2][0] >= 1 << 20
    assert tr.how(2) == how


# ------------------------------------------------------------------ hand-over to the robust path
def periodic_lms(m):
    """'ba' + 'c' * 20, m times: m LMS suffixes (the a's), all with the same 16-character window."""
    return np.tile(np.frombuffer(b"ba" + b"c" * 20, np.uint8), m)


def test_round1_tied(ctx, monkeypatch, capfd):
    t = periodic_lms(65)
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert ctx.stats()["m"] == 65
    assert direct == 0 and tr.hand_over == ["round1-tied"]
    t = periodic_lms(64)                      # m <= 64 is exempt from that rule (a later one may still apply)
    tr, _, _ = build(ctx, monkeypatch, capfd, t)
    assert ctx.stats()["m"] == 64
    assert "round1-tied" not in tr.hand_over and 2 in tr.rounds
    tr, _, direct = build(ctx, monkeypatch, capfd, gen.tiled(gen.fixture("AP009048_10000.fasta"), 200_000))
    assert direct == 0 and tr.hand_over == ["round1-tied"]


@pytest.mark.parametrize("kind", ["bytes", "dna2"])
def test_no_convergence(ctx, monkeypatch, capfd, kind):
    """A 1 MB random block, an exact copy of it, then 1 MB of fresh random text: round 2 keeps
    almost all of the ~2/3 tied after round 1."""
    rng = np.random.default_rng(3)
    block = _background(kind, 1 << 20, rng)
    t = np.concatenate([block, block, _background(kind, 1 << 20, rng)])
    tr, _, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 0 and tr.hand_over == ["no-convergence"]
    assert max(tr.rounds) == 2


def repeat_pairs(kind, length, pairs, n, seed):
    """Random text of `kind` with `pairs` random strings of `length` inserted twice each, the two copies
    preceded and followed by different characters: no two suffixes share more than `length` characters
    by way of a repeat."""
    rng = np.random.default_rng(seed)
    alpha = _alphabet(kind) if kind != "dna4" else np.frombuffer(b"ACGT\n", np.uint8)
    t = _background(kind, n, rng)
    cut = np.sort(rng.choice(n, 2 * pairs, replace=False))
    order = rng.permutation(2 * pairs)
    reps = alpha[rng.integers(0, len(alpha), (pairs, length))]
    parts, prev = [], 0
    for k, c in enumerate(cut):
        i = order[k] // 2
        edge = alpha[[(order[k] % 2 + i) % len(alpha)]]         # the two copies start and end differently
        parts += [t[prev:c], edge, reps[i], edge]
        prev = c
    parts.append(t[prev:])
    return np.concatenate(parts)


@pytest.mark.parametrize("kind", ["bytes", "dna2", "dna4"])
def test_round_limit(ctx, monkeypatch, capfd, kind):
    """Repeats just shorter than rounds x kc characters are settled by the last round the direct path
    allows; repeats just longer stay tied and hand over at the limit, with no environment variable."""
    limit = MAX_ROUNDS[kind] * KC[kind]
    n = 1 << 21
    tr, _, direct = build(ctx, monkeypatch, capfd, repeat_pairs(kind, limit - 1, 100, n, seed=1))
    assert direct == 1 and not tr.hand_over
    assert max(tr.rounds) == MAX_ROUNDS[kind]
    tr, _, direct = build(ctx, monkeypatch, capfd, repeat_pairs(kind, limit + 12, 100, n, seed=2))
    assert direct == 0 and tr.hand_over == ["round-limit"]
    assert max(tr.rounds) == MAX_ROUNDS[kind]


# ------------------------------------------------------------------ robust path: the reduced string
def _random_u32(m, names, seed):
    R = np.random.default_rng(seed).integers(0, names, m, dtype=np.uint32)
    R[m // 2] = names - 1                           # the largest symbol occurs
    return R


@pytest.mark.parametrize("m,names,bits", [(1 << 21, 1 << 17, 64), (1 << 21, 1 << 16, 64), (1 << 21, (1 << 16) - 1, 32)],
                         ids=["names_2^17", "names_2^16", "names_2^16-1"])
def test_round0_key_width(ctx, monkeypatch, capfd, m, names, bits):
    """Symbols are stored +1, so names = 2^16 needs 17 bits: two of them overflow a 32-bit key."""
    R = _random_u32(m, names, seed=names)
    tr, _ = reduced(ctx, monkeypatch, capfd, R, names)
    (k0, bw, got), = tr.round0
    assert bw == int(names).bit_length()
    assert got == bits and (k0 * bw > 32) == (bits == 64)


def test_overflow_then_radix(ctx, monkeypatch, capfd):
    """Random string with one run of 2000 equal symbols: the probe passes (the run is < 5 % of the tied),
    the local sort overflows on the run's group, and every later round is radix sorted."""
    R = _random_u32(300_000, 8, seed=11)
    R[100_000:102_000] = 5
    tr, out = reduced(ctx, monkeypatch, capfd, R, 8)
    hows = [how for _, _, _, how in tr.doubling]
    assert hows[0] == "radix(overflow)" and len(hows) > 1
    assert all(how == "radix(off)" for how in hows[1:])
    tr2, out2 = reduced(ctx, monkeypatch, capfd, R, 8, B200SA_NO_LOCAL_SORT="1")
    assert all(how == "radix(off)" for _, _, _, how in tr2.doubling)
    assert np.array_equal(out2, out)


def test_periodic_probe(ctx, monkeypatch, capfd):
    """A periodic string: every group is large, the probe rejects the local sort in the first round."""
    R = np.tile(np.array([3, 1, 2, 1], np.uint32), 75_000)
    tr, _ = reduced(ctx, monkeypatch, capfd, R, 4)
    assert tr.doubling[0][3] == "radix(probe)"


@pytest.mark.parametrize("k0", [1, "max", None], ids=["k0_1", "k0_max", "k0_default"])
def test_k0(ctx, monkeypatch, capfd, k0):
    rng = np.random.default_rng(13)
    block = rng.integers(0, 4096, 200_000, dtype=np.uint32)
    R = np.concatenate([block, block, rng.integers(0, 4096, 100_000, dtype=np.uint32)])
    names = int(R.max()) + 1
    bw = names.bit_length()
    env = {} if k0 is None else {"B200SA_K0": str(64 // bw if k0 == "max" else k0)}
    tr, _ = reduced(ctx, monkeypatch, capfd, R, names, **env)
    (got_k0, got_bw, bits), = tr.round0
    assert got_bw == bw
    if k0 is not None:
        assert got_k0 == (64 // bw if k0 == "max" else k0)
    assert bits == (64 if got_k0 * bw > 32 else 32)
    assert len(tr.doubling) > 1


# ------------------------------------------------------------------ robust path: full builds
def _long_repeats(kind):
    rng = np.random.default_rng(17)
    block = _background(kind, 100_000, rng)
    return np.concatenate([block, block, block[:70_000], _background(kind, 50_000, rng)])


_ROBUST_TEXTS = {"tiled": lambda: gen.tiled(gen.fixture("AP009048_10000.fasta"), 200_000),
                 "bytes": lambda: _long_repeats("bytes"), "dna4": lambda: _long_repeats("dna4")}


@pytest.mark.parametrize("kgram", ["0", "1", "2", None], ids=["kgram0", "kgram1", "kgram2", "kgram_default"])
@pytest.mark.parametrize("text", sorted(_ROBUST_TEXTS))
def test_robust_kgram(ctx, monkeypatch, capfd, text, kgram):
    """B200SA_NO_DIRECT=1: KGRAM 0 and 1 take the plain-pair first refinement, 2 the shortest k-gram of
    names and the default the widest one that fits 64 bits (at most 8)."""
    env = {"B200SA_NO_DIRECT": "1"} | ({} if kgram is None else {"B200SA_KGRAM": kgram})
    tr, _, direct = build(ctx, monkeypatch, capfd, _ROBUST_TEXTS[text](), **env)
    assert direct == 0 and tr.doubling
    names = ctx.stats()["names"]
    k = min(8, 64 // int(names).bit_length()) if kgram is None else int(kgram)
    first = tr.doubling[0]
    assert first[1] == 1
    if k >= 2:
        assert first[3] == "radix(kgram)"
        if len(tr.doubling) > 1:
            assert tr.doubling[1][1] == k                  # the second round starts at depth k
    else:
        assert all(how != "radix(kgram)" for _, _, _, how in tr.doubling)
        if len(tr.doubling) > 1:
            assert tr.doubling[1][1] == 2


def test_cross_checks(ctx, monkeypatch, capfd):
    """The default build sends the group of 2000 to the radix sort in round 2 (too large for the local
    sort); B200SA_NO_LOCAL_SORT=1 (radix sort in every round) gives the same result."""
    t = motif_copies("bytes", 2000, seed=2000)
    tr, sa, direct = build(ctx, monkeypatch, capfd, t)
    assert direct == 1 and tr.how(2) == "radix(overflow)"
    tr1, sa1, direct = build(ctx, monkeypatch, capfd, t, B200SA_NO_LOCAL_SORT="1")
    assert direct == 1 and all(how == "radix(off)" for _, _, how in tr1.rounds.values())
    assert np.array_equal(sa1, sa)
