"""Parity of the CUDA path (through the C-ABI) with the oracle: bit-exact SA
and LCP on the reference's KATs, the fixtures, adversarial families, random
properties, and size-independent properties at larger sizes."""
import hashlib

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

from oracle import oracle
from suffix_b200 import SuffixTable, _lib, gen
from tests import families

pytestmark = pytest.mark.gpu
KAT = families.kat()


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _np(b):
    return np.frombuffer(bytes(b), dtype=np.uint8)


@pytest.mark.parametrize("case", KAT["kat"], ids=lambda c: repr(c["text"])[:24])
def test_kat(case):
    # tests/tests.rs:22-70: naive(x) == sais(x) (text + table equality)
    t = case["text"].encode("utf-8")
    st_ = SuffixTable(case["text"])
    assert st_.table().tolist() == case["sa"]
    assert st_.text() == t and len(st_) == len(t)
    assert st_.lcp_lens().tolist() == case["lcp"]
    assert st_ == SuffixTable.from_parts(t, oracle.naive_sa(t))


@pytest.mark.parametrize("case", KAT["positions"], ids=lambda c: repr((c["text"], c["query"]))[:40])
def test_kat_positions(case):
    # tests/tests.rs:100-213
    st_ = SuffixTable(case["text"])
    assert st_.positions(case["query"]).tolist() == case["positions"]
    assert st_.contains(case["query"]) == bool(case["positions"])
    hit = st_.any_position(case["query"])
    assert (hit in case["positions"]) if case["positions"] else hit is None


def test_save_load_roundtrip(tmp_path):
    sa = SuffixTable("The quick brown fox was very quick.")
    sa.save(str(tmp_path / "idx"))
    sb = SuffixTable.load(str(tmp_path / "idx"))
    assert sa == sb and sb.positions("quick").tolist() == [4, 29]


def test_parts_roundtrip():
    # tests/tests.rs:171-179
    sa = SuffixTable("poëzie")
    data, table = sa.into_parts()
    assert sa == SuffixTable.from_parts(data, table)


@pytest.mark.parametrize("name", sorted(KAT["fixtures"]))
def test_fixture_sha256(ctx, name):
    info = KAT["fixtures"][name]
    t = gen.fixture(name)
    sa, lcp = ctx.build_lcp(t)
    assert sa[:8].tolist() == info["sa_head"]
    assert hashlib.sha256(sa.astype("<u4").tobytes()).hexdigest() == info["sa_sha256"]
    assert hashlib.sha256(lcp.astype("<u4").tobytes()).hexdigest() == info["lcp_sha256"]


@pytest.fixture(params=["direct", "robust"])
def lms_path(request, monkeypatch):
    """Both ways of sorting the LMS suffixes: directly by character windows
    (lms_sort.cuh; falls through to the robust path by itself on long repeats) and the
    robust path alone (stage-1 induce + naming + rank doubling)."""
    if request.param == "robust":
        monkeypatch.setenv("B200SA_NO_DIRECT", "1")
    return request.param


@pytest.mark.parametrize("name,data", families.adversarial(), ids=lambda x: x if isinstance(x, str) else "")
def test_adversarial(ctx, lms_path, name, data):
    t = _np(data)
    want = oracle.sais(t)
    sa, lcp = ctx.build_lcp(t)
    assert np.array_equal(sa, want), name
    assert np.array_equal(lcp, oracle.lcp_kasai(t, want)), name


@pytest.mark.parametrize("maker,n", [("dna", 1_000_000), ("dna_nl", 1_000_001), ("bytes", 1_000_000),
                                     ("english", 1_000_000), ("tiled", 1_000_000), ("dna", 5_000_000),
                                     ("bytes", 5_000_000)])
def test_medium_vs_oracle(ctx, lms_path, maker, n):
    if maker == "dna":
        t = gen.dna(n)
    elif maker == "dna_nl":
        t = gen.dna(n, newline_tail=True)
    elif maker == "bytes":
        t = gen.rand_bytes(n)
    elif maker == "english":
        t = gen.english(n)
    else:
        t = gen.tiled(gen.fixture("AP009048_100000.fasta"), n)
    want = oracle.sais(t)
    sa = ctx.build(t)
    assert np.array_equal(sa, want)
    if maker != "tiled":     # tiled text has LCP ~ n: quadratic in any LCP algorithm that restarts
        lcp = ctx.lcp(t, sa)
        assert np.array_equal(lcp, oracle.lcp_kasai(t, want))


@pytest.mark.parametrize("maker", ["dna", "bytes", "fixture"])
def test_lcp_both_paths(ctx, maker, monkeypatch):
    """lcp_lens has a direct fast path (the reference's per-pair lcp_len, capped)
    and the linear Phi/PLCP path; both must give the reference's array."""
    t = {"dna": lambda: gen.dna(2_000_000), "bytes": lambda: gen.rand_bytes(2_000_000),
         "fixture": lambda: gen.fixture("AP009048_100000.fasta")}[maker]()
    want_sa = oracle.sais(t)
    want = oracle.lcp_kasai(t, want_sa)
    assert np.array_equal(ctx.lcp(t, want_sa), want)
    monkeypatch.setenv("B200SA_LCP_LINEAR", "1")
    assert np.array_equal(ctx.lcp(t, want_sa), want)
    monkeypatch.setenv("B200SA_PHI_DIRECT", "1")
    assert np.array_equal(ctx.lcp(t, want_sa), want)


def _long_run_cases():
    rng = np.random.default_rng(99)
    d = gen.dna(600_000)
    out = [("a^2M", np.full(2_000_000, 97, dtype=np.uint8)),
           ("zeros_ff", np.concatenate([np.zeros(1_500_000, dtype=np.uint8), np.full(1_500_000, 255, dtype=np.uint8)])),
           ("ff_zeros", np.concatenate([np.full(1_500_000, 255, dtype=np.uint8), np.zeros(1_500_000, dtype=np.uint8)]))]
    # poly-N genome shape: DNA with a few very long and many short N runs
    parts = []
    for k in range(40):
        parts.append(d[k * 15000:(k + 1) * 15000])
        parts.append(np.full(int(rng.choice([1, 3, 70, 500, 4097, 65, 300_000 if k % 13 == 0 else 9])), ord("N"), dtype=np.uint8))
    out.append(("polyN", np.concatenate(parts)))
    # runs of the SMALLEST and of a MIDDLE symbol, ending the text with a run
    parts = []
    for k in range(30):
        parts.append(d[k * 7000:(k + 1) * 7000])
        parts.append(np.full(int(rng.choice([2, 64, 65, 4096, 100_000])), ord("A") if k % 2 else ord("G"), dtype=np.uint8))
    out.append(("polyA_G_tail", np.concatenate(parts)))
    return out


@pytest.mark.parametrize("name,t", _long_run_cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_long_runs(ctx, lms_path, name, t):
    """Run skipping in the induce (DESIGN.md 2.1): chains along runs of 10^5..10^6 equal bytes."""
    t = np.ascontiguousarray(t)
    sa = ctx.build(t)
    want = oracle.sais(t)
    assert np.array_equal(sa, want), name
    if name.startswith("poly"):          # LCP inside long runs: capped fast path -> two-level PLCP fallback
        assert np.array_equal(ctx.lcp(t, sa), oracle.lcp_kasai(t, want)), name


def _two_bit_cases():
    rng = np.random.default_rng(11)
    runs = []
    for k in range(300):                       # runs of the bucket chars of every length around the cascade depth
        runs.append(np.full(int(rng.integers(1, 12)), b"ACGT"[k % 4], dtype=np.uint8))
        runs.append(gen.dna(int(rng.integers(1, 40)), seed=k))
    return [("dna_3M", gen.dna(3_000_000, seed=5)),
            ("short_runs", np.concatenate(runs * 40)),
            ("polyA_mix", np.concatenate([gen.dna(200_000, seed=2), np.full(50_000, ord("A"), np.uint8), gen.dna(100_000, seed=3),
                                          np.full(9_000, ord("T"), np.uint8), gen.dna(1000, seed=4)])),
            ("two_symbols", rng.integers(0, 2, 700_000).astype(np.uint8) * 2 + ord("A")),
            ("tiny", gen.dna(37, seed=9))]


@pytest.mark.parametrize("variant", ["1", "6", "6_no_cascade", "6_cascade_4096"])
@pytest.mark.parametrize("name,t", _two_bit_cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_induce_variants_two_bit(ctx, monkeypatch, variant, name, t):
    """Every induce kernel variant for 2-bit text (DESIGN.md 2.2) and the cascade steps of the default
    one with their switch off / a low list limit: same table as the oracle."""
    monkeypatch.setenv("B200SA_INDUCE", variant[0])
    if variant == "6_no_cascade":
        monkeypatch.setenv("B200SA_NO_CASCADE", "1")
    if variant == "6_cascade_4096":
        monkeypatch.setenv("B200SA_CASCADE_MAX", "4096")
    t = np.ascontiguousarray(t)
    assert np.array_equal(ctx.build(t), oracle.sais(t)), (variant, name)


def _check_sa_properties(t, sa, samples=200000, seed=1):
    """Size-independent properties: permutation + sampled adjacent order."""
    n = len(t)
    assert len(sa) == n
    seen = np.zeros(n, dtype=np.uint8)
    seen[sa] = 1
    assert int(seen.sum()) == n                       # permutation of 0..n-1
    rng = np.random.default_rng(seed)
    idx = rng.integers(1, n, min(samples, n - 1))
    tb = t.tobytes()
    for i in idx.tolist():
        a, b = int(sa[i - 1]), int(sa[i])
        k = 64
        while True:
            x, y = tb[a:a + k], tb[b:b + k]
            if x != y or a + k >= n or b + k >= n:
                break
            k *= 4
        assert tb[a:a + k] < tb[b:b + k], (i, a, b)


@pytest.mark.slow
@pytest.mark.parametrize("name", ["G_dna_100MB", "G_bytes_100MB"])
def test_full_size_bit_exact(ctx, name):
    """BASELINE.json configs[1] and configs[2] at FULL size (100 MB): SA and LCP
    bit for bit against the oracle run right here (restated sais(), src/table.rs:388-574,
    and lcp_lens_quadratic, :348-361) and against the SHA-256 goldens pinned in
    tests/golden/full_size.json (tests/golden/make_full_size.py)."""
    info = families.full_size()[name]
    t = gen.dna(info["n"]) if name.startswith("G_dna") else gen.rand_bytes(info["n"])
    assert hashlib.sha256(t.tobytes()).hexdigest() == info["text_sha256"]
    sa, lcp = ctx.build_lcp(t)
    assert sa[:8].tolist() == info["sa_head"] and lcp[:8].tolist() == info["lcp_head"]
    assert hashlib.sha256(sa.astype("<u4").tobytes()).hexdigest() == info["sa_sha256"]
    assert hashlib.sha256(lcp.astype("<u4").tobytes()).hexdigest() == info["lcp_sha256"]
    want = oracle.sais(t)
    assert np.array_equal(sa, want)
    assert np.array_equal(lcp, oracle.lcp_quadratic(t, want))
    # lcp_lens on its own (text + table through b200sa_lcp) takes the stand-alone packing path
    assert np.array_equal(ctx.lcp(t, sa), lcp)


@pytest.mark.slow
def test_config4_english_1gb(ctx):
    """BASELINE.json configs[3]: 1 GB English-like UTF-8 text.  The oracle's sais()
    needs minutes at this size, so the SA is proven by the O(n) verifier
    (oracle.verify_sa: permutation + neighbour order through the inverse -- valid
    iff sa is THE suffix array, hence equal to the reference's) and the LCP array is
    compared bit for bit with the oracle's byte-level Kasai (pinned to
    lcp_lens_quadratic by tests/test_oracle.py)."""
    n = 1_000_000_000
    t = gen.english(n)
    sa, lcp = ctx.build_lcp(t)
    assert oracle.verify_sa(t, sa) == 0
    assert np.array_equal(lcp, oracle.lcp_kasai(t, sa))


@settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.text(max_size=300))
def test_prop_text(s):
    # tests/tests.rs:73-96 prop_naive_equals_sais / prop_matches_naive, :215-221 prop_length
    t = s.encode("utf-8")
    tab = SuffixTable(s)
    assert len(tab) == len(t)
    assert np.array_equal(tab.table(), oracle.naive_sa(t))


@settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.binary(max_size=600))
def test_prop_binary(b):
    tab = SuffixTable(b)
    assert np.array_equal(tab.table(), oracle.naive_sa(b))
    if len(b):
        assert np.array_equal(tab.lcp_lens(), oracle.lcp_quadratic(b, tab.table()))


@settings(max_examples=100, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.text(max_size=100), st.integers(0, 255))
def test_prop_positions(s, c):
    # tests/tests.rs:223-243 prop_contains / prop_positions
    q = chr(c)
    tab = SuffixTable(s)
    want = [i for i in range(len(s.encode())) if s.encode().startswith(q.encode(), i)]
    assert sorted(tab.positions(q).tolist()) == want
    assert tab.contains(q) == (q in s)


def test_positions_dev_batch(ctx):
    import torch
    t = gen.fixture("AP009048_100000.fasta")
    tab = SuffixTable(t.tobytes())
    queries = [b"ACGT", b"GATTACA", b"T", b"\n", b"ZZZ", b"A" * 30, t.tobytes()[500:540], b"ACGTACGTAC"]
    flat = np.frombuffer(b"".join(queries), dtype=np.uint8)
    off = np.cumsum([0] + [len(q) for q in queries]).astype(np.uint64)
    dev = torch.device("cuda:0")
    d_t = torch.from_numpy(t.copy()).to(dev)
    d_sa = torch.from_numpy(tab.table().astype(np.int64)).to(dev).to(torch.int32)  # same 4-byte payload
    d_q = torch.from_numpy(flat.copy()).to(dev)
    d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
    d_s = torch.zeros(len(queries), dtype=torch.int32, device=dev)
    d_e = torch.zeros(len(queries), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ctx.positions_dev(d_t.data_ptr(), len(t), d_sa.data_ptr(), d_q.data_ptr(), d_off.data_ptr(), len(queries),
                      d_s.data_ptr(), d_e.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    s, e = d_s.cpu().numpy(), d_e.cpu().numpy()
    for k, q in enumerate(queries):
        assert (int(s[k]), int(e[k])) == oracle.positions(t, tab.table(), q), q     # src/table.rs:223-259
        assert tab.table()[s[k]:e[k]].tolist() == tab.positions(q).tolist(), q


def test_direct_path_taken(ctx):
    """The direct LMS sort must actually be the path random-like texts take (and the
    robust path the one a tiled text ends up on)."""
    ctx.build(gen.dna(2_000_000))
    assert ctx.stats()["direct_sort"] == 1
    ctx.build(gen.rand_bytes(2_000_000))
    assert ctx.stats()["direct_sort"] == 1
    ctx.build(gen.dna(2_000_001, newline_tail=True))
    assert ctx.stats()["direct_sort"] == 1
    ctx.build(gen.english(2_000_000))                  # 4-5 byte windows, ~10 rounds
    assert ctx.stats()["direct_sort"] == 1
    ctx.build(gen.tiled(gen.fixture("AP009048_10000.fasta"), 2_000_000))
    assert ctx.stats()["direct_sort"] == 0


@pytest.mark.parametrize("rounds", [1, 2, 3])
def test_direct_round_limits(ctx, monkeypatch, rounds):
    """Giving up after any number of window rounds hands over to the robust path cleanly."""
    monkeypatch.setenv("B200SA_DIRECT_ROUNDS", str(rounds))
    for t in (gen.fixture("AP009048_100000.fasta"), gen.english(400_000), gen.dna(500_000)):
        assert np.array_equal(ctx.build(t), oracle.sais(t))


def test_build_dev_matches_host(ctx):
    import torch
    t = gen.dna(300_000)
    dev = torch.device("cuda:0")
    d_t = torch.from_numpy(t.copy()).to(dev)
    d_sa = torch.empty(len(t), dtype=torch.int32, device=dev)
    d_lcp = torch.empty(len(t), dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    ctx.build_dev(d_t.data_ptr(), len(t), d_sa.data_ptr(), stream)
    ctx.lcp_dev(d_t.data_ptr(), len(t), d_sa.data_ptr(), d_lcp.data_ptr(), stream)
    torch.cuda.synchronize()
    want = oracle.sais(t)
    assert np.array_equal(d_sa.cpu().numpy().view(np.uint32), want)
    assert np.array_equal(d_lcp.cpu().numpy().view(np.uint32), oracle.lcp_kasai(t, want))
    d_sa.zero_(); d_lcp.zero_()
    ctx.build_lcp_dev(d_t.data_ptr(), len(t), d_sa.data_ptr(), d_lcp.data_ptr(), stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_sa.cpu().numpy().view(np.uint32), want)
    assert np.array_equal(d_lcp.cpu().numpy().view(np.uint32), oracle.lcp_kasai(t, want))
    # unaligned device pointer (exercises the internal aligned copy)
    d_t2 = torch.from_numpy(np.concatenate([[0], t]).astype(np.uint8)).to(dev)[1:]
    ctx.build_dev(d_t2.data_ptr(), len(t), d_sa.data_ptr(), stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_sa.cpu().numpy().view(np.uint32), want)
    d_sa.zero_(); d_lcp.zero_()
    ctx.build_lcp_dev(d_t2.data_ptr(), len(t), d_sa.data_ptr(), d_lcp.data_ptr(), stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_sa.cpu().numpy().view(np.uint32), want)
    assert np.array_equal(d_lcp.cpu().numpy().view(np.uint32), oracle.lcp_kasai(t, want))


def test_error_codes(ctx):
    """Boundary error behaviour (include/b200sa.h): bad arguments and the size limit."""
    L = _lib.lib()
    buf = np.zeros(4, dtype=np.uint32)
    t = np.frombuffer(b"abcd", dtype=np.uint8)
    assert L.b200sa_build(ctx._h, None, 4, buf.ctypes.data) == -1                 # B200SA_ERR_BAD_ARG
    assert L.b200sa_build(ctx._h, t.ctypes.data, 4, None) == -1
    assert L.b200sa_build(None, t.ctypes.data, 4, buf.ctypes.data) == -1
    assert L.b200sa_build(ctx._h, t.ctypes.data, 0xFFFFF001, buf.ctypes.data) == -2  # B200SA_ERR_TOO_LARGE, nothing touched
    assert b"2^32" in L.b200sa_last_error(ctx._h)
    assert L.b200sa_build(ctx._h, None, 0, None) == 0                              # empty text: no launch
    assert ctx.stats()["kernel_launches"] == 0
    one = np.zeros(1, dtype=np.uint32) + 7
    assert L.b200sa_build(ctx._h, t.ctypes.data, 1, one.ctypes.data) == 0 and one[0] == 0


def test_lcp_rejects_bad_table(ctx):
    """from_parts accepts any table (src/table.rs:111-119); lcp_lens on a table that is
    not a permutation must fail cleanly instead of indexing out of bounds."""
    t = gen.dna(100_000)
    sa = oracle.sais(t)
    for bad in (np.full(len(t), 7, dtype=np.uint32), np.where(np.arange(len(t)) == 5, 0xFFFFFFF0, sa).astype(np.uint32)):
        with pytest.raises(_lib.B200SAError) as ei:
            ctx.lcp(t, bad)
        assert ei.value.code == -1 and "permutation" in str(ei.value)
    assert np.array_equal(ctx.lcp(t, sa), oracle.lcp_kasai(t, sa))     # the context is still usable


def test_two_contexts_two_threads():
    """Distinct contexts are independent (INTEGRATION.md section 4): two host threads,
    two contexts on the same device, interleaved builds."""
    import threading
    texts = [gen.dna(400_000, seed=11), gen.rand_bytes(300_000, seed=12)]
    want = [oracle.sais(t) for t in texts]
    errs = []

    def work(k):
        try:
            c = _lib.Context(0)
            for _ in range(5):
                sa, lcp = c.build_lcp(texts[k])
                assert np.array_equal(sa, want[k])
                assert np.array_equal(lcp, oracle.lcp_kasai(texts[k], want[k]))
            c.close()
        except Exception as e:          # noqa: BLE001
            errs.append(repr(e))

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs


def test_host_api_pinned_buffers_early_copy(ctx):
    """b200sa_build_lcp with pinned host buffers takes the early SA copy-out path
    (bucket parts leave as soon as they are final); result must be identical."""
    import torch
    t = gen.dna(3_000_000, newline_tail=True)
    want = oracle.sais(t)
    h_t = torch.from_numpy(t.copy()).pin_memory()
    h_sa = torch.empty(len(t), dtype=torch.int32).pin_memory()
    h_lcp = torch.empty(len(t), dtype=torch.int32).pin_memory()
    L = _lib.lib()
    for _ in range(2):
        h_sa.zero_()
        assert L.b200sa_build_lcp(ctx._h, h_t.data_ptr(), len(t), h_sa.data_ptr(), h_lcp.data_ptr()) == 0
        assert np.array_equal(h_sa.numpy().view(np.uint32), want)
        assert np.array_equal(h_lcp.numpy().view(np.uint32), oracle.lcp_kasai(t, want))
    h_sa.zero_()
    assert L.b200sa_build(ctx._h, h_t.data_ptr(), len(t), h_sa.data_ptr()) == 0
    assert np.array_equal(h_sa.numpy().view(np.uint32), want)
