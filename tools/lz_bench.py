"""f-12: longest previous factors and the LZ77 factorization (b200sa_lpf_dev, b200sa_lz77_dev) on
device-resident tables.  Prints one JSON line: card and power limit; per arm z, the parse's rounds, the
median CUDA-event time (one warm-up, then --reps) of b200sa_lpf_dev and of the count call + the fetch call of
b200sa_lz77_dev, the median of every phase of the fetch call, the workspace a context of its own grew to per
text byte, and agreement with the serial C statement of tests/lz_check.c on one host core over the WHOLE arm
(lpf, src and the factors), whose time is recorded, and with the text its decoder rebuilds from the factors.

    python tools/lz_bench.py [--n 100000000] [--reps 5]

Arms: G_dna, G_bytes and G_english (as bench.py), the AP009048 fixture tiled to n, and G_dna cut into
documents of about 1 kB with 10 % of them overwritten by copies of earlier documents with 1 % substitutions
(seeded)."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tests import lz_check
from tools.docs_bench import card, cut, phase_times, timed
from tools.repeat_bench import agrees, plant

PHASES = ("lz_levels", "lz_lpf", "lz_parse", "lz_count", "lz_emit")


def run_arm(build_ctx, stream, text, starts, reps):
    s, n = stream.cuda_stream, len(text)
    d_t = torch.from_numpy(text).cuda()
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
    if starts is None:
        build_ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    else:
        d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
        build_ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(starts), d_sa.data_ptr(), d_lcp.data_ptr(), s)
        del d_s
    torch.cuda.synchronize()
    del d_t
    ctx = _lib.Context(0)                        # a context of its own: its workspace is this row's alone
    P = (n, d_sa.data_ptr(), d_lcp.data_ptr())
    res = {"docs": 1 if starts is None else len(starts)}

    d_lpf, d_src = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
    lpf = lambda: ctx.lpf_dev(*P, d_lpf.data_ptr(), d_src.data_ptr(), s)
    lpf()
    ts = [timed(stream, lpf) for _ in range(reps)]
    res["lpf"] = {"ms_median": round(statistics.median(ts), 3), "ms_all": [round(v, 3) for v in ts]}

    z = ctx.lz77_dev(*P, stream=s)
    rounds = ctx.stats()["doubling_rounds"]
    bufs = [torch.empty(max(z, 1), dtype=torch.int32, device="cuda") for _ in range(3)]

    def lz77():                                  # the protocol a caller follows: count, then fetch
        ctx.lz77_dev(*P, stream=s)
        ctx.lz77_dev(*P, *(b.data_ptr() for b in bufs), z, s)

    lz77()
    ts = [timed(stream, lz77) for _ in range(reps)]
    ctx.set_timing(True)
    split = {p: [] for p in PHASES}
    for _ in range(reps):
        ctx.lz77_dev(*P, *(b.data_ptr() for b in bufs), z, s)
        for p, ms in phase_times(ctx):
            if p in split:
                split[p].append(ms)
    ctx.set_timing(False)
    ws = ctx.stats()["workspace_bytes"]
    sa, lcp = d_sa.cpu().numpy().view(np.uint32), d_lcp.cpu().numpy().view(np.uint32)
    t0 = time.perf_counter()
    want = lz_check.lz(sa, lcp)
    host = time.perf_counter() - t0
    got = [b[:z].cpu().numpy().view(np.uint32) for b in bufs]
    agree = (z == len(want[2]) and np.array_equal(d_lpf.cpu().numpy().view(np.uint32), want[0]) and
             np.array_equal(d_src.cpu().numpy().view(np.uint32), want[1]) and
             all(np.array_equal(a, b) for a, b in zip(got, want[2:])))
    decoded = bool(np.array_equal(lz_check.decode(text, *got), text))
    res["lz77"] = {"z": z, "parse_rounds": rounds, "count_plus_fetch_ms_median": round(statistics.median(ts), 3),
                   "count_plus_fetch_ms_all": [round(v, 3) for v in ts],
                   "fetch_phases_ms_median": {p: round(statistics.median(v), 3) for p, v in split.items() if v},
                   "serial_c_one_core_s": round(host, 2), "agree": bool(agree), "agree_decoded": decoded}
    res["workspace_bytes_per_text_byte"] = round(ws / n, 3)
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lz_bench: no CUDA device")
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    out = {"gpu": name, "power_limit": power, "n": a.n, "reps": a.reps}
    dna = gen.dna(a.n)
    starts = cut(a.n, 500, 1500, 1)
    arms = (("G_dna", lambda: (dna, None)), ("G_bytes", lambda: (gen.rand_bytes(a.n), None)),
            ("G_english", lambda: (gen.english(a.n), None)),
            ("AP009048_tiled", lambda: (gen.tiled(gen.fixture("AP009048_100000.fasta"), a.n), None)),
            ("planted_documents_1kB", lambda: (plant(dna, starts, np.random.default_rng(2)), starts)))
    for arm, make in arms:
        t, st = make()
        out[arm] = run_arm(ctx, stream, t, st, a.reps)
        torch.cuda.empty_cache()
    out["agree"] = agrees({k: v for k, v in out.items() if isinstance(v, dict)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
