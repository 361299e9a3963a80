"""f-6: the separator-free generalized suffix array (b200sa_docs_build_dev) against the plain
SA + LCP build (b200sa_build_lcp_dev) of the same concatenation.  Prints one JSON line: card and
power limit, and per cut of the text the median CUDA-event times of both calls (one warm-up, then
--reps each), |A| (ranks whose suffix in the concatenation reaches past their document's end:
the ones that are sorted), the phase split of one timed docs build, the device workspace of each
call on a fresh context in bytes per text byte, and
whether tests/docs_check.c accepts G and its LCP.

    python tools/docs_bench.py [--n 100000000] [--reps 5] [--no-check]

Cuts: G_dna into documents of about 1 kB (uniform 500..1499 bytes) and about 100 kB
(50,000..149,999 bytes), and n/4 copies of "ACGT" (every suffix but the first copy's crosses)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(stream, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def phase_times(ctx, cap=4096):
    """b200sa_last_phase_times without Context.phase_times' 64-entry limit (the robust build of
    periodic text records more phases than that)."""
    import ctypes
    names = (ctypes.c_char_p * cap)()
    ms = (ctypes.c_float * cap)()
    k = _lib.lib().b200sa_last_phase_times(ctx._h, names, ms, cap)
    return [(names[i].decode(), float(ms[i])) for i in range(max(0, min(k, cap)))]


def cut(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(lo, hi, n // lo + 1)
    starts = np.concatenate([[0], np.cumsum(lens)])
    return starts[starts < n].astype(np.uint32)


def run(ctx, stream, text, starts, reps, check):
    n = len(text)
    d_t = torch.from_numpy(text).cuda()
    d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
    d_g = torch.empty(n, dtype=torch.int32, device="cuda")
    d_gl = torch.empty(n, dtype=torch.int32, device="cuda")
    s = stream.cuda_stream
    build = lambda: ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    docs = lambda: ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(starts), d_g.data_ptr(), d_gl.data_ptr(), s)
    build()
    docs()
    tb, td = [], []
    for _ in range(reps):                        # alternated, so both see the same card state
        tb.append(timed(stream, build))
        td.append(timed(stream, docs))
    ctx.set_timing(True)
    docs()
    phases = {}
    for p, ms in phase_times(ctx):                # repeated names (refinement rounds) are summed
        phases[p] = round(phases.get(p, 0.0) + ms, 3)
    ctx.set_timing(False)
    ws = {}
    calls = {"build_lcp_dev": lambda f: f.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), s),
             "docs_build_dev": lambda f: f.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(starts), d_g.data_ptr(),
                                                          d_gl.data_ptr(), s)}
    for what, call in calls.items():
        fresh = _lib.Context(0)                   # workspace of one call on a fresh context
        call(fresh)
        torch.cuda.synchronize()
        ws[what] = round(fresh.stats()["workspace_bytes"] / n, 1)
        fresh.close()
    # |A| from SA and LCP of the concatenation
    st64 = d_s.long()
    sa = d_sa.long()
    ends = torch.cat([st64[1:], torch.tensor([n], device="cuda")])
    rem = ends[torch.searchsorted(st64, sa, right=True) - 1] - sa
    na = int((d_lcp.long() >= rem).sum())
    del sa, rem, ends, st64
    res = {"n": n, "docs": len(starts), "crossing_A": na,
           "docs_build_dev_ms_median": round(statistics.median(td), 3), "docs_build_dev_ms_all": [round(x, 3) for x in td],
           "build_lcp_dev_ms_median": round(statistics.median(tb), 3), "build_lcp_dev_ms_all": [round(x, 3) for x in tb],
           "overhead_ms": round(statistics.median(td) - statistics.median(tb), 3),
           "docs_phases_ms": phases, "workspace_bytes_per_text_byte": ws}
    if check:
        from tests import docs_check
        g = d_g.cpu().numpy().view(np.uint32)
        gl = d_gl.cpu().numpy().view(np.uint32)
        res["agree"] = docs_check.check(text, starts, g, gl) == 0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-check", action="store_true")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    n = a.n - a.n % 4
    t = gen.dna(n)
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": n}
    out["docs_1kB"] = run(ctx, stream, t, cut(n, 500, 1500, 1), a.reps, not a.no_check)
    out["docs_100kB"] = run(ctx, stream, t, cut(n, 50_000, 150_000, 2), a.reps, not a.no_check)
    acgt = np.tile(np.frombuffer(b"ACGT", np.uint8), n // 4)
    out["acgt_copies"] = run(ctx, stream, acgt, np.arange(0, n, 4, dtype=np.uint32), a.reps, not a.no_check)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
