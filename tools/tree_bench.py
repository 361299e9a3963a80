"""f-5: suffix tree from a device-resident SA + LCP (b200sa_suffix_tree_dev).
Prints one JSON line: card and power limit, n, N and the internal nodes, the tree-stage time
(CUDA events, one warm-up, median of --reps) with its phase split, the b200sa_build_lcp_dev
time of the same run for scale, and the single-core time of the C restatement of the
reference's insertion loop (tests/tree_oracle.c) with whether its arrays agree.

    python tools/tree_bench.py [--n 100000000] [--reps 5] [--no-oracle] [--max-n]

--max-n instead builds the tree of a^n (SA and LCP made on the device) for growing n to find
the largest n whose tree workspace fits next to its inputs and outputs."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen

FIELDS = _lib.TREE_FIELDS


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
    r = fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def max_n(stream):
    out = []
    for n in (1 << 28, 3 << 27, 1 << 29, 5 << 27, 3 << 28):
        ctx = _lib.Context(0)
        try:
            d_sa = torch.arange(n - 1, -1, -1, dtype=torch.int32, device="cuda")      # a^n: sa = n-1..0
            d_lcp = torch.arange(0, n, dtype=torch.int32, device="cuda")              # lcp = 0..n-1
            outs = [torch.empty(2 * n, dtype=torch.int32, device="cuda") for _ in FIELDS]
            ms, N = timed(stream, lambda: ctx.suffix_tree_dev(n, d_sa.data_ptr(), d_lcp.data_ptr(),
                                                              [o.data_ptr() for o in outs], 2 * n, stream.cuda_stream))
            ok = N == n + 1
            out.append({"n": n, "ok": bool(ok), "ms": round(ms, 1),
                        "workspace_bytes": ctx.stats()["workspace_bytes"],
                        "peak_allocated_by_torch": torch.cuda.max_memory_allocated()})
        except (_lib.B200SAError, torch.cuda.OutOfMemoryError) as e:
            out.append({"n": n, "error": str(e)[:120]})
            break
        finally:
            d_sa = d_lcp = outs = None
            ctx.close()
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--max-n", action="store_true")
    a = ap.parse_args()
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    if a.max_n:
        print(json.dumps({"gpu": name, "power_limit": power, "max_n": max_n(stream)}))
        return
    ctx = _lib.Context(0)
    n = a.n
    t = gen.dna(n)
    d_t = torch.from_numpy(t).cuda()
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
    build = lambda: ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), stream.cuda_stream)
    build()
    build_ms, _ = timed(stream, build)
    cap = max(1, 2 * n)
    outs = [torch.empty(cap, dtype=torch.int32, device="cuda") for _ in FIELDS]
    tree = lambda: ctx.suffix_tree_dev(n, d_sa.data_ptr(), d_lcp.data_ptr(), [o.data_ptr() for o in outs], cap,
                                       stream.cuda_stream)
    tree()                                       # warm-up
    times = []
    for _ in range(a.reps):
        ms, N = timed(stream, tree)
        times.append(ms)
    ctx.set_timing(True)
    tree()
    phases = {p: round(ms, 3) for p, ms in ctx.phase_times()}
    ctx.set_timing(False)
    got = {f: o[:N].cpu().numpy().view(np.uint32) for f, o in zip(FIELDS, outs)}
    internal = int(np.count_nonzero(got["sa_hi"][1:] - got["sa_lo"][1:] > 1))   # leaves span one rank
    res = {"gpu": name, "power_limit": power, "text": "G_dna", "n": n, "nodes": int(N),
           "internal_nodes": internal, "tree_ms_median": round(statistics.median(times), 3),
           "tree_ms_all": [round(x, 3) for x in times], "tree_phases_ms": phases,
           "build_lcp_dev_ms": round(build_ms, 3)}
    if not a.no_oracle:
        from tests import tree_oracle
        sa = d_sa.cpu().numpy().view(np.uint32)
        lcp = d_lcp.cpu().numpy().view(np.uint32)
        t0 = time.perf_counter()
        want = tree_oracle.suffix_tree(sa, lcp)
        res["oracle_c_tree_ms_1core"] = round((time.perf_counter() - t0) * 1e3, 1)
        lens = tree_oracle.label_lengths(want)
        res["agree"] = bool(all(np.array_equal(got[f], want[f]) for f in FIELDS) and
                            tree_oracle.labels_differ(t, got["label_start"], want["own_start"], lens) == -1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
