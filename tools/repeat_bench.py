"""f-11: repeat lengths, runs and duplicate spans (b200sa_repeat_lens_dev, b200sa_repeat_runs_dev,
b200sa_duplicate_spans_dev) on device-resident tables.  Prints one JSON line: card and power limit; per arm
and min_len the median CUDA-event time (one warm-up, then --reps) of the count call + the fetch call of every
mode, the phase split of one timed fetch, spans, covered bytes, the same for the runs with first / last, the
time of repeat_lens, the workspace a context of its own grew to per text byte, and agreement with two other
routes: the serial C statement of tests/repeats_check.c on one host core over the WHOLE arm, and for mode ANY
the same spans composed from torch ops on the device, timed in alternation with the library's two calls.

    python tools/repeat_bench.py [--n 100000000] [--reps 5]

Arms: G_dna (as bench.py) as a single text and cut into documents of about 1 kB; the same two with 10 % of
the documents overwritten by copies of earlier documents with 1 % substitutions (seeded); n/4 copies of ACGT
as a single text."""
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
from tests import repeats_check
from tools.docs_bench import card, cut, phase_times, timed

ALPHA = np.frombuffer(b"ACGT", dtype=np.uint8)
MODES = ("any", "earlier", "other_document", "earlier_document")


def plant(text, starts, rng, share=0.10, rate=0.01):
    """A copy of the text with `share` of the documents overwritten by an earlier document's head, `rate`
    of the copied bytes substituted.  Document lengths stay as they are."""
    out = text.copy()
    ends = np.append(starts[1:], len(text)).astype(np.int64)
    for k in rng.choice(np.arange(1, len(starts)), int(share * len(starts)), replace=False):
        j = int(rng.integers(0, k))
        m = int(min(ends[j] - starts[j], ends[k] - starts[k]))
        piece = text[int(starts[j]):int(starts[j]) + m].copy()
        sub = rng.random(m) < rate
        piece[sub] = rng.choice(ALPHA, int(sub.sum()))
        out[int(starts[k]):int(starts[k]) + m] = piece
    return out


def torch_any(d_sa, d_lcp, d_cut, L):
    """Mode ANY from torch ops: (begin, end) int64 tensors.  d_cut: bool[n + 1], True at document starts."""
    n = len(d_sa)
    nxt = torch.cat([d_lcp[1:], d_lcp.new_zeros(1)])
    flag = torch.zeros(n, dtype=torch.bool, device=d_sa.device)
    flag[d_sa.long()] = torch.maximum(d_lcp, nxt) >= L
    x = torch.arange(n, device=d_sa.device, dtype=torch.int32)
    near = torch.cummax(torch.where(flag, x + 1, torch.zeros_like(x)), 0).values
    cov = (near > 0) & (x - (near - 1) < L)
    pad = torch.cat([cov.new_zeros(1), cov, cov.new_zeros(1)])
    begin = torch.nonzero(cov & (~pad[:-2] | d_cut[:-1])).flatten()
    end = torch.nonzero(cov & (~pad[2:] | d_cut[1:])).flatten() + 1
    return begin, end


def run_arm(build_ctx, stream, text, starts, lens, reps):
    s, n = stream.cuda_stream, len(text)
    d_t = torch.from_numpy(text).cuda()
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lcp = torch.empty(n, dtype=torch.int32, device="cuda")
    d_s, nd = None, 0
    if starts is None:
        build_ctx.build_lcp_dev(d_t.data_ptr(), n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    else:
        d_s, nd = torch.from_numpy(starts.view(np.int32).copy()).cuda(), len(starts)
        build_ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), nd, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    torch.cuda.synchronize()
    del d_t
    sa, lcp = d_sa.cpu().numpy().view(np.uint32), d_lcp.cpu().numpy().view(np.uint32)
    d_cut = torch.zeros(n + 1, dtype=torch.bool, device="cuda")
    d_cut[0] = d_cut[n] = True
    if starts is not None:
        d_cut[d_s.long()] = True
    ctx = _lib.Context(0)                        # a context of its own: its workspace is the repeats' alone
    P = (n, d_sa.data_ptr(), d_lcp.data_ptr())
    res = {"docs": 1 if starts is None else nd}

    d_rl = torch.empty(n, dtype=torch.int32, device="cuda")
    rl = lambda: ctx.repeat_lens_dev(*P, d_rl.data_ptr(), s)
    rl()
    ts = [timed(stream, rl) for _ in range(reps)]
    want = np.zeros(n, dtype=np.uint32)
    want[sa] = np.maximum(lcp, np.append(lcp[1:], 0))
    res["repeat_lens"] = {"ms_median": round(statistics.median(ts), 3), "ms_all": [round(v, 3) for v in ts],
                          "agree": bool(np.array_equal(d_rl.cpu().numpy().view(np.uint32), want))}
    del d_rl, want
    ws = 0
    for L in lens:
        out = {}
        total = ctx.repeat_runs_dev(*P, L, stream=s)
        bufs = [torch.empty(max(total, 1), dtype=torch.int32, device="cuda") for _ in range(4)]

        def runs():                              # the protocol a caller follows: count, then fetch
            ctx.repeat_runs_dev(*P, L, stream=s)
            ctx.repeat_runs_dev(*P, L, *(b.data_ptr() for b in bufs), total, s)

        runs()
        ts = [timed(stream, runs) for _ in range(reps)]
        ctx.set_timing(True)
        ctx.repeat_runs_dev(*P, L, *(b.data_ptr() for b in bufs), total, s)
        phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
        ctx.set_timing(False)
        ws = max(ws, ctx.stats()["workspace_bytes"])
        t0 = time.perf_counter()
        cw = repeats_check.runs(sa, lcp, L)
        host = time.perf_counter() - t0
        out["runs"] = {"runs": total, "count_plus_fetch_ms_median": round(statistics.median(ts), 3),
                       "count_plus_fetch_ms_all": [round(v, 3) for v in ts], "fetch_phases_ms": phases,
                       "serial_c_one_core_s": round(host, 2),
                       "agree": total == len(cw[0]) and all(np.array_equal(b[:total].cpu().numpy().view(np.uint32), w)
                                                            for b, w in zip(bufs, cw))}
        del bufs
        for mode, name in enumerate(MODES[:2 if starts is None else 4]):
            A = P + (d_s.data_ptr() if nd else 0, nd, L, mode)
            total, covered = ctx.duplicate_spans_dev(*A, stream=s)
            b, e = (torch.empty(max(total, 1), dtype=torch.int32, device="cuda") for _ in range(2))

            def spans():
                ctx.duplicate_spans_dev(*A, stream=s)
                ctx.duplicate_spans_dev(*A, b.data_ptr(), e.data_ptr(), total, s)

            spans()
            ts, tt = [], []
            for _ in range(reps):                # alternated, so both see the same card state
                ts.append(timed(stream, spans))
                if mode == 0:
                    tt.append(timed(stream, lambda: torch_any(d_sa, d_lcp, d_cut, L)))
            ctx.set_timing(True)
            ctx.duplicate_spans_dev(*A, b.data_ptr(), e.data_ptr(), total, s)
            phases = {p: round(ms, 3) for p, ms in phase_times(ctx)}
            ctx.set_timing(False)
            ws = max(ws, ctx.stats()["workspace_bytes"])
            t0 = time.perf_counter()
            wb, we, wcov = repeats_check.spans(sa, lcp, starts, L, mode)
            host = time.perf_counter() - t0
            hb, he = (t[:total].cpu().numpy().view(np.uint32) for t in (b, e))
            r = {"spans": total, "covered_bytes": covered, "count_plus_fetch_ms_median": round(statistics.median(ts), 3),
                 "count_plus_fetch_ms_all": [round(v, 3) for v in ts], "fetch_phases_ms": phases,
                 "serial_c_one_core_s": round(host, 2),
                 "agree": (total, covered) == (len(wb), wcov) and np.array_equal(hb, wb) and np.array_equal(he, we)}
            if mode == 0:
                tb, te = torch_any(d_sa, d_lcp, d_cut, L)
                r["torch_ops_ms_median"] = round(statistics.median(tt), 3)
                r["torch_ops_ms_all"] = [round(v, 3) for v in tt]
                r["agree_torch_ops"] = bool(len(tb) == total and torch.equal(tb.int(), b[:total]) and
                                            torch.equal(te.int(), e[:total]))
                del tb, te
            out[name] = r
            del b, e
        res["min_len_%d" % L] = out
    res["workspace_bytes_per_text_byte"] = round(ws / n, 3)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    torch_any(d_sa, d_lcp, d_cut, lens[0])
    res["torch_ops_peak_bytes_per_text_byte"] = round((torch.cuda.max_memory_allocated() - base) / n, 2)
    ctx.close()
    return res


def agrees(v):
    if isinstance(v, dict):
        return all(agrees(x) for k, x in v.items() if isinstance(x, dict) or k.startswith("agree"))
    return bool(v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--lens", type=int, nargs="+", default=[12, 20, 50])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("repeat_bench: no CUDA device")
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    text = gen.dna(a.n)
    starts = cut(a.n, 500, 1500, 1)
    planted = plant(text, starts, np.random.default_rng(2))
    acgt = np.tile(ALPHA, a.n // 4)
    out = {"gpu": name, "power_limit": power, "text": "G_dna", "n": a.n, "reps": a.reps}
    for arm, (t, st) in (("text", (text, None)), ("documents_1kB", (text, starts)), ("planted_text", (planted, None)),
                         ("planted_documents_1kB", (planted, starts)), ("acgt_copies_text", (acgt, None))):
        out[arm] = run_arm(ctx, stream, t, st, a.lens, a.reps)
        torch.cuda.empty_cache()
    out["agree"] = agrees({k: v for k, v in out.items() if isinstance(v, dict)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
