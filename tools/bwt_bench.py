"""f-13: the Burrows-Wheeler transform and its inverse (b200sa_bwt_dev, b200sa_unbwt_dev) on device-resident
tables.  Prints one JSON line: card and power limit; per arm r, the median CUDA-event time (one warm-up, then
--reps) of the forward call (with r read back) and of the inverse call, the median of every phase of both,
the number of rulers, the longest walk and the rank rounds of the inverse (from its B200SA_TRACE line), the
workspace a context of its own grew to per text byte, the inverse's median at other ruler spacings
(B200SA_BWT_RULER), and agreement with the serial C statement of tests/bwt_check.c on one host core (forward
and inverse, their times recorded) and of the inverse with the text.

    python tools/bwt_bench.py [--n 100000000] [--reps 5] [--spacings 16 32 64 128 256]

Arms: G_dna, G_bytes and G_english (as bench.py), each as a single text and cut into documents of about
1 kB (seeded)."""
import argparse
import json
import os
import re
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.getcwd())
import numpy as np
import torch

from suffix_b200 import _lib, gen
from tests import bwt_check
from tools.docs_bench import card, cut, phase_times, timed
from tools.repeat_bench import agrees

FWD = ("bwt_check", "bwt_gather", "bwt_compact")
INV = ("unbwt_sort", "unbwt_walk", "unbwt_rank", "unbwt_emit")


def traced(fn):
    """Runs fn with B200SA_TRACE set and returns what the library wrote to stderr."""
    os.environ["B200SA_TRACE"] = "1"
    saved = os.dup(2)
    with tempfile.TemporaryFile() as tmp:
        os.dup2(tmp.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["B200SA_TRACE"]
        tmp.seek(0)
        return tmp.read().decode(errors="replace")


def median_phases(ctx, call, reps, names):
    ctx.set_timing(True)
    split = {p: [] for p in names}
    for _ in range(reps):
        call()
        for p, ms in phase_times(ctx):
            if p in split:
                split[p].append(ms)
    ctx.set_timing(False)
    return {p: round(statistics.median(v), 3) for p, v in split.items() if v}


def run_arm(build_ctx, stream, text, starts, reps, spacings):
    s, n = stream.cuda_stream, len(text)
    d_t = torch.from_numpy(text).cuda()
    d_sa = torch.empty(n, dtype=torch.int32, device="cuda")
    d_s = None
    if starts is None:
        build_ctx.build_dev(d_t.data_ptr(), n, d_sa.data_ptr(), s)
    else:
        d_s = torch.from_numpy(starts.view(np.int32).copy()).cuda()
        build_ctx.docs_build_dev(d_t.data_ptr(), n, d_s.data_ptr(), len(starts), d_sa.data_ptr(), 0, s)
    torch.cuda.synchronize()
    k = 1 if starts is None else len(starts)
    ctx = _lib.Context(0)                        # a context of its own: its workspace is this row's alone
    res = {"docs": k}
    d_b = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_term = torch.empty(k, dtype=torch.int32, device="cuda")
    fwd = lambda: ctx.bwt_dev(n, d_t.data_ptr(), d_sa.data_ptr(), 0 if d_s is None else d_s.data_ptr(),
                              0 if d_s is None else k, d_b.data_ptr(), d_term.data_ptr(), True, s)
    r = fwd()
    ts = [timed(stream, fwd) for _ in range(reps)]
    res["forward"] = {"r": r, "ms_median": round(statistics.median(ts), 3), "ms_all": [round(v, 3) for v in ts],
                      "phases_ms_median": median_phases(ctx, fwd, reps, FWD)}
    ws_fwd = ctx.stats()["workspace_bytes"]

    d_out = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_os = torch.empty(k, dtype=torch.int32, device="cuda")
    inv = lambda: ctx.unbwt_dev(n, k, d_b.data_ptr(), d_term.data_ptr(), d_out.data_ptr(), d_os.data_ptr(), s)
    line = traced(inv)
    m = re.search(r"rulers=(\d+) longest walk=(\d+) rank rounds=(\d+)", line)
    ts = [timed(stream, inv) for _ in range(reps)]
    res["inverse"] = {"ms_median": round(statistics.median(ts), 3), "ms_all": [round(v, 3) for v in ts],
                      "phases_ms_median": median_phases(ctx, inv, reps, INV),
                      "rulers": int(m.group(1)) if m else "not measured",
                      "longest_walk": int(m.group(2)) if m else "not measured",
                      "rank_rounds": int(m.group(3)) if m else "not measured"}
    res["workspace_bytes_per_text_byte"] = {"forward": round(ws_fwd / n, 3),
                                            "forward_and_inverse": round(ctx.stats()["workspace_bytes"] / n, 3)}
    sweep = {}
    for sp in spacings:
        os.environ["B200SA_BWT_RULER"] = str(sp)
        inv()
        sweep[str(sp)] = round(statistics.median([timed(stream, inv) for _ in range(3)]), 3)
        del os.environ["B200SA_BWT_RULER"]
    res["inverse"]["ms_median_by_spacing"] = sweep

    got_b, got_t = d_b.cpu().numpy().tobytes(), d_term.cpu().numpy().view(np.uint32).copy()
    inv()
    torch.cuda.synchronize()
    back = d_out.cpu().numpy()
    st = np.zeros(1, np.uint32) if starts is None else starts
    back_starts = d_os.cpu().numpy().view(np.uint32)
    sa = d_sa.cpu().numpy().view(np.uint32)
    t0 = time.perf_counter()
    wb, wt, wr = bwt_check.forward(text, sa, starts)
    t_fwd = time.perf_counter() - t0
    t0 = time.perf_counter()
    c_inv = bwt_check.inverse(wb, wt)
    t_inv = time.perf_counter() - t0
    res["serial_c_one_core_s"] = {"forward": round(t_fwd, 2), "inverse": round(t_inv, 2)}
    res["agree"] = bool(got_b == wb and np.array_equal(got_t, wt) and r == wr)
    res["agree_inverse"] = bool(np.array_equal(back, text) and np.array_equal(back_starts, st))
    res["agree_serial_inverse"] = bool(c_inv is not None and c_inv[0] == text.tobytes())
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--spacings", type=int, nargs="*", default=[16, 32, 64, 128, 256])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bwt_bench: no CUDA device")
    name, power = card()
    stream = torch.cuda.Stream()                 # a real stream: handle 0 means the library's own
    torch.cuda.set_stream(stream)
    ctx = _lib.Context(0)
    out = {"gpu": name, "power_limit": power, "n": a.n, "reps": a.reps}
    starts = cut(a.n, 500, 1500, 1)
    for arm, make in (("G_dna", lambda: gen.dna(a.n)), ("G_bytes", lambda: gen.rand_bytes(a.n)),
                      ("G_english", lambda: gen.english(a.n))):
        t = np.ascontiguousarray(make(), dtype=np.uint8)
        out[arm] = run_arm(ctx, stream, t, None, a.reps, a.spacings)
        torch.cuda.empty_cache()
        out[arm + "_documents_1kB"] = run_arm(ctx, stream, t, starts, a.reps, a.spacings)
        torch.cuda.empty_cache()
    out["agree"] = agrees({k: v for k, v in out.items() if isinstance(v, dict)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
