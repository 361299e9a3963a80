"""A/B of the LMS-suffix sort on the bench workload (100 MB G_dna, SA + LCP, device-resident):
in one process on one card, alternates the four-pass sort (B200SA_LMS_SORT4=1, arm "sort4") with the
default two passes + k_lms_bucket_sort (arm "bucket"), `--pairs` times `--steps` timed steps per arm.
Prints one JSON line: the card and its power limit, per arm the median / min / max step time over the
repeats (CUDA events around the steps) and the mean per-phase times, and whether both arms built the
same SA and LCP."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from suffix_b200 import _lib, gen  # noqa: E402

ARMS = {"sort4": "1", "bucket": None}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def set_arm(arm):
    if ARMS[arm] is None:
        os.environ.pop("B200SA_LMS_SORT4", None)
    else:
        os.environ["B200SA_LMS_SORT4"] = ARMS[arm]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--pairs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    text = gen.dna(a.n, seed=gen.SEED_DNA)
    d_text = torch.from_numpy(text).to(dev)
    d_sa = torch.empty(a.n, dtype=torch.int32, device=dev)
    d_lcp = torch.empty(a.n, dtype=torch.int32, device=dev)
    ctx = _lib.Context(0)
    ctx.set_timing(True)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream

    def step():
        ctx.build_lcp_dev(d_text.data_ptr(), a.n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
        return ctx.phase_times()

    res = {arm: {"ms": [], "phases": {}} for arm in ARMS}
    out = {}
    for arm in ARMS:                      # warm-up of both arms, and the results to compare
        set_arm(arm)
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        out[arm] = (d_sa.clone(), d_lcp.clone())
    for _ in range(a.pairs):
        for arm in ARMS:
            set_arm(arm)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                for k, v in step():
                    res[arm]["phases"].setdefault(k, []).append(v)
            e1.record(stream)
            torch.cuda.synchronize()
            res[arm]["ms"].append(e0.elapsed_time(e1) / a.steps)
    set_arm("bucket")
    same = bool(torch.equal(out["sort4"][0], out["bucket"][0]) and torch.equal(out["sort4"][1], out["bucket"][1]))
    report = {"card": card(), "n": a.n, "pairs": a.pairs, "steps": a.steps, "same_sa_lcp": same, "arms": {}}
    for arm, r in res.items():
        med = statistics.median(r["ms"])
        report["arms"][arm] = {"median_ms": round(med, 4), "min_ms": round(min(r["ms"]), 4), "max_ms": round(max(r["ms"]), 4),
                               "spread_pct": round(100 * (max(r["ms"]) - min(r["ms"])) / med, 2),
                               "MBps": round(a.n / 1e6 / (med / 1e3), 1),
                               "phase_ms": {k: round(statistics.mean(v), 4) for k, v in r["phases"].items()}}
    b, f = report["arms"]["bucket"]["median_ms"], report["arms"]["sort4"]["median_ms"]
    report["gain_pct"] = round(100 * (f - b) / f, 2)
    print(json.dumps(report), flush=True)


if __name__ == "__main__":
    main()
