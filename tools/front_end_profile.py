"""Per-kernel device time of the front of the SA + LCP build on the bench text (100 MB G_dna,
device-resident): everything from the start of a build up to the first one-sweep pass of the LMS
sort -- the classification phase (alphabet, classifier, histogram fold, bucket tables, packing),
the host read of m and sigma, and the key gathering of the LMS sort (`k_os_hist`).  torch.profiler
with CUDA activities, in a run of its own (the tracer slows the host).

A one-element add on the build's stream marks the start of every step, so the window of a step is
the events between its marker and its first `k_os_pass`.  Prints one JSON line: the card, its power
limit, the mean time per step of every kernel and memset of the window, the idle time between them
(split into the gap after the device-to-host copy of m and sigma -- the host read -- and the rest)
and the window's length.  `--env NAME=VALUE` sets a library switch first."""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from suffix_b200 import _lib, gen  # noqa: E402

# the kernels whose sum bounds what classifying from the packed text can save
FRONT_KERNELS = ("k_classify_fused", "k_classify_packed", "k_pack", "k_os_hist")


def short_name(name):
    """'void b200sa::k_os_pass<unsigned int, ...>(...)' -> 'k_os_pass'."""
    s = re.sub(r"<.*", "", name)
    s = re.sub(r"\(.*", "", s)
    s = s.split("::")[-1].replace("void ", "").strip()
    if "memset" in name.lower():
        return "Memset"
    return s or name


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--env", action="append", default=[])
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    for kv in a.env:
        k, _, v = kv.partition("=")
        os.environ[k] = v
    dev = torch.device("cuda:0")
    text = gen.dna(a.n, seed=gen.SEED_DNA)
    d_text = torch.from_numpy(text).to(dev)
    d_sa = torch.empty(a.n, dtype=torch.int32, device=dev)
    d_lcp = torch.empty(a.n, dtype=torch.int32, device=dev)
    marker = torch.zeros(1, dtype=torch.int32, device=dev)
    ctx = _lib.Context(0)
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        marker.add_(1)
        ctx.build_lcp_dev(d_text.data_ptr(), a.n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            marker.add_(1)
            ctx.build_lcp_dev(d_text.data_ptr(), a.n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
        torch.cuda.synchronize()
    evs = sorted(((ev.time_range.start, ev.time_range.end, ev.name) for ev in prof.events()
                  if ev.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e[0])
    per, calls = {}, {}
    host_gap = other_gap = window = 0.0
    steps = 0
    i = 0
    while i < len(evs):
        if "elementwise" not in evs[i][2]:            # the step marker (torch's add kernel)
            i += 1
            continue
        t0, prev_end, prev_name = evs[i][1], evs[i][1], "marker"
        j = i + 1
        while j < len(evs) and short_name(evs[j][2]) != "k_os_pass":
            st, en, nm = evs[j]
            nm = short_name(nm)
            per[nm] = per.get(nm, 0.0) + (en - st)
            calls[nm] = calls.get(nm, 0) + 1
            gap = max(0.0, st - prev_end)
            if prev_name.startswith("Memcpy DtoH"):
                host_gap += gap
            else:
                other_gap += gap
            prev_end, prev_name = max(prev_end, en), nm
            j += 1
        if j < len(evs):
            window += evs[j][0] - t0
            other_gap += max(0.0, evs[j][0] - prev_end)
            steps += 1
        i = j
    if steps == 0:
        raise SystemExit("no step found in the trace")
    us = 1e3 * steps                                   # us per run -> ms per step
    rows = sorted(per.items(), key=lambda r: -r[1])
    kern = {k: {"ms": round(v / us, 4), "calls": round(calls[k] / steps, 2)} for k, v in rows}
    front = sum(v for k, v in per.items() if k in FRONT_KERNELS) / us
    out = {"card": card(), "n": a.n, "steps": steps, "env": a.env, "m": ctx.stats().get("m"),
           "window_ms": round(window / us, 4), "host_read_gap_ms": round(host_gap / us, 4),
           "other_gaps_ms": round(other_gap / us, 4), "front_kernels_ms": round(front, 4),
           "kernels_ms_per_step": kern,
           "note": "device time per step from torch.profiler CUDA activities, from the start of a build to its "
                   "first k_os_pass; front_kernels_ms = " + " + ".join(FRONT_KERNELS)}
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
