"""Per-kernel device time of the LMS-suffix sort on the bench text (100 MB G_dna, SA + LCP,
device-resident) from torch.profiler with CUDA activities.  Diagnostic; run on its own (the
tracer slows the host).  Prints one JSON line: the card, its power limit, and the mean time per
step of every kernel and memset of the step, sorted by time, plus the sum over the LMS sort's
kernels.  `--env NAME=VALUE` sets a library switch first (e.g. B200SA_LMS_SORT4=1)."""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from suffix_b200 import _lib, gen  # noqa: E402

# kernels of the LMS sort and of the round-1 tie finding (both paths)
LMS_KERNELS = ("k_os_hist", "k_os_scan", "k_os_pass", "k_lms_mark_trunc", "k_lms_groups1", "k_scan_lb",
               "k_lms_bucket_sort", "Memset")


def short_name(name):
    """'void b200sa::k_os_pass<unsigned int, ...>(...)' -> 'k_os_pass'."""
    s = re.sub(r"<.*", "", name)
    s = re.sub(r"\(.*", "", s)
    s = s.split("::")[-1].replace("void ", "").strip()
    return s or name


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
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
    ctx = _lib.Context(0)
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        ctx.build_lcp_dev(d_text.data_ptr(), a.n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            ctx.build_lcp_dev(d_text.data_ptr(), a.n, d_sa.data_ptr(), d_lcp.data_ptr(), s)
        torch.cuda.synchronize()
    per = {}
    calls = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        nm = short_name(ev.name)
        if nm.startswith("Memset") or "memset" in nm.lower():
            nm = "Memset"
        per[nm] = per.get(nm, 0.0) + ev.time_range.elapsed_us() / 1e3      # us -> ms
        calls[nm] = calls.get(nm, 0) + 1
    rows = sorted(((k, v / a.steps, calls[k] / a.steps) for k, v in per.items()), key=lambda r: -r[1])
    kern = {k: {"ms": round(ms, 4), "calls": round(c, 2)} for k, ms, c in rows}
    lms = sum(ms for k, ms, _ in rows if k in LMS_KERNELS and k != "Memset")
    out = {"card": card(), "n": a.n, "steps": a.steps, "env": a.env, "stats": ctx.stats(),
           "lms_sort_kernels_ms": round(lms, 4), "kernels_ms_per_step": kern,
           "note": "device time per step from torch.profiler CUDA activities; Memset = all memsets of the step; "
                   "k_scan_lb also serves other phases"}
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
