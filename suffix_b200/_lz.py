"""Longest previous factors and the LZ77 factorization over a device-resident table: the part SuffixTable
and DocumentSuffixTable share.  A table supplies `_device` and `_repeat_arrays()` -> (d_table, d_lcp,
d_doc_starts or None, ndocs), its arrays on the device; doc_starts is not needed here."""
import numpy as np

from . import _lib
from .table import _lock


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _setup(table):
    import torch
    d_r, d_lcp, _, _ = table._repeat_arrays()
    dev = torch.device("cuda", table._device)
    return torch, dev, _lib.default_context(table._device), torch.cuda.current_stream(dev).cuda_stream, len(table), \
        d_r, d_lcp


def longest_previous_factors(table):
    torch, dev, ctx, stream, n, d_r, d_lcp = _setup(table)
    lpf, src = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
    if n:
        with _lock:
            ctx.lpf_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), lpf.data_ptr(), src.data_ptr(), stream)
        torch.cuda.synchronize(dev)
    return _host(lpf), _host(src)


def lz77_count(table):
    torch, dev, ctx, stream, n, d_r, d_lcp = _setup(table)
    if not n:
        return 0
    with _lock:
        return ctx.lz77_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), stream=stream)


def lz77_factors(table, cap_guess=None):
    """(start, length, source) u32[z].  One call into buffers of cap_guess factors (default n/8 + 4096,
    at most n); a second one, sized to z, only when that was short."""
    torch, dev, ctx, stream, n, d_r, d_lcp = _setup(table)
    cap = min(n, n // 8 + 4096) if cap_guess is None else int(cap_guess)

    def call(cap):
        out = [torch.empty(max(cap, 1), dtype=torch.int32, device=dev) for _ in range(3)]
        with _lock:
            z = ctx.lz77_dev(n, d_r.data_ptr(), d_lcp.data_ptr(), *(o.data_ptr() if cap else 0 for o in out), cap,
                             stream) if n else 0
        return z, out

    z, out = call(cap)
    if z > cap:
        z, out = call(z)
    return tuple(_host(o[:z]) for o in out)
