"""The Burrows-Wheeler transform over a device-resident table, and its inverse: the part SuffixTable and
DocumentSuffixTable share.  A table supplies `_device` and `_bwt_arrays()` -> (d_text, d_table,
d_doc_starts or None, ndocs), its text and table on the device; the LCP array is not needed."""
import numpy as np

from . import _lib
from .table import _as_bytes, _lock

MAX_N = 0xFFFFF000        # B200SA_MAX_N
BAD_ARG = -1


def _transform(table, runs):
    """(bwt bytes, term_rows u32[k], r or None)."""
    import torch
    d_t, d_r, d_s, ndocs = table._bwt_arrays()
    n, k = len(table), (1 if d_s is None else ndocs)
    if k == 0:                                    # no documents: no rows
        return b"", np.zeros(0, dtype=np.uint32), 0
    dev = torch.device("cuda", table._device)
    bwt = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    term = torch.empty(k, dtype=torch.int32, device=dev)
    with _lock:
        r = _lib.default_context(table._device).bwt_dev(
            n, d_t.data_ptr(), d_r.data_ptr(), 0 if d_s is None else d_s.data_ptr(), 0 if d_s is None else ndocs,
            bwt.data_ptr(), term.data_ptr(), runs, torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize(dev)
    return bwt[:n].cpu().numpy().tobytes(), term.cpu().numpy().view(np.uint32), r


def bwt(table):
    b, term, _ = _transform(table, False)
    return b, term


def bwt_runs(table):
    return _transform(table, True)[2]


def inverse_bwt_documents(bwt, term_rows, *, device=0):
    """The documents whose transform is (bwt, term_rows), as a list of bytes (b200sa_unbwt_dev).  Raises
    B200SAError when no documents have that transform."""
    import torch
    b = _as_bytes(bwt)
    t = np.asarray(term_rows, dtype=np.int64).reshape(-1)
    if len(t) and (t.min() < 0 or t.max() > 0xFFFFFFFF):
        raise _lib.B200SAError(BAD_ARG, "term rows out of range")
    n, k = len(b), len(t)
    dev = torch.device("cuda", device)
    d_b = torch.from_numpy(np.frombuffer(b or b"\0", dtype=np.uint8).copy()).to(dev)
    d_t = torch.from_numpy(t.astype(np.uint32).view(np.int32) if k else np.zeros(1, np.int32)).to(dev)
    out = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    starts = torch.empty(max(k, 1), dtype=torch.int32, device=dev)
    with _lock:
        _lib.default_context(device).unbwt_dev(n, k, d_b.data_ptr(), d_t.data_ptr(), out.data_ptr(),
                                               starts.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    text = out[:n].cpu().numpy().tobytes()
    ends = np.append(starts[:k].cpu().numpy().view(np.uint32)[1:], n).astype(np.int64)
    begins = starts[:k].cpu().numpy().view(np.uint32).astype(np.int64)
    return [text[s:e] for s, e in zip(begins.tolist(), ends.tolist())]


def inverse_bwt(bwt, primary, *, device=0):
    """The text whose transform is (bwt, primary), primary = the row of the terminator (1 + the rank of
    position 0).  Raises B200SAError when no text has that transform."""
    return inverse_bwt_documents(bwt, [int(primary)], device=device)[0]
