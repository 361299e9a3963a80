"""Every C-ABI entry point that takes a context leaves its own message in b200sa_last_error when it
rejects its arguments, never the message of an earlier failing call, and the context stays usable."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from suffix_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD_ARG = -1
STALE = "doc_starts rejected: doc_starts[0] != 0;"

# Declared entry points with no case below, and why.
EXCLUDED = {
    "b200sa_ctx_destroy": "returns nothing",
    "b200sa_last_error": "reports the previous call's error and has none of its own",
    "b200sa_set_timing": "accepts every value on a valid context",
    "b200sa_last_phase_times": "accepts every value on a valid context",
    "b200sa_comm_destroy": "accepts every valid context",
}


def _u64():
    return ctypes.byref(ctypes.c_uint64(0))


def _cases(p):
    """name -> (call(L, h), expected code, a substring of the expected message).  p is a device pointer;
    None is the argument being rejected.  Every case is rejected on the host before any launch."""
    host = ctypes.create_string_buffer(64)
    return {
        "b200sa_build": (lambda L, h: L.b200sa_build(h, None, 8, None), BAD_ARG, "null"),
        "b200sa_lcp": (lambda L, h: L.b200sa_lcp(h, None, 8, None, None), BAD_ARG, "null"),
        "b200sa_build_lcp": (lambda L, h: L.b200sa_build_lcp(h, None, 8, None, None), BAD_ARG, "null"),
        "b200sa_build_dev": (lambda L, h: L.b200sa_build_dev(h, None, 8, None, None), BAD_ARG, "null"),
        "b200sa_lcp_dev": (lambda L, h: L.b200sa_lcp_dev(h, None, 8, None, None, None), BAD_ARG, "null"),
        "b200sa_build_lcp_dev": (lambda L, h: L.b200sa_build_lcp_dev(h, None, 8, None, None, None), BAD_ARG, "null"),
        "b200sa_positions_dev": (lambda L, h: L.b200sa_positions_dev(h, p, 8, p, p, None, 1, p, p, None), BAD_ARG,
                                 "null"),
        "b200sa_shard_summary": (lambda L, h: L.b200sa_shard_summary(h, None, 8, -1, ctypes.byref(ctypes.c_int(0)),
                                                                     None), BAD_ARG, "null"),
        "b200sa_shard_classify": (lambda L, h: L.b200sa_shard_classify(h, None, 8, -1, -1, 0, None, None, None, 0,
                                                                       None, None, None), BAD_ARG, "null"),
        "b200sa_doc_ids_dev": (lambda L, h: L.b200sa_doc_ids_dev(h, p, 4, None, 1, p, p, None), BAD_ARG, "null"),
        "b200sa_lcp_intervals_dev": (lambda L, h: L.b200sa_lcp_intervals_dev(h, None, 8, p, p, None), BAD_ARG, "null"),
        "b200sa_suffix_tree_dev": (lambda L, h: L.b200sa_suffix_tree_dev(h, 8, p, p, None, 16, _u64(), None), BAD_ARG,
                                   "null"),
        "b200sa_suffix_tree": (lambda L, h: L.b200sa_suffix_tree(h, 8, None, None, None, 16, _u64()), BAD_ARG, "null"),
        "b200sa_docs_build": (lambda L, h: L.b200sa_docs_build(h, None, 8, None, 1, None, None), BAD_ARG, "null"),
        "b200sa_docs_build_dev": (lambda L, h: L.b200sa_docs_build_dev(h, None, 8, None, 1, None, None, None), BAD_ARG,
                                  "null"),
        "b200sa_docs_positions_dev": (lambda L, h: L.b200sa_docs_positions_dev(h, p, 8, p, p, 0, p, p, 1, p, p, None),
                                      BAD_ARG, "ndocs == 0"),
        "b200sa_docs_tree_dev": (lambda L, h: L.b200sa_docs_tree_dev(h, 8, p, p, p, 1, None, 16, _u64(), None),
                                 BAD_ARG, "null"),
        "b200sa_docs_tree": (lambda L, h: L.b200sa_docs_tree(h, 8, None, None, None, 1, None, 16, _u64()), BAD_ARG,
                             "null"),
        "b200sa_docs_tree_counts_dev": (lambda L, h: L.b200sa_docs_tree_counts_dev(h, None, None, None, 1, None, None,
                                                                                   1, None, None), BAD_ARG, "null"),
        "b200sa_docs_list_index_dev": (lambda L, h: L.b200sa_docs_list_index_dev(h, 8, None, None, 1, None, None,
                                                                                 None), BAD_ARG, "null"),
        "b200sa_docs_list_dev": (lambda L, h: L.b200sa_docs_list_dev(h, 8, p, p, 1, p, p, p, p, 1, None, p, p, 0,
                                                                     _u64(), None), BAD_ARG, "null"),
        "b200sa_docs_topk_dev": (lambda L, h: L.b200sa_docs_topk_dev(h, 8, p, p, 1, p, p, p, p, 1, 0, p, p, p, None),
                                 BAD_ARG, "k must be"),
        "b200sa_match_stats_dev": (lambda L, h: L.b200sa_match_stats_dev(h, None, 8, None, None, None, None, 0, 0,
                                                                         None, None, None, None), BAD_ARG, "null"),
        "b200sa_docs_match_stats_dev": (lambda L, h: L.b200sa_docs_match_stats_dev(h, None, 8, None, None, None, 0,
                                                                                   None, None, 0, 0, None, None, None,
                                                                                   None), BAD_ARG, "null"),
        "b200sa_smems_dev": (lambda L, h: L.b200sa_smems_dev(h, p, 1, 8, p, 0, p, p, 0, _u64(), None), BAD_ARG,
                             "min_len"),
        "b200sa_repeat_lens_dev": (lambda L, h: L.b200sa_repeat_lens_dev(h, 8, None, None, None, None), BAD_ARG,
                                   "null"),
        "b200sa_repeat_runs_dev": (lambda L, h: L.b200sa_repeat_runs_dev(h, 8, p, p, 0, None, None, None, None, 0,
                                                                         _u64(), None), BAD_ARG, "min_len"),
        "b200sa_duplicate_spans_dev": (lambda L, h: L.b200sa_duplicate_spans_dev(h, 8, p, p, None, 0, 1, 99, None,
                                                                                 None, 0, _u64(), _u64(), None),
                                       BAD_ARG, "unknown mode"),
        "b200sa_lpf_dev": (lambda L, h: L.b200sa_lpf_dev(h, 8, None, None, None, None, None), BAD_ARG, "null"),
        "b200sa_lz77_dev": (lambda L, h: L.b200sa_lz77_dev(h, 8, None, None, None, None, None, 0, _u64(), None),
                            BAD_ARG, "null"),
        "b200sa_bwt_dev": (lambda L, h: L.b200sa_bwt_dev(h, 8, None, None, None, 0, None, None, None, None), BAD_ARG,
                           "null"),
        "b200sa_unbwt_dev": (lambda L, h: L.b200sa_unbwt_dev(h, 8, 0, p, p, p, None, None), BAD_ARG, "ndocs"),
        "b200sa_approx_positions_dev": (lambda L, h: L.b200sa_approx_positions_dev(h, p, 8, p, p, p, 1, 99, p, p, None,
                                                                                   0, _u64(), None), BAD_ARG,
                                        "APPROX_MAX_K"),
        "b200sa_docs_approx_positions_dev": (lambda L, h: L.b200sa_docs_approx_positions_dev(
            h, p, 8, p, None, 1, p, p, 1, 0, p, p, None, 0, _u64(), None), BAD_ARG, "null"),
        "b200sa_comm_init": (lambda L, h: L.b200sa_comm_init(h, 0, 0, None), BAD_ARG, "null"),
        "b200sa_comm_attach": (lambda L, h: L.b200sa_comm_attach(h, None), BAD_ARG, "null"),
        "b200sa_shard_lms_sort": (lambda L, h: L.b200sa_shard_lms_sort(h, None, 8, None, None, 0, None, None),
                                  BAD_ARG, "null"),
        "b200sa_lcp_sharded": (lambda L, h: L.b200sa_lcp_sharded(h, None, 8, None, None, 0, None), BAD_ARG, "null"),
        "b200sa_last_stats": (lambda L, h: L.b200sa_last_stats(h, None), BAD_ARG, "null"),
        "b200sa_test_classify_fused": (lambda L, h: L.b200sa_test_classify_fused(h, None, 8, None, None, None, None, 0,
                                                                                 None), BAD_ARG, "null"),
        "b200sa_test_scan": (lambda L, h: L.b200sa_test_scan(h, None, 8, 0, None, None), BAD_ARG, "null"),
        "b200sa_test_sort_pairs32": (lambda L, h: L.b200sa_test_sort_pairs32(h, None, None, 8, 32), BAD_ARG, "null"),
        "b200sa_test_sort_pairs64": (lambda L, h: L.b200sa_test_sort_pairs64(h, None, None, 8, 64), BAD_ARG, "null"),
        "b200sa_test_reduced_sa": (lambda L, h: L.b200sa_test_reduced_sa(h, None, 8, 1, None, None), BAD_ARG, "null"),
        "b200sa_debug_fetch": (lambda L, h: L.b200sa_debug_fetch(h, 99, ctypes.addressof(host), 1), BAD_ARG,
                               "unknown"),
    }


def _declared_with_context():
    names = set()
    for h in os.listdir(os.path.join(ROOT, "include")):
        if h.endswith(".h"):
            src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", h)).read(), flags=re.S)
            names |= set(re.findall(r"\b(b200sa_[a-z0-9_]+)\s*\(\s*b200sa_ctx\s*\*", src))
    return names


def test_every_entry_point_has_a_case():
    cases = set(_cases(0))
    declared = _declared_with_context()
    assert len(declared) >= 45
    assert sorted(declared - cases - set(EXCLUDED)) == []
    assert sorted((cases | set(EXCLUDED)) - declared) == []


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0)
    yield c
    c.close()


def _fail_with_stale(L, h):
    text = np.frombuffer(b"abab", np.uint8)
    starts = np.array([1], np.uint32)
    gsa = np.empty(4, np.uint32)
    assert L.b200sa_docs_build(h, text.ctypes.data, 4, starts.ctypes.data, 1, gsa.ctypes.data, None) == BAD_ARG
    assert L.b200sa_last_error(h).decode() == STALE


def _valid_build(L, h):
    text = np.frombuffer(b"mississippi", np.uint8)
    sa = np.empty(len(text), np.uint32)
    assert L.b200sa_build(h, text.ctypes.data, len(text), sa.ctypes.data) == 0, L.b200sa_last_error(h)
    return sa.tolist()


@pytest.mark.parametrize("name", sorted(_cases(0)))
def test_argument_error_leaves_its_own_message(ctx, name):
    L, h = _lib.lib(), ctx._h
    want = _valid_build(L, h)
    assert want == [10, 7, 4, 1, 0, 9, 8, 6, 3, 5, 2]
    dev = torch.zeros(1024, dtype=torch.int32, device="cuda")
    call, code, part = _cases(dev.data_ptr())[name]
    _fail_with_stale(L, h)
    assert call(L, h) == code
    msg = L.b200sa_last_error(h).decode()
    assert msg and msg != STALE and part in msg, msg
    assert _valid_build(L, h) == want
