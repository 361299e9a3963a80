"""ctypes loader for libb200sa.so.  There is no CPU fallback: if the CUDA
library is missing or no device is usable, every call raises."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200SA_LIB") or os.path.join(_HERE, "libb200sa.so")


class B200SAError(RuntimeError):
    def __init__(self, code, detail=""):
        self.code = code
        super().__init__("b200sa error %d (%s)%s" % (code, strerror(code), (": " + detail) if detail else ""))


class Stats(ctypes.Structure):
    _fields_ = [("n", ctypes.c_uint64), ("m", ctypes.c_uint64), ("names", ctypes.c_uint64),
                ("doubling_rounds", ctypes.c_uint32), ("kernel_launches", ctypes.c_uint32),
                ("induce_blocks", ctypes.c_uint32), ("sm_count", ctypes.c_uint32),
                ("workspace_bytes", ctypes.c_uint64), ("direct_sort", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class ShardStats(ctypes.Structure):
    _fields_ = [("n_total", ctypes.c_uint64), ("m_total", ctypes.c_uint64), ("m_local", ctypes.c_uint64),
                ("lo", ctypes.c_uint64), ("recv_count", ctypes.c_uint64), ("distinct_local", ctypes.c_uint64),
                ("name_offset", ctypes.c_uint64), ("ties_total", ctypes.c_uint64),
                ("bytes_sent", ctypes.c_double), ("bytes_recv", ctypes.c_double),
                ("kc", ctypes.c_uint32), ("nranks", ctypes.c_uint32), ("rank", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class Tree(ctypes.Structure):
    """b200sa_tree: six u32 arrays indexed by preorder id."""
    _fields_ = [(f, ctypes.c_void_p) for f in ("parent", "depth", "sa_lo", "sa_hi", "label_start", "subtree_end")]


TREE_FIELDS = tuple(f for f, _ in Tree._fields_)


class DocsTree(ctypes.Structure):
    """b200sa_docs_tree_out: the six tree arrays, term_end and doc_count, indexed by preorder id."""
    _fields_ = [("tree", Tree), ("term_end", ctypes.c_void_p), ("doc_count", ctypes.c_void_p)]


DOCS_TREE_FIELDS = TREE_FIELDS + ("term_end", "doc_count")

_lib = None


def lib():
    """Loads libb200sa.so (built by __graft_entry__.build()); raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libb200sa.so is not built (run `python __graft_entry__.py`); "
                           "suffix_b200 has no CPU fallback")
    L = ctypes.CDLL(LIB_PATH)
    vp, u64, u32, ci = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int
    sig = {
        "b200sa_ctx_create": ([ci, ctypes.POINTER(vp)], ci),
        "b200sa_ctx_destroy": ([vp], None),
        "b200sa_build": ([vp, vp, u64, vp], ci),
        "b200sa_lcp": ([vp, vp, u64, vp, vp], ci),
        "b200sa_build_lcp": ([vp, vp, u64, vp, vp], ci),
        "b200sa_build_dev": ([vp, vp, u64, vp, vp], ci),
        "b200sa_lcp_dev": ([vp, vp, u64, vp, vp, vp], ci),
        "b200sa_build_lcp_dev": ([vp, vp, u64, vp, vp, vp], ci),
        "b200sa_positions_dev": ([vp, vp, u64, vp, vp, vp, u32, vp, vp, vp], ci),
        "b200sa_shard_summary": ([vp, vp, u64, ci, ctypes.POINTER(ci), vp], ci),
        "b200sa_shard_classify": ([vp, vp, u64, ci, ci, ci, vp, vp, vp, u64, vp, ctypes.POINTER(u64), vp], ci),
        "b200sa_comm_unique_id": ([vp], ci),
        "b200sa_comm_init": ([vp, ci, ci, vp], ci),
        "b200sa_comm_attach": ([vp, vp], ci),
        "b200sa_comm_destroy": ([vp], ci),
        "b200sa_shard_lms_sort": ([vp, vp, u64, vp, vp, u64, ctypes.POINTER(ShardStats), vp], ci),
        "b200sa_doc_ids_dev": ([vp, vp, u64, vp, u32, vp, vp, vp], ci),
        "b200sa_lcp_intervals_dev": ([vp, vp, u64, vp, vp, vp], ci),
        "b200sa_lcp_sharded": ([vp, vp, u64, vp, vp, ci, vp], ci),
        "b200sa_suffix_tree_dev": ([vp, u64, vp, vp, ctypes.POINTER(Tree), u64, ctypes.POINTER(u64), vp], ci),
        "b200sa_suffix_tree": ([vp, u64, vp, vp, ctypes.POINTER(Tree), u64, ctypes.POINTER(u64)], ci),
        "b200sa_docs_build": ([vp, vp, u64, vp, u32, vp, vp], ci),
        "b200sa_docs_build_dev": ([vp, vp, u64, vp, u32, vp, vp, vp], ci),
        "b200sa_docs_positions_dev": ([vp, vp, u64, vp, vp, u32, vp, vp, u32, vp, vp, vp], ci),
        "b200sa_docs_tree_dev": ([vp, u64, vp, vp, vp, u32, ctypes.POINTER(DocsTree), u64, ctypes.POINTER(u64), vp], ci),
        "b200sa_docs_tree": ([vp, u64, vp, vp, vp, u32, ctypes.POINTER(DocsTree), u64, ctypes.POINTER(u64)], ci),
        "b200sa_docs_tree_counts_dev": ([vp, vp, vp, vp, u64, vp, vp, u32, vp, vp], ci),
        "b200sa_docs_list_index_dev": ([vp, u64, vp, vp, u32, vp, vp, vp], ci),
        "b200sa_docs_list_dev": ([vp, u64, vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u64, ctypes.POINTER(u64), vp],
                                 ci),
        "b200sa_docs_topk_dev": ([vp, u64, vp, vp, u32, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp], ci),
        "b200sa_match_stats_dev": ([vp, vp, u64, vp, vp, vp, vp, u32, u64, vp, vp, vp, vp], ci),
        "b200sa_docs_match_stats_dev": ([vp, vp, u64, vp, vp, vp, u32, vp, vp, u32, u64, vp, vp, vp, vp], ci),
        "b200sa_smems_dev": ([vp, vp, u32, u64, vp, u32, vp, vp, u64, ctypes.POINTER(u64), vp], ci),
        "b200sa_repeat_lens_dev": ([vp, u64, vp, vp, vp, vp], ci),
        "b200sa_repeat_runs_dev": ([vp, u64, vp, vp, u32, vp, vp, vp, vp, u64, ctypes.POINTER(u64), vp], ci),
        "b200sa_duplicate_spans_dev": ([vp, u64, vp, vp, vp, u32, u32, ci, vp, vp, u64, ctypes.POINTER(u64),
                                        ctypes.POINTER(u64), vp], ci),
        "b200sa_lpf_dev": ([vp, u64, vp, vp, vp, vp, vp], ci),
        "b200sa_lz77_dev": ([vp, u64, vp, vp, vp, vp, vp, u64, ctypes.POINTER(u64), vp], ci),
        "b200sa_bwt_dev": ([vp, u64, vp, vp, vp, u32, vp, vp, ctypes.POINTER(u64), vp], ci),
        "b200sa_unbwt_dev": ([vp, u64, u32, vp, vp, vp, vp, vp], ci),
        "b200sa_approx_positions_dev": ([vp, vp, u64, vp, vp, vp, u32, u32, vp, vp, vp, u64, ctypes.POINTER(u64), vp],
                                        ci),
        "b200sa_docs_approx_positions_dev": ([vp, vp, u64, vp, vp, u32, vp, vp, u32, u32, vp, vp, vp, u64,
                                              ctypes.POINTER(u64), vp], ci),
        "b200sa_last_stats": ([vp, ctypes.POINTER(Stats)], ci),
        "b200sa_set_timing": ([vp, ci], ci),
        "b200sa_last_phase_times": ([vp, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_float), ci], ci),
        "b200sa_strerror": ([ci], ctypes.c_char_p),
        "b200sa_last_error": ([vp], ctypes.c_char_p),
        "b200sa_version": ([], ctypes.c_char_p),
        "b200sa_test_classify_fused": ([vp, vp, u64, vp, vp, vp, vp, u64, ctypes.POINTER(u64)], ci),
        "b200sa_test_scan": ([vp, vp, u64, ci, vp, ctypes.POINTER(u32)], ci),
        "b200sa_test_sort_pairs32": ([vp, vp, vp, u64, ci], ci),
        "b200sa_test_sort_pairs64": ([vp, vp, vp, u64, ci], ci),
        "b200sa_test_reduced_sa": ([vp, vp, u64, u32, vp, ctypes.POINTER(u32)], ci),
        "b200sa_debug_fetch": ([vp, ci, vp, u64], ctypes.c_int64),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = res
    _lib = L
    return L


def strerror(code):
    try:
        return lib().b200sa_strerror(code).decode()
    except Exception:
        return "?"


class Context:
    """One CUDA device + stream + reusable device workspace (b200sa_ctx)."""

    def __init__(self, device: int = 0):
        self._h = ctypes.c_void_p()
        rc = lib().b200sa_ctx_create(device, ctypes.byref(self._h))
        if rc != 0:
            raise B200SAError(rc, "b200sa_ctx_create(device=%d)" % device)
        self.device = device

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().b200sa_ctx_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise B200SAError(rc, lib().b200sa_last_error(self._h).decode())

    # ---- host-buffer API
    def build(self, text: np.ndarray) -> np.ndarray:
        sa = np.empty(len(text), dtype=np.uint32)
        self._check(lib().b200sa_build(self._h, text.ctypes.data, len(text), sa.ctypes.data))
        return sa

    def lcp(self, text: np.ndarray, sa: np.ndarray) -> np.ndarray:
        out = np.empty(len(text), dtype=np.uint32)
        self._check(lib().b200sa_lcp(self._h, text.ctypes.data, len(text), sa.ctypes.data, out.ctypes.data))
        return out

    def build_lcp(self, text: np.ndarray):
        sa = np.empty(len(text), dtype=np.uint32)
        lcp = np.empty(len(text), dtype=np.uint32)
        self._check(lib().b200sa_build_lcp(self._h, text.ctypes.data, len(text), sa.ctypes.data, lcp.ctypes.data))
        return sa, lcp

    # ---- device-pointer API (raw integer device pointers, e.g. torch .data_ptr())
    def build_dev(self, d_text: int, n: int, d_sa: int, stream: int = 0):
        self._check(lib().b200sa_build_dev(self._h, d_text, n, d_sa, stream))

    def lcp_dev(self, d_text: int, n: int, d_sa: int, d_lcp: int, stream: int = 0):
        self._check(lib().b200sa_lcp_dev(self._h, d_text, n, d_sa, d_lcp, stream))

    def build_lcp_dev(self, d_text: int, n: int, d_sa: int, d_lcp: int, stream: int = 0):
        self._check(lib().b200sa_build_lcp_dev(self._h, d_text, n, d_sa, d_lcp, stream))

    def positions_dev(self, d_text, n, d_sa, d_q, d_qoff, nq, d_start, d_end, stream: int = 0):
        self._check(lib().b200sa_positions_dev(self._h, d_text, n, d_sa, d_q, d_qoff, nq, d_start, d_end, stream))

    # ---- multi-GPU shards (SURVEY 8e)
    def shard_summary(self, d_shard: int, length: int, next_char: int, stream: int = 0) -> int:
        st = ctypes.c_int(0)
        self._check(lib().b200sa_shard_summary(self._h, d_shard, length, next_char, ctypes.byref(st), stream))
        return int(st.value)

    def shard_classify(self, d_shard: int, length: int, prev_char: int, next_char: int, tail_carry: int,
                       d_stype: int = 0, d_lms: int = 0, d_lmspos: int = 0, cap_lms: int = 0, stream: int = 0):
        hist = np.zeros(768, dtype=np.uint64)
        m = ctypes.c_uint64(0)
        self._check(lib().b200sa_shard_classify(self._h, d_shard, length, prev_char, next_char, tail_carry,
                                                d_stype, d_lms, d_lmspos, cap_lms, hist.ctypes.data,
                                                ctypes.byref(m), stream))
        return hist, int(m.value)

    # communicator of the sharded entry points: NCCL inside the library (resolved at run time)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (ctypes.c_uint8 * 128)()
        rc = lib().b200sa_comm_unique_id(buf)
        if rc != 0:
            raise B200SAError(rc, "b200sa_comm_unique_id")
        return bytes(buf)

    def comm_init(self, nranks: int, rank: int, unique_id: bytes):
        buf = (ctypes.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(lib().b200sa_comm_init(self._h, nranks, rank, buf))

    def comm_destroy(self):
        self._check(lib().b200sa_comm_destroy(self._h))

    def shard_lms_sort(self, d_shard: int, length: int, d_gpos: int, d_names: int, cap: int, stream: int = 0) -> dict:
        """Collective (b200sa_shard_lms_sort): this rank's slice of the global LMS-suffix order."""
        st = ShardStats()
        self._check(lib().b200sa_shard_lms_sort(self._h, d_shard, length, d_gpos, d_names, cap, ctypes.byref(st), stream))
        return {f: getattr(st, f) for f, _ in ShardStats._fields_}

    def doc_ids_dev(self, d_pos: int, count: int, d_doc_starts: int, ndocs: int, d_doc: int, d_off: int, stream: int = 0):
        self._check(lib().b200sa_doc_ids_dev(self._h, d_pos, count, d_doc_starts, ndocs, d_doc, d_off, stream))

    def lcp_intervals_dev(self, d_lcp: int, n: int, d_psv: int, d_nsv: int, stream: int = 0):
        self._check(lib().b200sa_lcp_intervals_dev(self._h, d_lcp, n, d_psv, d_nsv, stream))

    def suffix_tree(self, sa: np.ndarray, lcp: np.ndarray) -> dict:
        """b200sa_suffix_tree: the reference's suffix tree as six u32 arrays of N entries."""
        sa = np.ascontiguousarray(sa, dtype=np.uint32)
        lcp = np.ascontiguousarray(lcp, dtype=np.uint32)
        if len(sa) != len(lcp):
            raise ValueError("sa and lcp lengths differ")
        n = len(sa)
        cap = max(1, 2 * n)
        arrs = {f: np.empty(cap, dtype=np.uint32) for f in TREE_FIELDS}
        t = Tree(*[arrs[f].ctypes.data for f in TREE_FIELDS])
        N = ctypes.c_uint64(0)
        self._check(lib().b200sa_suffix_tree(self._h, n, sa.ctypes.data, lcp.ctypes.data, ctypes.byref(t), cap,
                                             ctypes.byref(N)))
        return {f: a[:N.value] for f, a in arrs.items()}

    def suffix_tree_dev(self, n: int, d_sa: int, d_lcp: int, out_ptrs, cap: int, stream: int = 0) -> int:
        """b200sa_suffix_tree_dev; out_ptrs: six device pointers in TREE_FIELDS order.  Returns N."""
        t = Tree(*out_ptrs)
        N = ctypes.c_uint64(0)
        self._check(lib().b200sa_suffix_tree_dev(self._h, n, d_sa, d_lcp, ctypes.byref(t), cap, ctypes.byref(N), stream))
        return int(N.value)

    def docs_build(self, text: np.ndarray, doc_starts: np.ndarray, with_lcp: bool = True):
        """b200sa_docs_build: (gsa, glcp) of the documents concatenated in `text`; glcp is None
        without with_lcp."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        starts = np.ascontiguousarray(doc_starts, dtype=np.uint32)
        n = len(text)
        gsa = np.empty(n, dtype=np.uint32)
        glcp = np.empty(n, dtype=np.uint32) if with_lcp else None
        self._check(lib().b200sa_docs_build(self._h, text.ctypes.data, n, starts.ctypes.data, len(starts),
                                            gsa.ctypes.data, glcp.ctypes.data if with_lcp else None))
        return gsa, glcp

    def docs_build_dev(self, d_text: int, n: int, d_doc_starts: int, ndocs: int, d_gsa: int, d_glcp: int = 0,
                       stream: int = 0):
        self._check(lib().b200sa_docs_build_dev(self._h, d_text, n, d_doc_starts, ndocs, d_gsa, d_glcp or None,
                                                stream))

    def docs_positions_dev(self, d_text, n, d_gsa, d_doc_starts, ndocs, d_q, d_qoff, nq, d_start, d_end,
                           stream: int = 0):
        self._check(lib().b200sa_docs_positions_dev(self._h, d_text, n, d_gsa, d_doc_starts, ndocs, d_q, d_qoff, nq,
                                                    d_start, d_end, stream))

    def docs_tree(self, gsa: np.ndarray, glcp: np.ndarray, doc_starts: np.ndarray) -> dict:
        """b200sa_docs_tree: the generalized suffix tree of (G, glcp) as eight u32 arrays of N entries."""
        gsa = np.ascontiguousarray(gsa, dtype=np.uint32)
        glcp = np.ascontiguousarray(glcp, dtype=np.uint32)
        starts = np.ascontiguousarray(doc_starts, dtype=np.uint32)
        if len(gsa) != len(glcp):
            raise ValueError("gsa and glcp lengths differ")
        n = len(gsa)
        cap = max(1, 2 * n)
        arrs = {f: np.empty(cap, dtype=np.uint32) for f in DOCS_TREE_FIELDS}
        t = DocsTree(Tree(*[arrs[f].ctypes.data for f in TREE_FIELDS]), arrs["term_end"].ctypes.data,
                     arrs["doc_count"].ctypes.data)
        N = ctypes.c_uint64(0)
        self._check(lib().b200sa_docs_tree(self._h, n, gsa.ctypes.data, glcp.ctypes.data,
                                           starts.ctypes.data if len(starts) else None, len(starts), ctypes.byref(t),
                                           cap, ctypes.byref(N)))
        return {f: a[:N.value] for f, a in arrs.items()}

    def docs_tree_dev(self, n: int, d_gsa: int, d_glcp: int, d_doc_starts: int, ndocs: int, out_ptrs, cap: int,
                      stream: int = 0) -> int:
        """b200sa_docs_tree_dev; out_ptrs: eight device pointers in DOCS_TREE_FIELDS order.  Returns N."""
        t = DocsTree(Tree(*out_ptrs[:6]), out_ptrs[6], out_ptrs[7])
        N = ctypes.c_uint64(0)
        self._check(lib().b200sa_docs_tree_dev(self._h, n, d_gsa, d_glcp, d_doc_starts or None, ndocs, ctypes.byref(t),
                                               cap, ctypes.byref(N), stream))
        return int(N.value)

    def docs_tree_counts_dev(self, d_sa_lo, d_sa_hi, d_doc_count, num_nodes, d_start, d_end, nq, d_count,
                             stream: int = 0):
        self._check(lib().b200sa_docs_tree_counts_dev(self._h, d_sa_lo, d_sa_hi, d_doc_count, num_nodes, d_start,
                                                      d_end, nq, d_count, stream))

    def docs_list_index_dev(self, n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev, stream: int = 0):
        """b200sa_docs_list_index_dev: byd and prev (n u32 each) of G for document listing."""
        self._check(lib().b200sa_docs_list_index_dev(self._h, n, d_gsa, d_doc_starts or None, ndocs, d_byd, d_prev,
                                                     stream))

    def docs_list_dev(self, n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev, d_start, d_end, nq, d_offsets, d_docs,
                      d_tf, cap, stream: int = 0) -> int:
        """b200sa_docs_list_dev: writes the offsets, and docs / tf when the listing fits in cap.  Returns the total."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_docs_list_dev(self._h, n, d_gsa, d_doc_starts or None, ndocs, d_byd, d_prev, d_start,
                                               d_end, nq, d_offsets, d_docs or None, d_tf or None, cap,
                                               ctypes.byref(total), stream))
        return int(total.value)

    def docs_topk_dev(self, n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev, d_start, d_end, nq, k, d_count, d_docs, d_tf,
                      stream: int = 0):
        """b200sa_docs_topk_dev: count[q] = min(k, df(q)); docs / tf[q*k + j] for j < count[q], best first."""
        self._check(lib().b200sa_docs_topk_dev(self._h, n, d_gsa, d_doc_starts or None, ndocs, d_byd, d_prev, d_start,
                                               d_end, nq, k, d_count, d_docs, d_tf, stream))

    def match_stats_dev(self, d_text, n, d_sa, d_lcp, d_q, d_qoff, nq, q_bytes, d_len, d_start=0, d_end=0,
                        stream: int = 0):
        """b200sa_match_stats_dev: len (and the table range, when d_start / d_end are given) of every pattern
        position; d_lcp may be 0 without the ranges."""
        self._check(lib().b200sa_match_stats_dev(self._h, d_text, n, d_sa, d_lcp or None, d_q, d_qoff, nq, q_bytes,
                                                 d_len, d_start or None, d_end or None, stream))

    def docs_match_stats_dev(self, d_text, n, d_gsa, d_glcp, d_doc_starts, ndocs, d_q, d_qoff, nq, q_bytes, d_len,
                             d_start=0, d_end=0, stream: int = 0):
        """b200sa_docs_match_stats_dev: the same over G, every suffix cut at its document's end."""
        self._check(lib().b200sa_docs_match_stats_dev(self._h, d_text, n, d_gsa, d_glcp or None, d_doc_starts or None,
                                                      ndocs, d_q, d_qoff, nq, q_bytes, d_len, d_start or None,
                                                      d_end or None, stream))

    def smems_dev(self, d_qoff, nq, q_bytes, d_len, min_len, d_offsets, d_qpos, cap, stream: int = 0) -> int:
        """b200sa_smems_dev: writes the offsets, and qpos when the SMEMs fit in cap.  Returns the total."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_smems_dev(self._h, d_qoff, nq, q_bytes, d_len, min_len, d_offsets, d_qpos or None,
                                           cap, ctypes.byref(total), stream))
        return int(total.value)

    def repeat_lens_dev(self, n, d_sa, d_lcp, d_rl, stream: int = 0):
        """b200sa_repeat_lens_dev: d_rl[p] = the longest prefix of the suffix at p that starts elsewhere too."""
        self._check(lib().b200sa_repeat_lens_dev(self._h, n, d_sa or None, d_lcp or None, d_rl or None, stream))

    def repeat_runs_dev(self, n, d_sa, d_lcp, min_len, d_start=0, d_end=0, d_first=0, d_last=0, cap=0,
                        stream: int = 0) -> int:
        """b200sa_repeat_runs_dev: writes the runs at min_len when they fit in cap.  Returns the total."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_repeat_runs_dev(self._h, n, d_sa or None, d_lcp or None, min_len, d_start or None,
                                                 d_end or None, d_first or None, d_last or None, cap,
                                                 ctypes.byref(total), stream))
        return int(total.value)

    def duplicate_spans_dev(self, n, d_sa, d_lcp, d_doc_starts, ndocs, min_len, mode, d_begin=0, d_end=0, cap=0,
                            stream: int = 0):
        """b200sa_duplicate_spans_dev: writes the spans when they fit in cap.  Returns (total, covered)."""
        total, covered = ctypes.c_uint64(0), ctypes.c_uint64(0)
        self._check(lib().b200sa_duplicate_spans_dev(self._h, n, d_sa or None, d_lcp or None, d_doc_starts or None,
                                                     ndocs, min_len, mode, d_begin or None, d_end or None, cap,
                                                     ctypes.byref(total), ctypes.byref(covered), stream))
        return int(total.value), int(covered.value)

    def lpf_dev(self, n, d_sa, d_lcp, d_lpf, d_src=0, stream: int = 0):
        """b200sa_lpf_dev: d_lpf[p] = the longest previous factor at p, d_src[p] (if given) one earlier start."""
        self._check(lib().b200sa_lpf_dev(self._h, n, d_sa or None, d_lcp or None, d_lpf or None, d_src or None,
                                         stream))

    def lz77_dev(self, n, d_sa, d_lcp, d_start=0, d_len=0, d_src=0, cap=0, stream: int = 0) -> int:
        """b200sa_lz77_dev: writes the factors when they fit in cap.  Returns z."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_lz77_dev(self._h, n, d_sa or None, d_lcp or None, d_start or None, d_len or None,
                                          d_src or None, cap, ctypes.byref(total), stream))
        return int(total.value)

    def bwt_dev(self, n, d_text, d_sa, d_doc_starts, ndocs, d_bwt, d_term_rows, runs=False, stream: int = 0):
        """b200sa_bwt_dev: writes the bwt (n bytes) and the term rows; d_doc_starts = 0 with ndocs = 0 is a single
        text.  Returns r when runs is true (the call then synchronises), else None."""
        r = ctypes.c_uint64(0)
        self._check(lib().b200sa_bwt_dev(self._h, n, d_text or None, d_sa or None, d_doc_starts or None, ndocs,
                                         d_bwt or None, d_term_rows or None, ctypes.byref(r) if runs else None,
                                         stream))
        return int(r.value) if runs else None

    def unbwt_dev(self, n, ndocs, d_bwt, d_term_rows, d_text, d_doc_starts=0, stream: int = 0):
        """b200sa_unbwt_dev: writes the documents' concatenation (n bytes) and, if given, their starts (ndocs)."""
        self._check(lib().b200sa_unbwt_dev(self._h, n, ndocs, d_bwt or None, d_term_rows or None, d_text or None,
                                           d_doc_starts or None, stream))

    def approx_positions_dev(self, d_text, n, d_sa, d_q, d_qoff, nq, k, d_offsets, d_pos=0, d_mis=0, cap=0,
                             stream: int = 0) -> int:
        """b200sa_approx_positions_dev: writes the offsets, and the positions (and mismatches, if given) of the
        occurrences with at most k mismatches when they fit in cap.  Returns the total."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_approx_positions_dev(self._h, d_text or None, n, d_sa or None, d_q or None,
                                                      d_qoff or None, nq, k, d_offsets or None, d_pos or None,
                                                      d_mis or None, cap, ctypes.byref(total), stream))
        return int(total.value)

    def docs_approx_positions_dev(self, d_text, n, d_gsa, d_doc_starts, ndocs, d_q, d_qoff, nq, k, d_offsets,
                                  d_pos=0, d_mis=0, cap=0, stream: int = 0) -> int:
        """b200sa_docs_approx_positions_dev: the same over G, no window crossing a document end."""
        total = ctypes.c_uint64(0)
        self._check(lib().b200sa_docs_approx_positions_dev(self._h, d_text or None, n, d_gsa or None,
                                                           d_doc_starts or None, ndocs, d_q or None, d_qoff or None,
                                                           nq, k, d_offsets or None, d_pos or None, d_mis or None,
                                                           cap, ctypes.byref(total), stream))
        return int(total.value)

    def lcp_sharded(self, d_text: int, n: int, d_sa: int, d_lcp: int, replicated: bool = False, stream: int = 0):
        self._check(lib().b200sa_lcp_sharded(self._h, d_text, n, d_sa, d_lcp, 1 if replicated else 0, stream))

    # ---- introspection
    def set_timing(self, on: bool):
        self._check(lib().b200sa_set_timing(self._h, 1 if on else 0))

    def phase_times(self):
        names = (ctypes.c_char_p * 64)()
        ms = (ctypes.c_float * 64)()
        k = lib().b200sa_last_phase_times(self._h, names, ms, 64)
        return [(names[i].decode(), float(ms[i])) for i in range(max(0, min(k, 64)))]

    def stats(self) -> dict:
        s = Stats()
        self._check(lib().b200sa_last_stats(self._h, ctypes.byref(s)))
        return {f: int(getattr(s, f)) for f, _ in Stats._fields_}

    def debug_fetch(self, which: int, cap: int = 1 << 26) -> np.ndarray:
        out = np.empty(cap, dtype=np.uint32)
        k = lib().b200sa_debug_fetch(self._h, which, out.ctypes.data, cap)
        if k < 0:
            raise B200SAError(int(k))
        return out[:min(k, cap)].copy()


_default = {}


def default_context(device: int = 0) -> Context:
    """Lazily created per-device context used by SuffixTable."""
    if device not in _default:
        _default[device] = Context(device)
    return _default[device]
