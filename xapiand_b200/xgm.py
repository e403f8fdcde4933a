"""ctypes bindings of the C-ABI in include/xgm.h (libxgm.so) plus a thin Enquire/MSet-shaped layer.

PyTorch is not needed to search; it is only used by bench.py / the multi-GPU tests for device
buffers, streams and torch.distributed.  There is no CPU path: importing works anywhere (so the
`not gpu` tests can check the exported symbols), but building an index without a CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Union

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libxgm.so")

OP_AND, OP_OR = 0, 1
SORT_REL, SORT_VAL_REL, SORT_VAL, SORT_REL_VAL = 0, 1, 2, 3
MSET_BOUNDS_APPROX, MSET_COUNT_LOWER_BOUND = 1, 2  # xgm_mset_info.flags (include/xgm.h)
FILTER_NONE, FILTER_VALUE_RANGE, FILTER_MULTI_RANGE = 0, 1, 2
OK, E_INVALID, E_UNIMPLEMENTED, E_CUDA, E_NOMEM, E_IO, E_STALE, E_NODEVICE = range(8)
MAX_TERMS = 16
MAX_TOPK = 4096

EXPORTS = [
    "xgm_last_error", "xgm_abi_version", "xgm_builder_new", "xgm_builder_set_docs", "xgm_builder_add_term",
    "xgm_builder_add_value_slot", "xgm_builder_finish", "xgm_builder_free", "xgm_index_build_synthetic",
    "xgm_index_load_flat", "xgm_index_close", "xgm_index_info_get", "xgm_term_stats_get",
    "xgm_index_decode_term", "xgm_index_copy_doclengths", "xgm_searcher_new", "xgm_searcher_free", "xgm_search_submit", "xgm_search_wait",
    "xgm_search_submit_async", "xgm_search_launched", "xgm_search_batch", "xgm_search", "xgm_search_replay",
    "xgm_search_device_results", "xgm_search_device_slab", "xgm_search_device_slab_keys",
    "xgm_searcher_stream", "xgm_search_last_stats", "xgm_unshard", "xgm_merge_msets", "xgm_merge_topk_device",
    "xgm_merge_topk_device_slab", "xgm_merge_mset_device_slab",
    "xgm_builder_add_value_slot_serialised", "xgm_builder_set_revision", "xgm_index_value_freq",
    "xgm_value_key", "xgm_value_key_bytes", "xgm_sort_key_bytes", "xgm_term_stats_many",
    "xgm_index_open", "xgm_glass_revision", "xgm_glass_export_flat", "xgm_searcher_set_results_on_device",
]


class XgmError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"xgm status {status}: {msg}")
        self.status = status


class IndexInfo(C.Structure):
    _fields_ = [("doccount", C.c_uint32), ("lastdocid", C.c_uint32), ("total_length", C.c_uint64),
                ("doclen_lower_bound", C.c_uint32), ("doclen_upper_bound", C.c_uint32),
                ("nterms", C.c_uint32), ("npostings", C.c_uint64), ("nblocks", C.c_uint64),
                ("bytes_docids", C.c_uint64), ("bytes_wdfs", C.c_uint64), ("bytes_headers", C.c_uint64),
                ("bytes_doclen", C.c_uint64), ("device", C.c_int), ("revision", C.c_uint64),
                ("bytes_bitmaps", C.c_uint64), ("nbitmaps", C.c_uint32)]


class TermStats(C.Structure):
    _fields_ = [("term_id", C.c_uint32), ("termfreq", C.c_uint32), ("collfreq", C.c_uint64),
                ("wdf_upper_bound", C.c_uint32), ("bytes", C.c_uint64)]


class CStats(C.Structure):
    _fields_ = [("collection_size", C.c_uint32), ("total_length", C.c_uint64),
                ("termfreq", C.POINTER(C.c_uint32))]


class CQuery(C.Structure):
    _fields_ = [("op", C.c_uint32), ("nterms", C.c_uint32), ("terms", C.POINTER(C.c_char_p)),
                ("term_lens", C.POINTER(C.c_uint32)), ("term_ids", C.POINTER(C.c_uint32)),
                ("wqf", C.POINTER(C.c_uint32)), ("first", C.c_uint32), ("maxitems", C.c_uint32),
                ("check_at_least", C.c_uint32), ("stats", C.POINTER(CStats)),
                ("k1", C.c_double), ("k3", C.c_double), ("b", C.c_double), ("min_normlen", C.c_double),
                ("filter", C.c_uint32), ("filter_slot", C.c_uint32), ("range_lo", C.c_uint64),
                ("range_hi", C.c_uint64), ("sort_by", C.c_uint32), ("sort_slot", C.c_uint32),
                ("sort_reverse", C.c_uint32), ("sort_use_max", C.c_uint32),
                ("nfilter", C.c_uint32), ("nnot", C.c_uint32), ("nmaybe", C.c_uint32), ("reserved", C.c_uint32),
                ("factors", C.POINTER(C.c_double)),
                # ABI 2
                ("revision", C.c_uint64), ("filter_weighted", C.c_uint32), ("reserved2", C.c_uint32),
                ("filter_factor", C.c_double), ("sort_missing_key", C.c_uint64)]


class MSetInfo(C.Structure):
    _fields_ = [("n", C.c_uint32), ("first", C.c_uint32), ("matches_lower_bound", C.c_uint32),
                ("matches_estimated", C.c_uint32), ("matches_upper_bound", C.c_uint32),
                ("uncollapsed_lower_bound", C.c_uint32), ("uncollapsed_estimated", C.c_uint32),
                ("uncollapsed_upper_bound", C.c_uint32), ("exact_matches", C.c_uint32), ("status", C.c_uint32),
                ("flags", C.c_uint32), ("reserved", C.c_uint32),
                ("max_possible", C.c_double), ("max_attained", C.c_double), ("percent_scale_factor", C.c_double)]


class BatchStats(C.Structure):
    _fields_ = [("algorithmic_bytes", C.c_uint64), ("postings", C.c_uint64), ("work_items", C.c_uint32),
                ("kernel_launches", C.c_uint32), ("match_kernel_ms", C.c_float), ("topk_kernel_ms", C.c_float),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("host_plan_ms", C.c_float), ("host_wait_ms", C.c_float),
                ("second_pass_queries", C.c_uint32), ("reserved", C.c_uint32)]


_lib = None


def lib():
    """Load libxgm.so; fail loudly when it has not been built (there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(LIB_PATH)
    L.xgm_last_error.restype = C.c_char_p
    L.xgm_abi_version.restype = C.c_uint32
    L.xgm_builder_new.argtypes = [C.POINTER(C.c_void_p)]
    L.xgm_builder_set_docs.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32,
                                       C.c_void_p]
    L.xgm_builder_add_term.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                       C.c_uint64, C.c_uint32, C.POINTER(C.c_uint32)]
    L.xgm_builder_add_value_slot.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.xgm_builder_add_value_slot_serialised.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.xgm_builder_set_revision.argtypes = [C.c_void_p, C.c_uint64]
    L.xgm_index_value_freq.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    L.xgm_value_key.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64)]
    L.xgm_value_key.restype = C.c_int
    L.xgm_value_key_bytes.argtypes = [C.c_uint64, C.c_char_p]
    L.xgm_value_key_bytes.restype = C.c_size_t
    L.xgm_sort_key_bytes.argtypes = [C.c_uint64, C.c_int, C.c_char_p]
    L.xgm_sort_key_bytes.restype = C.c_size_t
    L.xgm_builder_finish.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.xgm_builder_free.argtypes = [C.c_void_p]
    L.xgm_builder_free.restype = None
    L.xgm_index_build_synthetic.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int,
                                            C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.xgm_index_load_flat.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
    L.xgm_index_open.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
    L.xgm_glass_revision.argtypes = [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.xgm_glass_export_flat.argtypes = [C.c_char_p, C.c_char_p]
    L.xgm_index_close.argtypes = [C.c_void_p]
    L.xgm_index_close.restype = None
    L.xgm_index_info_get.argtypes = [C.c_void_p, C.POINTER(IndexInfo)]
    L.xgm_term_stats_get.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.POINTER(TermStats)]
    L.xgm_term_stats_many.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_char_p), C.c_void_p, C.c_void_p]
    L.xgm_index_decode_term.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                        C.POINTER(C.c_uint32)]
    L.xgm_searcher_new.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
    L.xgm_searcher_free.argtypes = [C.c_void_p]
    L.xgm_searcher_free.restype = None
    L.xgm_index_copy_doclengths.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    L.xgm_search_submit.argtypes = [C.c_void_p, C.POINTER(CQuery), C.c_uint32]
    L.xgm_search_submit_async.argtypes = [C.c_void_p, C.POINTER(CQuery), C.c_uint32]
    L.xgm_search_launched.argtypes = [C.c_void_p]
    L.xgm_search_wait.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(MSetInfo)]
    L.xgm_search_batch.argtypes = [C.c_void_p, C.POINTER(CQuery), C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_uint32, C.POINTER(MSetInfo)]
    L.xgm_search.argtypes = [C.c_void_p, C.POINTER(CQuery), C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                             C.POINTER(MSetInfo)]
    L.xgm_search_replay.argtypes = [C.c_void_p]
    L.xgm_searcher_set_results_on_device.argtypes = [C.c_void_p, C.c_int]
    L.xgm_search_device_results.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
    L.xgm_search_device_slab.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                         C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.xgm_search_device_slab_keys.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.xgm_merge_topk_device_slab.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
                                             C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.xgm_merge_mset_device_slab.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p,
                                             C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.xgm_searcher_stream.argtypes = [C.c_void_p]
    L.xgm_searcher_stream.restype = C.c_void_p
    L.xgm_search_last_stats.argtypes = [C.c_void_p, C.POINTER(BatchStats)]
    L.xgm_unshard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    L.xgm_unshard.restype = None
    L.xgm_merge_msets.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                  C.POINTER(MSetInfo), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MSetInfo)]
    L.xgm_merge_topk_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    _lib = L
    return L


def _check(st: int):
    if st != OK:
        raise XgmError(st, lib().xgm_last_error().decode(errors="replace"))


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------


@dataclass
class Query:
    """Mirror of what reaches Matcher::get_local_mset for one Enquire::get_mset call."""
    op: int
    terms: Sequence[Union[str, bytes, int]]      # term strings, or pre-resolved ids when ints
    first: int = 0
    maxitems: int = 10
    check_at_least: int = 0
    wqf: Optional[Sequence[int]] = None
    stats: Optional[tuple] = None                # (collection_size, total_length, [global termfreq...])
    filter: int = FILTER_NONE
    filter_slot: int = 0
    range_lo: int = 0
    range_hi: int = 0
    sort_by: int = SORT_REL
    sort_slot: int = 0
    sort_reverse: bool = False
    sort_use_max: bool = False
    # OP_FILTER(q, AND of boolean terms) / OP_AND_NOT(q, OR of terms) / OP_AND_MAYBE(q, OR of terms): AND base only
    filter_terms: Sequence[Union[str, bytes, int]] = ()
    not_terms: Sequence[Union[str, bytes, int]] = ()
    maybe_terms: Sequence[Union[str, bytes, int]] = ()
    factors: Optional[Sequence[float]] = None     # OP_SCALE_WEIGHT factor per base term
    bm25: Optional[tuple] = None                  # (k1, k3, b, min_normlen); None = BM25Weight defaults
    revision: int = 0                             # expected Database::get_revision (0 = any)
    filter_weighted: bool = False                 # the range source is an AND child with weight factor * 1.0
    filter_factor: float = 0.0
    sort_missing_key: int = 0                     # key of documents without a value in sort_slot


class QueryBatch:
    """A batch of queries marshalled once into the C structs (host memory the C-ABI reads)."""

    def __init__(self, queries: Sequence[Query]):
        self.n = len(queries)
        self.arr = (CQuery * self.n)()
        self._keep = []
        for i, q in enumerate(queries):
            cq = self.arr[i]
            cq.op, cq.nterms = q.op, len(q.terms)
            cq.nfilter, cq.nnot, cq.nmaybe = len(q.filter_terms), len(q.not_terms), len(q.maybe_terms)
            allterms = list(q.terms) + list(q.filter_terms) + list(q.not_terms) + list(q.maybe_terms)
            if all(isinstance(t, (int, np.integer)) for t in allterms):
                ids = (C.c_uint32 * len(allterms))(*[int(t) for t in allterms])
                cq.term_ids = ids
                self._keep.append(ids)
            else:
                bs = [t.encode() if isinstance(t, str) else bytes(t) for t in allterms]
                names = (C.c_char_p * len(bs))(*bs)
                lens = (C.c_uint32 * len(bs))(*[len(b) for b in bs])
                cq.terms, cq.term_lens = names, lens
                self._keep += [names, lens, bs]
            if q.wqf is not None:
                w = (C.c_uint32 * len(q.wqf))(*q.wqf)
                cq.wqf = w
                self._keep.append(w)
            cq.first, cq.maxitems, cq.check_at_least = q.first, q.maxitems, q.check_at_least
            if q.factors is not None:
                fac = (C.c_double * len(q.factors))(*[float(x) for x in q.factors])
                cq.factors = fac
                self._keep.append(fac)
            if q.bm25 is not None:
                cq.k1, cq.k3, cq.b, cq.min_normlen = [float(x) for x in q.bm25]
            if q.stats is not None:
                gtf = list(q.stats[2]) + [0] * (len(allterms) - len(q.stats[2]))
                tf = (C.c_uint32 * len(gtf))(*gtf)
                st = CStats(q.stats[0], q.stats[1], tf)
                cq.stats = C.pointer(st)
                self._keep += [tf, st]
            cq.filter, cq.filter_slot = q.filter, q.filter_slot
            cq.range_lo, cq.range_hi = q.range_lo, q.range_hi
            cq.sort_by, cq.sort_slot = q.sort_by, q.sort_slot
            cq.sort_reverse, cq.sort_use_max = int(q.sort_reverse), int(q.sort_use_max)
            cq.revision, cq.filter_weighted, cq.filter_factor = q.revision, int(q.filter_weighted), float(q.filter_factor)
            cq.sort_missing_key = q.sort_missing_key


def _attach_global_stats(self):
    """Give every query of the batch an xgm_stats block backed by ONE (nq, MAX_TERMS) uint32 matrix, so that the
    global statistics of a batch (phase 1 of the two-phase scheme) can be filled in with two vectorised writes
    after the all-reduce instead of re-marshalling the queries."""
    self.gtf = np.zeros((self.n, MAX_TERMS), np.uint32)
    self.cstats = (CStats * self.n)()
    view = np.frombuffer(self.cstats, dtype=[("coll", "<u4"), ("pad", "<u4"), ("tlen", "<u8"), ("ptr", "<u8")])
    view["ptr"] = self.gtf.ctypes.data + np.arange(self.n, dtype=np.uint64) * (MAX_TERMS * 4)
    self._stats_view = view
    base = C.addressof(self.cstats)
    for i in range(self.n):
        self.arr[i].stats = C.cast(base + i * C.sizeof(CStats), C.POINTER(CStats))


def _set_global_stats(self, collection_size: int, total_length: int, termfreqs: np.ndarray):
    """termfreqs: (nq, k) global termfreq per query term, in query order."""
    self._stats_view["coll"] = collection_size
    self._stats_view["tlen"] = total_length
    self.gtf[:, :termfreqs.shape[1]] = termfreqs


QueryBatch.attach_global_stats = _attach_global_stats
QueryBatch.set_global_stats = _set_global_stats


@dataclass
class MSet:
    """Fields of the reference's MSet::Internal (src/xapian/api/msetinternal.h:58-99)."""
    docids: np.ndarray
    weights: np.ndarray
    sort_keys: Optional[np.ndarray]
    first: int
    matches_lower_bound: int
    matches_estimated_raw: int
    matches_upper_bound: int
    max_possible: float
    max_attained: float
    percent_scale_factor: float
    exact_matches: int
    status: int
    flags: int = 0

    def size(self) -> int:
        return len(self.docids)

    def get_matches_lower_bound(self) -> int:
        return self.matches_lower_bound

    def get_matches_upper_bound(self) -> int:
        return self.matches_upper_bound

    def get_matches_estimated(self) -> int:
        """MSet::get_matches_estimated rounds (api/mset.cc:145-153, api/roundestimate.h:35-64)."""
        return round_estimate(self.matches_lower_bound, self.matches_upper_bound, self.matches_estimated_raw)

    def __iter__(self):
        return iter(zip(self.docids.tolist(), self.weights.tolist()))


def round_estimate(m: int, M: int, e: int) -> int:
    """round_estimate<Xapian::doccount>, src/xapian/api/roundestimate.h:35-64 (uint32 arithmetic)."""
    import math
    D = M - m
    if D == 0 or e == 0:
        return e
    r = 10 ** int(math.log10(D))
    while r > e:
        r //= 10
    R = e // r * r
    if R < m:
        R += r
    elif R > M:
        R -= r
    elif R < e and r % 2 == 0 and e - R == r // 2:
        if e - m < M - e:
            R += r
    if R < m or R > M:
        R = e
    return R


class Index:
    def __init__(self, handle):
        self._h = handle

    @classmethod
    def synthetic(cls, ndocs: int, vocab: int, seed: int = 12345, nshards: int = 1, shard: int = 0,
                  values: bool = False, device: int = 0, host_threads: int = 0) -> "Index":
        h = C.c_void_p()
        _check(lib().xgm_index_build_synthetic(ndocs, vocab, seed, nshards, shard, int(values), device,
                                               host_threads, C.byref(h)))
        return cls(h)

    @classmethod
    def load_flat(cls, path: str, device: int = 0) -> "Index":
        h = C.c_void_p()
        _check(lib().xgm_index_load_flat(path.encode(), device, C.byref(h)))
        return cls(h)

    @classmethod
    def open_glass(cls, path: str, device: int = 0) -> "Index":
        """A glass database directory read directly by the library (xgm_index_open)."""
        h = C.c_void_p()
        _check(lib().xgm_index_open(path.encode(), device, C.byref(h)))
        return cls(h)

    @classmethod
    def from_postings(cls, doclen: np.ndarray, terms, doccount: Optional[int] = None,
                      total_length: Optional[int] = None, value_slots=None, device: int = 0,
                      serialised_slots=None, revision: int = 0) -> "Index":
        """terms: iterable of (name, docids u32[], wdfs u32[]) — what PostingIterator yields.
        serialised_slots: {slot: [bytes per docid 0..lastdocid]} — Document::get_value bytes as Xapiand stores
        them (StringList of serialised values)."""
        L = lib()
        b = C.c_void_p()
        _check(L.xgm_builder_new(C.byref(b)))
        try:
            doclen = np.ascontiguousarray(doclen, np.uint32)
            lastdocid = len(doclen) - 1
            used = doclen[1:][doclen[1:] > 0] if lastdocid else doclen[:0]
            dc = int(doccount if doccount is not None else len(used))
            tl = int(total_length if total_length is not None else int(doclen.sum()))
            lb = int(used.min()) if len(used) else 0
            ub = int(used.max()) if len(used) else 0
            _check(L.xgm_builder_set_docs(b, dc, lastdocid, tl, lb, ub, _ptr(doclen)))
            for name, d, w in terms:
                d = np.ascontiguousarray(d, np.uint32)
                w = np.ascontiguousarray(w, np.uint32)
                nm = name.encode() if isinstance(name, str) else bytes(name)
                _check(L.xgm_builder_add_term(b, nm, len(nm), _ptr(d), _ptr(w), len(d), int(w.sum()), 0, None))
            for slot, (voff, vals) in (value_slots or {}).items():
                voff = np.ascontiguousarray(voff, np.uint64)
                vals = np.ascontiguousarray(vals, np.uint64)
                _check(L.xgm_builder_add_value_slot(b, slot, _ptr(voff), _ptr(vals)))
            for slot, per_doc in (serialised_slots or {}).items():
                per_doc = list(per_doc) + [b""] * (lastdocid + 1 - len(per_doc))
                off = np.zeros(lastdocid + 2, np.uint64)
                off[1:] = np.cumsum([len(x) for x in per_doc])
                blob = b"".join(per_doc)
                buf = np.frombuffer(blob + b"\0", np.uint8)
                _check(L.xgm_builder_add_value_slot_serialised(b, slot, _ptr(off), _ptr(buf)))
            if revision:
                _check(L.xgm_builder_set_revision(b, revision))
            h = C.c_void_p()
            st = L.xgm_builder_finish(b, device, C.byref(h))
            b = None
            _check(st)
            return cls(h)
        finally:
            if b is not None:
                L.xgm_builder_free(b)

    def close(self):
        if self._h:
            lib().xgm_index_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self) -> IndexInfo:
        o = IndexInfo()
        _check(lib().xgm_index_info_get(self._h, C.byref(o)))
        return o

    def term_stats(self, term: Union[str, bytes]) -> TermStats:
        t = term.encode() if isinstance(term, str) else term
        o = TermStats()
        _check(lib().xgm_term_stats_get(self._h, t, len(t), C.byref(o)))
        return o

    def term_freqs(self, names: Sequence[Union[str, bytes]]) -> np.ndarray:
        """Local termfreq of many terms in one C call (xgm_term_stats_many)."""
        return self.term_freq_lookup(names)()

    def term_freq_lookup(self, names: Sequence[Union[str, bytes]]):
        """A callable that looks the same terms up again and again (the marshalling is done once)."""
        bs = [t.encode() if isinstance(t, str) else bytes(t) for t in names]
        arr = (C.c_char_p * len(bs))(*bs)
        lens = np.array([len(b) for b in bs], np.uint32)
        out = np.zeros(len(bs), np.uint32)
        L, h, n = lib(), self._h, len(bs)

        def lookup(_keep=(bs, arr, lens)):
            _check(L.xgm_term_stats_many(h, n, arr, _ptr(lens), _ptr(out)))
            return out
        return lookup

    def decode_term(self, term_id: int):
        n = C.c_uint32()
        _check(lib().xgm_index_decode_term(self._h, term_id, None, None, 0, C.byref(n)))
        d = np.zeros(n.value, np.uint32)
        w = np.zeros(n.value, np.uint32)
        if n.value:
            _check(lib().xgm_index_decode_term(self._h, term_id, _ptr(d), _ptr(w), n.value, C.byref(n)))
        return d, w

    def doclengths(self, first_docid: int = 0, n: Optional[int] = None) -> np.ndarray:
        if n is None:
            n = self.info().lastdocid + 1 - first_docid
        out = np.zeros(n, np.uint32)
        _check(lib().xgm_index_copy_doclengths(self._h, first_docid, n, _ptr(out)))
        return out


class Searcher:
    """One CUDA stream + staging buffers; use from one thread at a time (like one Xapian::Enquire)."""

    def __init__(self, index: Index, max_batch: int = 1024, max_topk: int = 128):
        self.index = index
        self.max_batch, self.max_topk = max_batch, max_topk
        h = C.c_void_p()
        _check(lib().xgm_searcher_new(index._h, max_batch, max_topk, C.byref(h)))
        self._h = h
        n = max_batch * max_topk
        self._docids = np.zeros(n, np.uint32)
        self._weights = np.zeros(n, np.float64)
        self._keys = np.zeros(n, np.uint64)
        self._info = (MSetInfo * max_batch)()
        self._nq = 0
        self._batch = None

    def close(self):
        if self._h:
            lib().xgm_searcher_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, batch: QueryBatch, background: bool = False):
        """Plan + enqueue a batch.  background=True hands the host half to the searcher's worker thread
        (xgm_search_submit_async); call launched() before enqueuing dependent work on stream()."""
        if background:
            _check(lib().xgm_search_submit_async(self._h, batch.arr, batch.n))
        else:
            _check(lib().xgm_search_submit(self._h, batch.arr, batch.n))
        self._batch = batch  # keeps the query array and term strings alive until wait
        self._nq = batch.n

    def launched(self):
        _check(lib().xgm_search_launched(self._h))

    def results_on_device(self, on: bool = True):
        """Leave results in the device slab (multi-GPU exchange + merge); wait_device() then only synchronises."""
        _check(lib().xgm_searcher_set_results_on_device(self._h, int(on)))

    def wait_device(self):
        _check(lib().xgm_search_wait(self._h, None, None, None, self.max_topk, None))

    def wait_raw(self):
        """Results left in the searcher's flat host buffers (stride = max_topk)."""
        _check(lib().xgm_search_wait(self._h, _ptr(self._docids), _ptr(self._weights), _ptr(self._keys),
                                     self.max_topk, self._info))
        return self._docids, self._weights, self._keys, self._info

    def wait(self) -> List[MSet]:
        d, w, k, info = self.wait_raw()
        out = []
        for i in range(self._nq):
            m = info[i]
            a, b = i * self.max_topk, i * self.max_topk + m.n
            out.append(MSet(d[a:b].copy(), w[a:b].copy(), k[a:b].copy(), m.first, m.matches_lower_bound,
                            m.matches_estimated, m.matches_upper_bound, m.max_possible, m.max_attained,
                            m.percent_scale_factor, m.exact_matches, m.status, m.flags))
        return out

    def search(self, queries: Union[QueryBatch, Sequence[Query]]) -> List[MSet]:
        if not isinstance(queries, QueryBatch) and len(queries) > self.max_batch:
            out: List[MSet] = []  # split into max_batch chunks
            for a in range(0, len(queries), self.max_batch):
                out += self.search(queries[a:a + self.max_batch])
            return out
        batch = queries if isinstance(queries, QueryBatch) else QueryBatch(queries)
        if batch.n <= self.max_batch:
            self.submit(batch)
            return self.wait()
        raise XgmError(E_INVALID, "batch larger than searcher max_batch")

    def replay(self):
        _check(lib().xgm_search_replay(self._h))

    def stream(self) -> int:
        return lib().xgm_searcher_stream(self._h) or 0

    def last_stats(self) -> BatchStats:
        o = BatchStats()
        _check(lib().xgm_search_last_stats(self._h, C.byref(o)))
        return o

    def device_results(self):
        w, d, c, s = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint32()
        _check(lib().xgm_search_device_results(self._h, C.byref(w), C.byref(d), C.byref(c), C.byref(s)))
        return w.value, d.value, c.value, s.value

    def device_slab(self):
        """(base pointer, bytes, docids offset, counts offset, stride) of the one-allocation result slab."""
        b, n, od, oc, s = C.c_void_p(), C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint32()
        _check(lib().xgm_search_device_slab(self._h, C.byref(b), C.byref(n), C.byref(od), C.byref(oc), C.byref(s)))
        return b.value, n.value, od.value, oc.value, s.value

    def device_slab_keys(self) -> int:
        """Offset of the result slab's sort-key region (u64 per record, stride as device_slab's)."""
        ok = C.c_uint64()
        _check(lib().xgm_search_device_slab_keys(self._h, C.byref(ok)))
        return ok.value


def unshard(docids: np.ndarray, shard: int, nshards: int) -> np.ndarray:
    d = np.ascontiguousarray(docids, np.uint32).copy()
    lib().xgm_unshard(_ptr(d), len(d), shard, nshards)
    return d


def merge_msets(parts: Sequence[MSet], first: int, maxitems: int, sort_by: int = SORT_REL,
                sort_reverse: bool = False) -> MSet:
    """Matcher::merge_mset over per-shard MSets whose docids were already unsharded."""
    n = len(parts)
    dptr = (C.c_void_p * n)()
    wptr = (C.c_void_p * n)()
    kptr = (C.c_void_p * n)()
    infos = (MSetInfo * n)()
    keep = []
    for i, p in enumerate(parts):
        d = np.ascontiguousarray(p.docids, np.uint32)
        w = np.ascontiguousarray(p.weights, np.float64)
        k = np.ascontiguousarray(p.sort_keys if p.sort_keys is not None and len(p.sort_keys) == len(d)
                                 else np.zeros(len(d), np.uint64), np.uint64)
        keep += [d, w, k]
        dptr[i], wptr[i], kptr[i] = d.ctypes.data, w.ctypes.data, k.ctypes.data
        m = infos[i]
        m.n, m.first = len(d), 0
        m.matches_lower_bound = m.uncollapsed_lower_bound = p.matches_lower_bound
        m.matches_estimated = m.uncollapsed_estimated = p.matches_estimated_raw
        m.matches_upper_bound = m.uncollapsed_upper_bound = p.matches_upper_bound
        m.exact_matches, m.status, m.flags = p.exact_matches, p.status, p.flags
        m.max_possible, m.max_attained = p.max_possible, p.max_attained
        m.percent_scale_factor = p.percent_scale_factor
    od = np.zeros(maxitems, np.uint32)
    ow = np.zeros(maxitems, np.float64)
    ok = np.zeros(maxitems, np.uint64)
    oi = MSetInfo()
    _check(lib().xgm_merge_msets(dptr, wptr, kptr, infos, n, first, maxitems, sort_by, int(sort_reverse),
                                 _ptr(od), _ptr(ow), _ptr(ok), C.byref(oi)))
    return MSet(od[:oi.n], ow[:oi.n], ok[:oi.n], first, oi.matches_lower_bound, oi.matches_estimated,
                oi.matches_upper_bound, oi.max_possible, oi.max_attained, oi.percent_scale_factor,
                oi.exact_matches, oi.status, oi.flags)


def merge_device_slabs(gathered, slab_bytes: int, off_docids: int, off_counts: int, off_keys: int, orders,
                       nparts: int, nq: int, stride: int, first: int, maxitems: int, stream=None):
    """xgm_merge_mset_device_slab over nparts gathered result slabs (a CUDA tensor, slab p at byte p * slab_bytes):
    Matcher::merge_mset of every query under its own order.  orders: a CUDA uint8 tensor [nq] (bits 0-1 the query's
    SORT_*, bit 2 its sort_reverse) or None for relevance order everywhere.  Returns (counts, docids, weights, keys)
    as CUDA tensors: int32 [nq] (UINT32_MAX, i.e. -1, for a query some part lost), int32 [nq, maxitems] (the
    uint32 docids' bits), float64 and int64 [nq, maxitems] (the uint64 keys' bits); entries past a query's count,
    and the keys of queries ordered by relevance, are zero.  Runs on `stream` (a cudaStream_t as int) or the
    current torch stream."""
    import torch
    dev = gathered.device
    counts = torch.zeros(nq, dtype=torch.int32, device=dev)
    docids = torch.zeros((nq, maxitems), dtype=torch.int32, device=dev)
    weights = torch.zeros((nq, maxitems), dtype=torch.float64, device=dev)
    keys = torch.zeros((nq, maxitems), dtype=torch.int64, device=dev)
    if orders is not None and (orders.dtype != torch.uint8 or orders.numel() != nq or not orders.is_contiguous()
                               or orders.device != dev):
        raise ValueError("orders must be a contiguous uint8 tensor of nq entries on the slabs' device")
    if stream is None:
        stream = torch.cuda.current_stream(dev).cuda_stream
    _check(lib().xgm_merge_mset_device_slab(gathered.data_ptr(), slab_bytes, off_docids, off_counts, off_keys,
                                            None if orders is None else orders.data_ptr(), nparts, nq, stride, first,
                                            maxitems, weights.data_ptr(), docids.data_ptr(), keys.data_ptr(),
                                            counts.data_ptr(), stream or None))
    return counts, docids, weights, keys


def value_key(b: bytes):
    """(key, exact): the device's 8-byte big-endian key of a serialised slot value (include/xgm.h)."""
    k = C.c_uint64()
    exact = lib().xgm_value_key(b, len(b), C.byref(k))
    return int(k.value), bool(exact)


def value_key_bytes(key: int) -> bytes:
    buf = C.create_string_buffer(8)
    n = lib().xgm_value_key_bytes(key, buf)
    return buf.raw[:n]


def sort_key_bytes(key: int, reverse: bool) -> bytes:
    """MSetIterator::get_sort_key under Xapiand's Multi_MultiValueKeyMaker with one SerialiseKey slot."""
    buf = C.create_string_buffer(20)
    n = lib().xgm_sort_key_bytes(key, int(reverse), buf)
    return buf.raw[:n]
