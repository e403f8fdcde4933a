"""A plain restatement of the multi-shard merge, the yardstick for both of the library's merges.

merge_ref is Matcher::merge_mset (matcher/matcher.cc:653-782) over per-shard MSets whose docids are still
shard-local: each part's docids are unsharded as unshard() does (backends/multi.h:66-70: part p of n holds
global docid (d - 1) * n + p + 1), the parts are merged by popping the best head under the reference's
ordering (matcher/msetcmp.cc), and the statistics are folded as MSet::Internal::merge_stats does
(api/mset.cc:376-395).  No percentage cut-off and no collapsing: the library has neither."""
from __future__ import annotations

import functools
import heapq
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

SORT_REL, SORT_VAL_REL, SORT_VAL, SORT_REL_VAL = 0, 1, 2, 3
SORT_DOCID = -1  # Enquire::Internal::DOCID: what REL becomes when every weight is zero


@dataclass
class Part:
    """One shard's MSet: docids shard-local, in the shard's own MSet order."""
    docids: Sequence[int]
    weights: Sequence[float]
    keys: Optional[Sequence[int]] = None
    lb: int = 0
    est: int = 0
    ub: int = 0
    max_possible: float = 0.0
    max_attained: float = 0.0
    percent_scale_factor: float = 0.0

    @classmethod
    def of_oracle(cls, m) -> "Part":
        return cls(m.docids.tolist(), m.weights.tolist(), m.sortvals.tolist(), m.lb, m.est, m.ub,
                   m.max_possible, m.max_attained, m.percent_scale_factor)

    @classmethod
    def of_xgm(cls, m) -> "Part":
        keys = m.sort_keys.tolist() if m.sort_keys is not None and len(m.sort_keys) == len(m.docids) else None
        return cls(m.docids.tolist(), m.weights.tolist(), keys, m.matches_lower_bound, m.matches_estimated_raw,
                   m.matches_upper_bound, m.max_possible, m.max_attained, m.percent_scale_factor)


@dataclass
class Merged:
    docids: list
    weights: list
    keys: list
    lb: int
    est: int
    ub: int
    max_possible: float
    max_attained: float
    percent_scale_factor: float


def msetcmp(sort_by: int, reverse: bool):
    """get_msetcmp_function(sort_by, sort_forward=True, sort_val_reverse=reverse): 'a ranks before b' over
    (weight, docid, key) triples.  Keys compare as the byte strings they stand for (the library's keys are
    order-preserving integers)."""
    def by_docid(a, b):
        return a[1] < b[1]

    def by_key(a, b):
        if a[2] > b[2]:
            return 1 if reverse else 0
        if a[2] < b[2]:
            return 0 if reverse else 1
        return None

    def by_weight(a, b):
        if a[0] > b[0]:
            return True
        if a[0] < b[0]:
            return False
        return None

    def before(a, b):
        steps = {SORT_DOCID: (), SORT_REL: (by_weight,), SORT_VAL: (by_key,), SORT_VAL_REL: (by_key, by_weight),
                 SORT_REL_VAL: (by_weight, by_key)}[sort_by]
        for step in steps:
            r = step(a, b)
            if r is not None:
                return bool(r)
        return by_docid(a, b)
    return before


def merge_ref(parts: Sequence[Part], first: int, maxitems: int, sort_by: int = SORT_REL,
              reverse: bool = False) -> Merged:
    n = len(parts)
    lb = est = ub = 0
    max_possible = max_attained = percent_scale_factor = 0.0
    for p in parts:  # merge_stats, in part order
        lb += p.lb
        est += p.est
        ub += p.ub
        max_possible = max(max_possible, p.max_possible)
        if p.max_attained > max_attained:
            max_attained, percent_scale_factor = p.max_attained, p.percent_scale_factor
    if max_possible == 0.0:  # every weight is zero: REL sorts by docid, REL_VAL and VAL_REL by value
        sort_by = {SORT_REL: SORT_DOCID, SORT_REL_VAL: SORT_VAL, SORT_VAL_REL: SORT_VAL}.get(sort_by, sort_by)
    if sort_by == SORT_REL:  # msetcmp_by_relevance as a tuple key: the sweeps of the device merge run it a lot
        key = lambda t: (-t[0], t[1])  # noqa: E731
    else:
        before = msetcmp(sort_by, reverse)
        key = functools.cmp_to_key(lambda a, b: -1 if before(a, b) else (1 if before(b, a) else 0))
    runs = []
    for pi, p in enumerate(parts):  # no part contributes more than first + maxitems items
        m = min(len(p.docids), first + maxitems)
        ks = p.keys if p.keys is not None else [0] * m
        runs.append([(float(w), (int(d) - 1) * n + pi + 1, int(k))
                     for d, w, k in zip(p.docids[:m], p.weights[:m], ks[:m])])
    out = []
    # heapq.merge pops the best head of the runs, as merge_mset's Heap of per-shard cursors does
    for item in heapq.merge(*runs, key=key):
        if len(out) == first + maxitems:
            break
        out.append(item)
    out = out[first:]
    return Merged([d for _, d, _ in out], [w for w, _, _ in out], [k for _, _, k in out], lb, est, ub,
                  max_possible, max_attained, percent_scale_factor)


def rel_top(docids: np.ndarray, weights: np.ndarray, counts: np.ndarray, k: int):
    """merge_ref's relevance-order docids and weights of ranks [0, k) for one query of the device merge's
    gathered layout: docids / weights [nparts][stride] (shard-local), counts [nparts]."""
    parts = [Part(docids[p, :min(c, k)].tolist(), weights[p, :min(c, k)].tolist(), max_possible=1.0)
             for p, c in enumerate(counts.tolist())]
    m = merge_ref(parts, 0, k)
    return m.docids, m.weights
