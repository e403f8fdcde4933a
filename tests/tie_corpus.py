"""A corpus built to make BM25 weights tie: a few document lengths and wdf 1 or 2, so every term contributes a
handful of distinct weights and large sets of matches share the top weight.  Written as an XGMFLAT1 file
(tests/flatfile.write_flat), so the CUDA index and the oracle load the very same postings.

What it holds (names ascending, as the flat format wants):
  b_bool        a boolean term (wdf 0 everywhere)
  eNNNNa/b      for every N in EDGE_SIZES, two wdf-1 terms whose intersection is exactly N documents
  f_flat        35k documents, wdf 1: the weight depends on the document length alone
  r_rare        fewer documents than the membership-bitmap threshold
  t01 .. t08    frequent terms (3k .. 37k documents), wdf 2 more often than 1
Docids have gaps: 40000 of 42000 are used.
"""
import os

import numpy as np

from tests.flatfile import write_flat

LASTDOCID = 42000
NDOCS = 40000
LENGTHS = (96, 128, 160)           # a document's length is one of these
LENGTH_P = (0.5, 0.3, 0.2)
EDGE_SIZES = (63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049)
EDGE_EXTRA = 2500                  # documents of each edge term outside the intersection
T_DF = (37000, 36000, 35000, 34000, 33000, 30000, 9000, 3000)
T_WDF2 = 0.85                      # share of a t-term's postings with wdf 2
FLAT_DF = 35000
BOOL_DF = 20000
RARE_DF = 100


KEEP_CAP = 2048                    # survivors the top-k kernel holds in shared memory when max_topk <= 256

# Tie-heavy query sets, one per matching route: (operator, base terms, OP_SCALE_WEIGHT factors or None).
# Each one's top weight is shared by more than KEEP_CAP matches (tests/test_tie_corpus.py pins that).
TIE_ROUTES = {
    "single": [("AND", ["f_flat"], None), ("AND", ["t01"], None), ("AND", ["t03"], None)],
    "and2": [("AND", ["t01", "t02"], None), ("AND", ["t02", "t04"], None), ("AND", ["f_flat", "t01"], None)],
    "and3": [("AND", ["t01", "t02", "t03"], None), ("AND", ["t02", "t03", "t05"], None)],
    "or": [("OR", ["t01", "t02"], None), ("OR", ["t01", "t02", "t03"], None),
           ("OR", ["t02", "t03", "t04", "t05"], None), ("OR", ["t01", "t02", "t03", "t04", "t05"], None)],
    "or_wide": [("OR", ["t01", "t02", "t03", "t04", "t05", "t06"], None)],
    "and_zero": [("AND", ["t01", "t02"], [0.0, 0.0]), ("AND", ["t03", "t04", "t05"], [0.0, 0.0, 0.0])],
}


def edge_names(n):
    return f"e{n:04d}a", f"e{n:04d}b"


def build_terms(seed=7):
    """(doclen indexed by docid, [(name, docids, wdfs)] sorted by name)."""
    rng = np.random.default_rng(seed)
    alive = np.sort(rng.choice(np.arange(1, LASTDOCID + 1), size=NDOCS, replace=False)).astype(np.uint32)
    terms = []

    def pick(pool, k):
        return np.sort(rng.choice(pool, size=k, replace=False)).astype(np.uint32)

    for i, df in enumerate(T_DF):
        d = pick(alive, df)
        terms.append((f"t{i + 1:02d}", d, np.where(rng.random(df) < T_WDF2, 2, 1).astype(np.uint32)))
    d = pick(alive, FLAT_DF)
    terms.append(("f_flat", d, np.ones(FLAT_DF, np.uint32)))
    d = pick(alive, BOOL_DF)
    terms.append(("b_bool", d, np.zeros(BOOL_DF, np.uint32)))
    d = pick(alive, RARE_DF)
    terms.append(("r_rare", d, rng.integers(1, 3, size=RARE_DF).astype(np.uint32)))
    for n in EDGE_SIZES:
        perm = rng.permutation(alive)
        both, only_a, only_b = perm[:n], perm[n:n + EDGE_EXTRA], perm[n + EDGE_EXTRA:n + 2 * EDGE_EXTRA]
        a, b = edge_names(n)
        da = np.sort(np.concatenate([both, only_a])).astype(np.uint32)
        db = np.sort(np.concatenate([both, only_b])).astype(np.uint32)
        terms.append((a, da, np.ones(len(da), np.uint32)))
        terms.append((b, db, np.ones(len(db), np.uint32)))
    terms.sort(key=lambda t: t[0])
    doclen = np.zeros(LASTDOCID + 1, np.uint32)
    doclen[alive] = rng.choice(np.array(LENGTHS, np.uint32), size=NDOCS, p=LENGTH_P)
    # BM25's per-term bound relies on doclen >= wdf: every document's wdfs must fit in its length
    total = np.zeros(LASTDOCID + 1, np.uint64)
    for _, d, w in terms:
        total[d] += w
    assert int(total.max()) <= min(LENGTHS), "document lengths too small for the wdfs they hold"
    return doclen, terms


def write_tie_corpus(tmp, seed=7):
    """Write the corpus under tmp; returns (path, term names in id order)."""
    doclen, terms = build_terms(seed)
    path = os.path.join(tmp, "ties.flat")
    write_flat(path, doclen, terms)
    return path, [t[0] for t in terms]


# Value sorts on the oracle's synthetic value corpus with most documents lacking slot 0: the documents without
# a value share one sort key, and the keys below put that mass at the top of the order in either direction.
VALUE_NDOCS, VALUE_VOCAB, VALUE_MISSING_SHARE = 30000, 3000, 0.9
VALUE_AND_SETS = ([0, 1], [0, 2], [1, 2], [0, 1, 2])
VALUE_OR_SETS = ([0, 1], [1, 2, 3])


def missing_key(reverse):
    """Sort key of a document without a value: the empty string for a forward sort (what
    Enquire::set_sort_by_value does), the largest key for a reverse one."""
    return (1 << 64) - 1 if reverse else 0


def value_slot_arrays(orc, missing_share=VALUE_MISSING_SHARE, seed=5):
    """Drop slot-0 values of the oracle's synthetic value corpus (O.Index.synthetic(..., values=True)) from a
    random `missing_share` of its documents, in place, and return the slot as xgm_builder_add_value_slot takes
    it: (voff[lastdocid + 2], keys).  A key is the value plus one, which is what the oracle's key-maker mode
    compares (oracle/xgm_oracle.c sort_value), so key 0 is free for documents without a value."""
    nv, v0, _ = orc.values()
    last = orc.lastdocid
    rng = np.random.default_rng(seed)
    drop = rng.random(last + 1) < missing_share
    drop[0] = True
    nv[drop] = 0
    voff = np.zeros(last + 2, np.uint64)
    voff[1:] = np.cumsum(nv.astype(np.uint64))
    keys = np.concatenate([v0[d, :nv[d]] for d in range(last + 1)]).astype(np.uint64) + 1
    return voff, keys
