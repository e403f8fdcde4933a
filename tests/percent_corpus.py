"""A corpus built for the percentage scale: percent_scale_factor = 100 * subqs / nweighted / max_attained, where
subqs is the number of subqueries matching the FIRST document in docid order that attains max_attained
(ProtoMSet::update_max_weight).  Written as an XGMFLAT1 file (tests/flatfile.write_flat) with the slot-0 values
beside it, so the CUDA index and the oracle load the very same postings and values.

What it holds (tests/test_percent_corpus.py pins each witness with the oracle and numpy alone):
  W1 fa fb fc / ma mb mc
                 OR sets whose best weight is tied, bit for bit, by TIE documents with different numbers of matching
                 leaves.  The three leaves of a set have one termfreq, so one termweight; factors W1_FACTORS make the
                 first leaf weigh twice the others, exactly (a power-of-two scale), so a document holding the first
                 leaf alone weighs what one holding the other two does when wdf and length are equal.  The TIE
                 documents have length TIE_LEN and wdf TIE_WDF; every other posting has wdf <= 3 and length >= 2000,
                 so nothing else reaches that weight.  In the f set the lowest tie docid holds one leaf and the other
                 four hold two; in the m set the reverse.  The lowest docid's count is unique among the ties, so any
                 other choice of tie document gives another percentage.
     r_few r_more + y25 y5a y5b
                 the same for OP_AND_MAYBE, whose optional leaves take no factor: the collection has NDOCS = 39038
                 documents, so termfreq 1501 makes idf log(25) and termfreq 6506 log(5), and log(25) == 2 * log(5)
                 exactly.  r_few / r_more are the AND base with r_wide (a second base list with a bitmap).
  W2             the tie documents are kept out of value-sorted MSets in more than one way: the lowest tie docid and
                 two others carry the middle value MID_VALUE (past k in either direction: hundreds of matches have
                 values on each side), two carry no value (sorted last by the key of a missing value).
  W3             the f set under k1 = 0: every posting weighs its termweight, so all of fa's documents and the
                 fb + fc ties share the best weight, far more than the raise log (64 entries) holds.
  W4 pa pb pc pz large lists; pa is weighted 20 in the queries and its HEAVY documents (wdf 30, length TIE_LEN,
                 no pb / pc / pz) top every relevance order, so the best document matches fewer leaves than the query
                 has.  Document lengths spread over BASE_LEN, so that few of these lists' documents share a weight:
                 value-sorted queries over them keep a short raise log.  pz is weighted 1e-3 in the
                 queries, so MaxScore skips its work items.  w_all is a large second AND base list.
  wide g0 .. g9  fillers for 6..13-leaf ORs, in a pool of their own; g0 and g1 have no membership bitmap.
  groups         z_bool (boolean, wdf 0) holds every tie document; z_not holds none of them.
Docids have gaps: NDOCS of LASTDOCID are used, and LASTDOCID is not a multiple of 32 or 256.
"""
import os

import numpy as np

from tests.flatfile import write_flat

LASTDOCID = 41017
NDOCS = 39038                        # with termfreqs 1501 / 6506 this gives the idfs log(25) / log(5)
BITMAP_MIN = max(64, LASTDOCID // 256)
BASE_LEN = (2000, 5900)              # wide, and above min_normlen * average length: few documents share a weight
TIE_LEN, TIE_WDF = 40, 8
NTIE = 5                             # tie documents per set
OR_TF = 600
W1_OR_SETS = {"fewer": ("fa", "fb", "fc"), "more": ("ma", "mb", "mc")}  # lowest tie docid has fewer / more leaves
W1_FACTORS = (2.0, 1.0, 1.0)
R_TF, R_WIDE_TF, R_SINGLE = 600, 9000, 30
Y25_TF, Y5_TF = 1501, 6506
W1_MAYBE_SETS = {"fewer": (("r_few", "r_wide"), ("y25", "y5a", "y5b")),
                 "more": (("r_more", "r_wide"), ("y25", "y5a", "y5b"))}
P_TF, PZ_TF, W_ALL_TF, HEAVY, HEAVY_WDF = 12000, 15000, 30000, 5, 30
W4_OR_SETS = (("pa", "pb", "pc"), ("pa", "pb", "pc", "pz"))
W4_OR_FACTORS = {3: (20.0, 1.0, 1.0), 4: (20.0, 1.0, 1.0, 1e-3)}
W4_MAYBE = (("pa", "w_all"), ("pb", "pc"))
W4_MAYBE_FACTORS = (20.0, 1.0)
G_DF = (100, 140, 200, 300, 400, 600, 900, 1300, 2000, 3000)
G_NAMES = tuple(f"g{k}" for k in range(len(G_DF)))
G_POOL = 10000
FILLER_FACTOR = 0.25
WIDE_SETS = (W1_OR_SETS["fewer"] + G_NAMES[:3],                  # 6 leaves, two without a bitmap
             W1_OR_SETS["more"] + G_NAMES[3:],                    # 10
             W1_OR_SETS["fewer"] + G_NAMES)                       # 13
BOOL_DF, NOT_DF = 20000, 3000
MID_VALUE, VALUE_MAX, MISSING_SHARE = 500000, 1000000, 0.1
RANGE = (300000, 700000)             # a value range that holds MID_VALUE
MISSING_FWD = 0xFF << 56             # xgm_value_key("\xff"): SerialiseKey's missing value in a forward sort
MISSING_REV = 0                      # the empty string: last in a reverse sort


def wide_factors(names):
    return list(W1_FACTORS) + [FILLER_FACTOR] * (len(names) - 3)


def missing_key(reverse):
    """The key of a document without a value that sorts it after every valued document."""
    return MISSING_REV if reverse else MISSING_FWD


def build(seed=23):
    """(doclen indexed by docid, [(name, docids, wdfs)] sorted by name, nvals[lastdocid + 1],
    vals[lastdocid + 1, 3], {set key: tie docids ascending})."""
    rng = np.random.default_rng(seed)
    alive = np.sort(rng.choice(np.arange(1, LASTDOCID + 1), size=NDOCS, replace=False)).astype(np.uint32)
    perm = rng.permutation(alive)
    # an OR set's pool: its ties, then singles of the lone leaf and of the two paired leaves
    sizes = [NTIE + (OR_TF - 1) + 2 * (OR_TF - (NTIE - 1)), NTIE + (OR_TF - (NTIE - 1)) + 2 * (OR_TF - 1), 2 * R_TF,
             HEAVY, G_POOL]
    f_pool, m_pool, r_pool, heavy, g_pool, rest = np.split(perm, np.cumsum(sizes))
    terms = {}
    total = np.zeros(LASTDOCID + 1, np.int64)
    doclen = np.zeros(LASTDOCID + 1, np.int64)
    doclen[alive] = rng.integers(BASE_LEN[0], BASE_LEN[1] + 1, size=NDOCS)
    ties = {}

    def add(name, d, w):
        d = np.asarray(d, np.uint32)
        o = np.argsort(d)
        d, w = d[o], np.asarray(w, np.uint32)[o]
        assert len(np.unique(d)) == len(d), name
        terms[name] = (d, w)
        total[d] += w

    def small(n):
        return rng.integers(1, 4, size=n)

    def pick(pool, k, exclude=()):
        pool = np.setdiff1d(pool, np.concatenate([np.asarray(e, np.uint32) for e in exclude])) if exclude else pool
        return rng.choice(pool, size=k, replace=False).astype(np.uint32)

    # W1 OR sets: NTIE tie documents, then singles that pad every leaf to OR_TF
    for key, pool in (("fewer", f_pool), ("more", m_pool)):
        a, b, c = W1_OR_SETS[key]
        tie = np.sort(pool[:NTIE])
        ties[key] = tie
        lone, pair = (tie[:1], tie[1:]) if key == "fewer" else (tie[1:], tie[:1])
        singles = pool[NTIE:]
        na, nb = OR_TF - len(lone), OR_TF - len(pair)
        sa, sb, sc = np.split(singles, [na, na + nb])
        assert len(sc) == nb
        add(a, np.concatenate([lone, sa]), np.concatenate([np.full(len(lone), TIE_WDF), small(na)]))
        for name, s in ((b, sb), (c, sc)):
            add(name, np.concatenate([pair, s]), np.concatenate([np.full(len(pair), TIE_WDF), small(nb)]))
        doclen[tie] = TIE_LEN
    # W1 AND_MAYBE sets: the base r_x + r_wide; the optional leaves y25 (idf log 25) and y5a, y5b (idf log 5)
    r_few, r_more = np.split(r_pool, 2)
    y = {"y25": [], "y5a": [], "y5b": []}
    for key, r in (("fewer", r_few), ("more", r_more)):
        order = rng.permutation(r)
        tie = np.sort(order[:NTIE])
        ties["maybe_" + key] = tie
        lone, pair = (tie[:1], tie[1:]) if key == "fewer" else (tie[1:], tie[:1])
        y["y25"].append(lone)
        y["y5a"].append(pair)
        y["y5b"].append(pair)
        y["y5a" if key == "fewer" else "y5b"].append(order[NTIE:NTIE + R_SINGLE])  # lower weights, one leaf
        rw = small(R_TF)
        rw[np.isin(r, tie)] = 3
        add(W1_MAYBE_SETS[key][0][0], r, rw)
        doclen[tie] = TIE_LEN
    r_all = np.concatenate([r_few, r_more])
    rw = small(len(r_pool) + R_WIDE_TF - len(r_all))
    rd = np.concatenate([r_all, pick(rest, R_WIDE_TF - len(r_all))])
    rw[np.isin(rd, np.concatenate([ties["maybe_fewer"], ties["maybe_more"]]))] = 3
    add("r_wide", rd, rw)
    for name, tf in (("y25", Y25_TF), ("y5a", Y5_TF), ("y5b", Y5_TF)):
        mine = np.concatenate(y[name])
        wd = np.where(np.isin(mine, np.concatenate([ties["maybe_fewer"], ties["maybe_more"]])), TIE_WDF,
                      small(len(mine)))
        extra = pick(rest, tf - len(mine))
        add(name, np.concatenate([mine, extra]), np.concatenate([wd, small(len(extra))]))
    # W4: large lists; pa's heavy documents hold nothing else the W4 queries name but w_all
    add("pa", np.concatenate([heavy, pick(rest, P_TF)]), np.concatenate([np.full(HEAVY, HEAVY_WDF), small(P_TF)]))
    for name in ("pb", "pc"):
        add(name, pick(rest, P_TF), small(P_TF))
    add("pz", pick(rest, PZ_TF), small(PZ_TF))
    add("w_all", np.concatenate([heavy, pick(np.setdiff1d(alive, heavy), W_ALL_TF - HEAVY)]), small(W_ALL_TF))
    doclen[heavy] = TIE_LEN
    for name, df in zip(G_NAMES, G_DF):
        add(name, pick(g_pool, df), small(df))
    every_tie = np.concatenate(list(ties.values()))
    add("z_bool", np.concatenate([every_tie, pick(alive, BOOL_DF - len(every_tie), exclude=[every_tie])]),
        np.zeros(BOOL_DF, np.uint32))
    w1_docs = np.concatenate([f_pool, m_pool, r_pool])
    add("z_not", pick(w1_docs, NOT_DF, exclude=[every_tie]), np.ones(NOT_DF, np.uint32))

    # BM25's per-term bound relies on doclen >= wdf; the tie and heavy documents keep their short length
    assert (total[doclen == TIE_LEN] <= TIE_LEN).all()
    doclen[alive] = np.maximum(doclen[alive], total[alive])
    # slot 0: one value per document (or none); the tie documents: the middle value, or none (W2)
    nvals = (rng.random(LASTDOCID + 1) >= MISSING_SHARE).astype(np.uint8)
    nvals[0] = 0
    nvals[np.setdiff1d(np.arange(LASTDOCID + 1), alive)] = 0
    vals = np.zeros((LASTDOCID + 1, 3), np.uint64)
    vals[:, 0] = rng.integers(0, VALUE_MAX, size=LASTDOCID + 1)
    for tie in ties.values():
        nvals[tie] = 1
        vals[tie, 0] = MID_VALUE
        nvals[tie[[1, 3]]] = 0
    vals[nvals == 0, 0] = 0
    return doclen.astype(np.uint32), sorted((n, d, w) for n, (d, w) in terms.items()), nvals, vals, ties


def write_percent_corpus(tmp, seed=23):
    """Write the corpus under tmp; returns (path, term names in id order, nvals, vals, ties)."""
    doclen, terms, nvals, vals, ties = build(seed)
    path = os.path.join(tmp, "percent.flat")
    write_flat(path, doclen, terms)
    return path, [t[0] for t in terms], nvals, vals, ties


def device_slot(nvals, vals):
    """Slot 0 as xgm_builder_add_value_slot takes it: (voff[lastdocid + 2], keys).  A key is the value plus one,
    which is what the oracle's key-maker mode compares, so key 0 is free for documents without a value."""
    voff = np.zeros(len(nvals) + 1, np.uint64)
    voff[1:] = np.cumsum(nvals.astype(np.uint64))
    keys = vals[nvals > 0, 0].astype(np.uint64) + 1
    return voff, keys
