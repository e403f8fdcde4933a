"""A corpus built so that every MaxScore bound of the OR kernels is met or nearly met by documents the MSet needs:
a bound that is too small drops them, and only a comparison with the oracle notices.  Written as an XGMFLAT1 file
(tests/flatfile.write_flat), so the CUDA index and the oracle load the very same postings.

What it holds (tests/test_bound_corpus.py pins each witness with the oracle alone):
  W1 a_sat / b_pair   a_sat's blocks mostly hold wdf <= 20; five of its single-leaf documents have wdf 254, 255,
                      256, 1000 and 70000 (the block header keeps min(255, largest wdf)), and a band of two-leaf
                      documents (a_sat wdf 255 + b_pair wdf 1) weighs, under a large k1 with b = 0, between
                      sumpart(255) and the saturated documents: the tile kernel's threshold lands in that gap
  W2 m_x m_y m_d m_z  under k1 = 0 every posting weighs its leaf's termweight: with tie_factors() the m_d singles
                      (thousands, one weight) sit in the bucket of the m_x + m_y band, just above it
  W3 p_rare l_mid h_freq
                      weight order opposite to termfreq order by factors, wqf or global statistics; h_freq holds
                      documents with wdf 20 (with l_mid) and 21 (alone) that top the MSet
  W4 w_att            documents of length doclen_lb whose wdf is their block's largest: they meet the block bound
  W5 g00 .. g15       termfreq 2^(k+1): g00..g08 have no membership bitmap; 16 of them make the deepest OR tree
  z_bool              a boolean term (wdf 0), for FILTER / AND_NOT groups only (k1 = 0 makes a weighted wdf 0 a 0/0)
Docids have gaps: NDOCS of LASTDOCID are used, and LASTDOCID is not a multiple of 32, 256 or 65536.
"""
import math
import os

import numpy as np

from tests.flatfile import write_flat

LASTDOCID = 140003
NDOCS = 128000
DOCLEN_LB = 30                      # only the W4 documents are this short
BASE_LEN = (40, 200)                # everyone else: uniform in this range, raised to the sum of its wdfs
BITMAP_MIN = max(64, LASTDOCID // 256)  # termfreq that earns a membership bitmap
BLOCK = 128                         # postings per block

SAT_DF, SAT_WDFS = 20000, (254, 255, 256, 1000, 70000)
PAIR_BAND, PAIR_DF = 2000, 25000
M_BAND, M_X_ONLY, M_D_DF, M_Z_DF = 1500, 1500, 3000, 2000
P_DF, L_DF, H_DF, H_TOP = 3000, 9000, 40000, 300
W_DF, W4_DOCS, W4_WDF = 15000, 200, 5
BOOL_DF = 20000
G_LEAVES = 16

# query sets (leaf names); factors and statistics that go with them are built by the functions below
W1_SETS = (("a_sat", "b_pair"), ("a_sat", "b_pair", "w_att"))
W2_SET = ("m_d", "m_x", "m_y", "m_z")
W3_SET = ("p_rare", "l_mid", "h_freq")
W3_FACTORS = ((0.05, 1e-3, 3.25), (1e-3, 0.05, 3.25), (1e-3, 1e-3, 3.25))  # the largest on the most frequent leaf
W3_WQF = (1, 3, 7)
W4_SETS = (("w_att", "m_z"), ("w_att", "m_z", "m_d"))
W4_FACTOR = 1e-3                    # on the leaves after w_att: their singles stay below the W4 documents
G_NAMES = tuple(f"g{k:02d}" for k in range(G_LEAVES))
WIDE_SETS = (G_NAMES,                                            # 16 leaves
             G_NAMES[:9] + ("g12",),                             # 10: nine without a bitmap
             G_NAMES[3:],                                        # 13
             G_NAMES[1::2] + ("h_freq",),                        # 9
             G_NAMES[:6] + ("p_rare", "l_mid", "h_freq", "a_sat", "b_pair", "w_att", "m_d", "m_z", "g15"),  # 15
             ("g05", "p_rare", "l_mid", "h_freq", "a_sat", "g13"))  # 6: one without a bitmap


def g_df(k):
    return 2 ** (k + 1)


def build_terms(seed=11):
    """(doclen indexed by docid, [(name, docids, wdfs)] sorted by name)."""
    rng = np.random.default_rng(seed)
    alive = np.sort(rng.choice(np.arange(1, LASTDOCID + 1), size=NDOCS, replace=False)).astype(np.uint32)
    # disjoint pools where a structure needs documents that hold none of its query's other leaves; the W1 band is
    # a run of consecutive live docids, so that it fills few of a_sat's blocks
    band = alive[50000:50000 + PAIR_BAND]
    others = rng.permutation(np.concatenate([alive[:50000], alive[50000 + PAIR_BAND:]]))
    cut = np.cumsum([W4_DOCS, len(SAT_WDFS), M_BAND, M_X_ONLY, M_X_ONLY, M_D_DF, M_Z_DF])
    w4, sat1, mband, mx, my, md, mz, rest = np.split(others, cut)
    terms = {}
    total = np.zeros(LASTDOCID + 1, np.int64)

    def add(name, d, w):
        d = np.asarray(d, np.uint32)
        o = np.argsort(d)
        d, w = d[o], np.asarray(w, np.uint32)[o]
        assert len(np.unique(d)) == len(d), name
        terms[name] = (d, w)
        total[d] += w

    def pick(pool, k, exclude=()):
        pool = np.setdiff1d(pool, np.concatenate([np.asarray(e, np.uint32) for e in exclude])) if exclude else pool
        return rng.choice(pool, size=k, replace=False).astype(np.uint32)

    # W1: a band of consecutive docids (few blocks) holds both leaves; the saturated postings sit in single-leaf
    # documents spread over a_sat's list
    sat_rest = pick(rest, SAT_DF - PAIR_BAND - len(SAT_WDFS))
    a_d = np.concatenate([band, sat1, sat_rest])
    a_w = np.concatenate([np.full(PAIR_BAND, 255), np.array(SAT_WDFS), rng.integers(1, 21, size=len(sat_rest))])
    add("a_sat", a_d, a_w)
    b_rest = pick(rest, PAIR_DF - PAIR_BAND, exclude=[sat_rest])
    add("b_pair", np.concatenate([band, b_rest]), np.ones(PAIR_DF, np.uint32))
    # W2: wdf 1 everywhere, four disjoint populations besides the m_x + m_y band
    add("m_x", np.concatenate([mband, mx]), np.ones(M_BAND + M_X_ONLY, np.uint32))
    add("m_y", np.concatenate([mband, my]), np.ones(M_BAND + M_X_ONLY, np.uint32))
    add("m_d", md, np.ones(M_D_DF, np.uint32))
    add("m_z", mz, np.ones(M_Z_DF, np.uint32))
    # W3: h_freq's heaviest postings, half of them in documents with l_mid (which p_rare does not hold)
    p_d = pick(rest, P_DF)
    l_d = pick(rest, L_DF, exclude=[p_d])
    top_l = l_d[:H_TOP]
    top_h = pick(rest, H_TOP, exclude=[p_d, l_d])
    h_rest = pick(rest, H_DF - 2 * H_TOP, exclude=[top_l, top_h])
    add("p_rare", p_d, rng.integers(1, 4, size=P_DF))
    add("l_mid", l_d, rng.integers(1, 4, size=L_DF))
    add("h_freq", np.concatenate([top_l, top_h, h_rest]),
        np.concatenate([np.full(H_TOP, 20), np.full(H_TOP, 21), rng.integers(1, 4, size=len(h_rest))]))
    # W4: the short documents hold w_att alone, at the largest wdf of the list
    w_rest = pick(rest, W_DF - W4_DOCS)
    add("w_att", np.concatenate([w4, w_rest]),
        np.concatenate([np.full(W4_DOCS, W4_WDF), rng.integers(1, W4_WDF, size=len(w_rest))]))
    # W5
    for k, name in enumerate(G_NAMES):
        add(name, pick(rest, g_df(k)), rng.integers(1, 4, size=g_df(k)))
    add("z_bool", pick(np.concatenate([rest, band, md]).astype(np.uint32), BOOL_DF), np.zeros(BOOL_DF, np.uint32))

    doclen = np.zeros(LASTDOCID + 1, np.int64)
    doclen[alive] = np.maximum(rng.integers(BASE_LEN[0], BASE_LEN[1] + 1, size=NDOCS), total[alive])
    doclen[w4] = DOCLEN_LB
    # BM25's per-term bound (get_maxpart) relies on doclen >= wdf: every document's wdfs fit in its length
    assert (doclen[alive] >= total[alive]).all() and (total[doclen == 0] == 0).all()
    assert int(doclen[alive].min()) == DOCLEN_LB and (doclen[w4] == DOCLEN_LB).all()
    return doclen.astype(np.uint32), sorted((n, d, w) for n, (d, w) in terms.items())


def write_bound_corpus(tmp, seed=11):
    """Write the corpus under tmp; returns (path, term names in id order)."""
    doclen, terms = build_terms(seed)
    path = os.path.join(tmp, "bounds.flat")
    write_flat(path, doclen, terms)
    return path, [t[0] for t in terms]


def termweight_k1_0(n, tf):
    """BM25Weight::init's termweight at k1 = 0, factor 1 and wqf 1 (the oracle's orc_bm25_init): the idf alone."""
    tw = ((n - tf) + 0.5) / (tf + 0.5)
    return math.log(tw * 0.5 + 1 if tw < 2 else tw)


def tie_factors(termfreqs, n=NDOCS):
    """Factors of W2_SET for k1 = 0 (every posting weighs its termweight): m_d's termweight is that of the
    m_x + m_y band times 1 + 1e-4, m_z's 0.3 times it, so max_possible = 2.3 band weights and the band and the m_d
    singles share bucket floor(1024 / 2.3) = 445 (at 0.2 and 0.25 of its width)."""
    tf = dict(zip(W2_SET, termfreqs))
    band = termweight_k1_0(n, tf["m_x"]) + termweight_k1_0(n, tf["m_y"])
    return (band * (1 + 1e-4) / termweight_k1_0(n, tf["m_d"]), 1.0, 1.0, 0.3 * band / termweight_k1_0(n, tf["m_z"]))


def reversed_stats(termfreqs, total_length, n=NDOCS):
    """Global statistics (collection_size, total_length, termfreq per leaf) of a two-phase search whose termfreq
    order is the reverse of the local one: the locally rarest leaf gets the largest global termfreq."""
    asc = sorted(termfreqs)
    rank = np.argsort(np.argsort(termfreqs, kind="stable"), kind="stable")
    return (n, total_length, [asc[len(asc) - 1 - int(r)] for r in rank])


def w4_factors(names):
    """Factors of a W4 set: w_att weighs in full, the other leaves next to nothing."""
    return [1.0] + [W4_FACTOR] * (len(names) - 1)
