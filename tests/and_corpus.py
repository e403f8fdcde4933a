"""A corpus built so that a slightly wrong weight sum in the AND kernels changes the result bits: which wdf is read,
which leaves are summed, and where the weighted range source joins the sum.  Written as an XGMFLAT1 file
(tests/flatfile.write_flat) with slot-0 values beside it, so the CUDA index and the oracle see the same postings.

Every weighted list holds the core documents CORE, so each AND of weighted lists matches at least CORE (about 100
documents, which a top-100 MSet shows in full).  What it holds (tests/test_and_corpus.py pins each witness with the
oracle alone):
  W1 z_rare z_freq    boolean terms (wdf 0) as Document::add_boolean_term writes them; z_rare is rarer than every
                      weighted list (an OP_FILTER term that drives the AND), z_freq has a bitmap.  Both hold the
                      documents of length 0 (ZERO), which hold nothing else.  Under k1 = 0 a wdf-0 sumpart is 0 / 0.
  W2 slot 0           VALUE_FREQ documents have a value, between the termfreqs of p_coarse and p_fine: the range source
                      sorts in at every place 0 .. n of the 1- to 3-term bases in SRC_SETS
  W3 m00 .. m14       termfreq 2^(k+1): an OrPostList tree over 9..15 of them is deeper than 8; the ALL_MAYBE
                      documents of CORE hold every one
  W4 every list       wdf 1 + (i + off) % 7 at posting i, times 40 at every 13th: no wdf equals a neighbour's.  CORE
                      holds docids 256g - 1, 256g, 256g + 1 and 32w - 1, 32w; the probe lists are laid out so that
                      CORE documents sit at the first and last posting of 128-posting blocks
  W5 n_bm1 n_bm2 n_bm3 n_nobm
                      AND_NOT lists with and without a bitmap, each holding some CORE documents
Docids have gaps, and LASTDOCID is not a multiple of 32, 256 or 65536.
"""
import os

import numpy as np

from oracle import oracle as O
from tests.flatfile import write_flat

LASTDOCID = 70003
NDOCS = 60000
BLOCK = 128
BITMAP_MIN = max(64, LASTDOCID // 256)  # termfreq that earns a membership bitmap (XGM_BITMAP_K = 256)
MID_BITMAP_K = 30                       # XGM_BITMAP_K at which p_coarse loses its bitmap and p_fine keeps it
ZERO_DOCS = 200
VALUE_FREQ = 2000
VALUE_MAX = 1000000
ALL_MAYBE = 2
M_LEAVES = 15
# weighted lists: extra postings beyond CORE
EXTRA = dict(b_drv=0, p_nobm=140, b_drvbm=250, p_coarse=600, p_fine=5900, p_big=19900, p_huge=34900)
NOT_DF = dict(n_bm1=5000, n_bm2=3000, n_bm3=1500, n_nobm=150)
M_NAMES = tuple(f"m{k:02d}" for k in range(M_LEAVES))
# bases of the W2 witnesses: the source sorts in at 0 .. len(base)
SRC_SETS = (("b_drv",), ("p_big",), ("b_drv", "p_coarse"), ("b_drv", "p_fine"), ("p_fine", "p_big"),
            ("b_drv", "b_drvbm", "p_coarse"), ("b_drv", "p_coarse", "p_fine"), ("b_drv", "p_fine", "p_big"),
            ("p_fine", "p_big", "p_huge"))
SRC_FACTORS = (1e-3, 1 / 3)


def m_df(k):
    return 2 ** (k + 1)


def wdf_pattern(n, off):
    i = np.arange(n) + off
    return ((1 + i % 7) * np.where(i % 13 == 0, 40, 1)).astype(np.uint32)


def core_docids(alive):
    g = np.arange(1, LASTDOCID // 256 + 1, 11)
    w = np.arange(5, LASTDOCID // 32, 173)
    want = np.concatenate([256 * g - 1, 256 * g, 256 * g + 1, 32 * w - 1, 32 * w])
    return np.intersect1d(want, alive).astype(np.uint32)


def lay_out(core, extra, pool, rng):
    """CORE plus `extra` documents of pool, the fillers between two CORE documents chosen so that the later one sits
    at the first or last posting of a block where that takes few extra fillers."""
    density = extra / max(1, len(pool))
    pool = np.setdiff1d(pool, core)
    out, idx, prev = [], 0, 0
    for c in core:
        gap = pool[(pool > prev) & (pool < c)]
        natural = min(len(gap), int(round(density * len(gap))))
        # nearest block edge at or after idx + natural: 128k - 1 or 128k
        b = idx + natural
        edge = (b // BLOCK) * BLOCK + (BLOCK - 1 if b % BLOCK else 0)
        if edge < b:
            edge += 1
        need = edge - idx
        take = need if need <= len(gap) and need - natural <= max(3, natural) else natural
        out.append(rng.choice(gap, size=take, replace=False) if take else gap[:0])
        out.append(np.array([c], np.uint32))
        idx += take + 1
        prev = c
    rest = pool[pool > prev]
    left = max(0, len(core) + extra - idx)
    out.append(rng.choice(rest, size=min(left, len(rest)), replace=False))
    return np.sort(np.concatenate(out)).astype(np.uint32)


def build(seed=5):
    """(doclen, [(name, docids, wdfs)] sorted by name, doccount, nvals, vals, groups) where groups holds CORE, ZERO
    and ALL_MAYBE."""
    rng = np.random.default_rng(seed)
    alive = np.sort(rng.choice(np.arange(1, LASTDOCID + 1), size=NDOCS, replace=False)).astype(np.uint32)
    if alive[-1] != LASTDOCID:
        alive[-1] = LASTDOCID
    core = core_docids(alive)
    zero = np.sort(rng.choice(np.setdiff1d(alive, core), size=ZERO_DOCS, replace=False)).astype(np.uint32)
    weighted_pool = np.setdiff1d(alive, zero)
    terms = {}
    total = np.zeros(LASTDOCID + 1, np.int64)

    def add(name, d, w):
        d = np.asarray(d, np.uint32)
        assert len(np.unique(d)) == len(d) and (np.diff(d) > 0).all(), name
        terms[name] = (d, np.asarray(w, np.uint32))
        total[d] += terms[name][1]

    off = 0
    for name, extra in EXTRA.items():
        d = lay_out(core, extra, weighted_pool, rng) if extra else core
        add(name, d, wdf_pattern(len(d), off))
        off += 3
    all_maybe = core[::len(core) // ALL_MAYBE][:ALL_MAYBE]
    for k, name in enumerate(M_NAMES):
        d = np.union1d(all_maybe, rng.choice(np.setdiff1d(weighted_pool, all_maybe), size=m_df(k) - ALL_MAYBE,
                                             replace=False))
        add(name, d, wdf_pattern(len(d), off))
        off += 3
    for j, (name, df) in enumerate(NOT_DF.items()):
        some_core = core[j::7]
        others = rng.choice(np.setdiff1d(weighted_pool, core), size=df - len(some_core), replace=False)
        d = np.union1d(some_core, others)
        add(name, d, wdf_pattern(len(d), off))
        off += 3
    z_rare = np.union1d(core[::2][:50], zero[:30])
    add("z_rare", z_rare, np.zeros(len(z_rare), np.uint32))
    z_freq = np.union1d(np.union1d(core, zero), rng.choice(np.setdiff1d(alive, core), size=8000, replace=False))
    add("z_freq", z_freq, np.zeros(len(z_freq), np.uint32))

    doclen = np.zeros(LASTDOCID + 1, np.int64)
    doclen[alive] = total[alive] + rng.integers(1, 301, size=len(alive))
    doclen[zero] = 0
    assert (total[zero] == 0).all() and (doclen[alive] >= total[alive]).all()
    # slot 0: one value on VALUE_FREQ documents, every CORE document among them
    nvals = np.zeros(LASTDOCID + 1, np.uint8)
    valued = np.union1d(core, rng.choice(np.setdiff1d(alive, core), size=VALUE_FREQ - len(core), replace=False))
    nvals[valued] = 1
    vals = np.zeros((LASTDOCID + 1, 3), np.uint64)
    vals[valued, 0] = rng.integers(0, VALUE_MAX, size=len(valued))
    groups = dict(core=core, zero=zero, all_maybe=all_maybe)
    return (doclen.astype(np.uint32), sorted((n, d, w) for n, (d, w) in terms.items()), len(alive), nvals, vals,
            groups)


def write_and_corpus(tmp, seed=5):
    """Write the corpus under tmp; returns (path, build(seed))."""
    built = build(seed)
    doclen, terms, doccount = built[:3]
    path = os.path.join(tmp, "and.flat")
    write_flat(path, doclen, terms, doccount=doccount)
    return path, built


def spec(names, factors=None, filter_terms=(), not_terms=(), maybe=(), src=None, witness=""):
    """One witness query shape; src: the weighted range source's factor (None: no source)."""
    return dict(names=tuple(names), factors=factors, filter_terms=tuple(filter_terms), not_terms=tuple(not_terms),
                maybe=tuple(maybe), src=src, witness=witness)


def witness_specs():
    out = [  # W1: boolean FILTER terms as the driver and as a probe list, factor-0 leaves over wdf-0 postings
        spec(("b_drv", "p_fine"), filter_terms=("z_rare",), witness="W1"),
        spec(("b_drvbm", "p_coarse"), filter_terms=("z_rare",), witness="W1"),
        spec(("b_drv",), filter_terms=("z_freq",), witness="W1"),
        spec(("b_drv", "p_nobm"), filter_terms=("z_rare", "z_freq"), witness="W1"),
        spec(("z_rare", "p_fine"), factors=(0.0, 1.0), witness="W1"),
        spec(("b_drv", "z_freq"), factors=(1.0, 0.0), witness="W1"),
        spec(("b_drvbm", "z_freq", "p_big"), factors=(1.0, 0.0, 1.0), witness="W1"),
        spec(("z_rare", "z_freq"), factors=(0.0, 0.0), witness="W1"),
        spec(("z_rare",), factors=(0.0,), witness="W1"),
        spec(("z_freq",), factors=(0.0,), filter_terms=("z_rare",), witness="W1"),
    ]
    out += [spec(s, src=f, witness="W2") for s in SRC_SETS for f in SRC_FACTORS]
    out += [  # W3: 9..15 optional leaves
        spec(("b_drv",), maybe=M_NAMES, witness="W3"),
        spec(("b_drv", "p_fine"), maybe=M_NAMES[:14], witness="W3"),
        spec(("b_drvbm", "p_big"), maybe=M_NAMES[3:], witness="W3"),
        spec(("b_drv", "p_nobm"), maybe=M_NAMES[5:] + M_NAMES[:1], witness="W3"),
    ]
    out += [  # W4: drivers with and without a bitmap against probes with and without one
        spec(names, witness="W4") for names in (
            ("b_drv", "p_nobm"), ("b_drv", "p_coarse"), ("b_drv", "p_fine"), ("b_drvbm", "p_coarse"),
            ("b_drvbm", "p_nobm", "p_fine"), ("b_drv", "p_coarse", "p_fine", "p_big"), ("b_drvbm", "p_fine", "p_huge"),
            ("p_nobm",), ("p_coarse",), ("b_drv", "b_drvbm", "p_nobm", "p_coarse", "p_fine", "p_big", "p_huge"))]
    out += [  # W5: several excluded lists in one query
        spec(("b_drv", "p_fine"), not_terms=("n_bm1", "n_bm2", "n_bm3"), witness="W5"),
        spec(("b_drvbm", "p_coarse", "p_big"), not_terms=("n_bm3", "n_bm1"), witness="W5"),
        spec(("b_drv", "p_coarse"), not_terms=("n_bm2", "n_nobm", "n_bm1"), witness="W5"),
        spec(("b_drv",), not_terms=("n_nobm", "n_bm3"), filter_terms=("z_freq",), maybe=M_NAMES[:9], witness="W5"),
    ]
    return out


# k1 x b x min_normlen, with k3 = 1 so that k1 = b = min_normlen = 0 is not read as "use the defaults"
WEIGHTINGS = {f"k1={k1} b={b} mnl={m}": (k1, 1.0, b, m) for k1 in (0.0, 1.2, 20.0) for b in (0.0, 0.5, 1.0)
              for m in (0.0, 0.5)}
WEIGHTINGS.update({"k3=0 wqf": (1.2, 0.0, 0.75, 0.5), "k3=7 wqf factors": (1.2, 7.0, 0.75, 0.5)})
CELL_FACTORS = (2.5, 0.3, 0.0, 1.0)  # factors of the base leaves in the "factors" cell, in turn
CELL_WQF = (1, 3, 7)


def cell_spec(s, cell):
    """(factors, wqf) of spec s in a weighting cell: the factors cell weighs base leaves of witnesses without factors
    of their own by CELL_FACTORS, one leaf of each query left weighted."""
    n = len(s["names"])
    # the oracle weighs optional leaves at wqf 1: theirs stay 1, as do those of the unweighted groups
    rest = len(s["filter_terms"]) + len(s["not_terms"]) + len(s["maybe"])
    wqf = [CELL_WQF[j % 3] for j in range(n)] + [1] * rest if cell.endswith(("wqf", "factors")) else None
    fac = s["factors"]
    if fac is None and cell.endswith("factors") and n > 1:
        fac = tuple(CELL_FACTORS[j % 4] if j else 1.0 for j in range(n))
    return fac, wqf


def oracle_query(ids, s, cell, maxitems=100, first=0, check_at_least=0):
    fac, wqf = cell_spec(s, cell)
    kw = dict(first=first, maxitems=maxitems, check_at_least=check_at_least, factors=fac, wqf=wqf,
              bm25=WEIGHTINGS[cell])
    if s["src"] is not None:
        kw.update(filter=O.FILTER_MULTI_RANGE, range_lo=0, range_hi=VALUE_MAX, filter_weighted=True,
                  filter_factor=s["src"])
    return O.Query(op=O.OP_AND, terms=[ids[n] for n in s["names"]], filter_terms=[ids[n] for n in s["filter_terms"]],
                   not_terms=[ids[n] for n in s["not_terms"]], maybe_terms=[ids[n] for n in s["maybe"]], **kw)
