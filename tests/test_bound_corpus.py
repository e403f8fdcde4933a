"""Pins the corpus of tests/test_gpu_or_bounds.py with the oracle and numpy alone (no GPU): an edit to
tests/bound_corpus.py that took a witness away would leave the GPU tests passing without testing the bound it is
for.  A bucket is floor(w * 1024 / max_possible), the kernels' pruning histogram."""
import ctypes as C
import shutil
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import bound_corpus as B

NBINS = 1024


@pytest.fixture(scope="module")
def bound_oracle():
    tmp = tempfile.mkdtemp(prefix="xgm_bounds_")
    path, names = B.write_bound_corpus(tmp)
    yield {n: i for i, n in enumerate(names)}, O.Index.load_flat(path)
    shutil.rmtree(tmp, ignore_errors=True)


def weigh(orc, t, bm25, factor=1.0, wqf=1, stats=None):
    """(termweight, len_factor, maxpart) of leaf t as the oracle computes them; bm25 = (k1, k3, b, min_normlen)."""
    k1, k3, b, mnl = bm25
    coll, tlen, tf = stats if stats else (orc.doccount, orc.total_length, orc.termfreq(t))
    tw, lf = C.c_double(), C.c_double()
    O.lib().orc_bm25_init(coll, tlen, tf, wqf, factor, k1, k3, b, C.byref(tw), C.byref(lf))
    mp = O.lib().orc_bm25_maxpart(tw.value, lf.value, k1, b, mnl, int(orc.wdf_ub()[t]), orc.doclen_lb)
    return tw.value, lf.value, mp


def sumpart(bm25, tw, lf, wdf, length):
    k1, _, b, mnl = bm25
    return O.lib().orc_bm25_sumpart(tw, lf, k1, b, mnl, wdf, length)


def bucket(w, max_possible):
    return min(NBINS - 1, int(w * (NBINS / max_possible)))


def top(orc, ids, names, k, bm25=None, factors=None, wqf=None, stats=None, first=0):
    return orc.match(O.Query(op=O.OP_OR, terms=[ids[n] for n in names], maxitems=k, first=first, bm25=bm25,
                             factors=factors, wqf=wqf, stats=stats))


def test_corpus_shape(bound_oracle):
    ids, orc = bound_oracle
    assert orc.doccount == B.NDOCS and orc.lastdocid == B.LASTDOCID
    assert all(B.LASTDOCID % m for m in (32, 256, 65536)) and B.LASTDOCID > 2 * 65536
    dl = orc.doclen()
    assert orc.doclen_lb == B.DOCLEN_LB and int((dl == B.DOCLEN_LB).sum()) == B.W4_DOCS
    total = np.zeros(orc.lastdocid + 1, np.int64)
    for t in range(orc.nterms):
        d, w = orc.postings(t)
        total[d] += w
        if orc.name(t) != "z_bool":
            assert w.min() >= 1, orc.name(t)  # k1 = 0 would make a weighted wdf 0 a 0/0
    assert (total <= dl).all()
    bm = [orc.termfreq(ids[n]) >= B.BITMAP_MIN for n in B.G_NAMES]
    assert bm == [k >= 9 for k in range(B.G_LEAVES)]
    for s in B.WIDE_SETS:
        assert len(s) >= 6 and not all(orc.termfreq(ids[n]) >= B.BITMAP_MIN for n in s)


def block_max(w):
    """Largest wdf of each posting's block (128 consecutive postings)."""
    m = np.maximum.reduceat(w, np.arange(0, len(w), B.BLOCK))
    return np.repeat(m, B.BLOCK)[:len(w)]


@pytest.mark.parametrize("k1", [20.0, 100.0])
@pytest.mark.parametrize("names", B.W1_SETS)
def test_w1_saturated_blocks_hold_top_documents(bound_oracle, k1, names):
    """The top-k holds a single-leaf a_sat document from a block whose largest wdf is above 255, and both it and
    the k-th result lie above the bucket of sumpart(255): a block bound that trusted the saturated header byte
    would skip that block."""
    ids, orc = bound_oracle
    bm25 = (k1, 1.0, 0.0, 0.5)
    d, w = orc.postings(ids["a_sat"])
    bmax = dict(zip(d.tolist(), block_max(w).tolist()))
    others = set()
    for n in names[1:]:
        others |= set(orc.postings(ids[n])[0].tolist())
    tw, lf, _ = weigh(orc, ids["a_sat"], bm25)
    assert sorted(np.unique(block_max(w))[-6:].tolist())[-3:] == [256, 1000, 70000]
    assert int((block_max(w)[::B.BLOCK] <= 20).sum()) > 0.8 * len(w) / B.BLOCK
    for k in (1, 10, 100):
        r = top(orc, ids, names, k, bm25)
        wrong = bucket(sumpart(bm25, tw, lf, 255, orc.doclen_lb) * (1 + 1e-12), r.max_possible)
        sat = [(x, y) for x, y in zip(r.docids.tolist(), r.weights.tolist())
               if bmax.get(x, 0) > 255 and x not in others]
        assert sat, (k, names)
        assert all(bucket(y, r.max_possible) > wrong for _, y in sat)
        assert bucket(r.weights[-1], r.max_possible) > wrong, (k, names)


@pytest.mark.parametrize("bm25", [(0.0, 1.0, 0.5, 0.5), (0.0, 1.0, 1.0, 0.0), (1.2, 1.0, 0.0, 0.5)])
def test_w2_threshold_bucket_is_a_tie_mass(bound_oracle, bm25):
    """Under k1 = 0 (and under b = 0 with wdf 1 everywhere) the k-th weight is shared by more documents than k;
    with k1 = 0 those are the m_d singles, in the very bucket of the >= 1024 two-leaf band below them, which is
    where the tile kernel leaves the threshold."""
    ids, orc = bound_oracle
    fac = B.tie_factors([orc.termfreq(ids[n]) for n in B.W2_SET])
    band = orc.match(O.Query(op=O.OP_AND, terms=[ids["m_x"], ids["m_y"]], maxitems=5, check_at_least=B.NDOCS,
                             bm25=bm25, factors=fac[1:3]))
    assert band.exact >= 1024
    md = set(orc.postings(ids["m_d"])[0].tolist())
    for k in (1, 10, 100):
        r = top(orc, ids, B.W2_SET, k, bm25, factors=fac)
        full = top(orc, ids, B.W2_SET, B.NDOCS, bm25, factors=fac)
        assert int((full.weights == r.weights[-1]).sum()) > k
        if bm25[0] == 0.0:
            assert set(r.docids.tolist()) <= md
            assert bucket(r.weights[-1], r.max_possible) == bucket(band.weights[0], r.max_possible)
            assert band.weights[0] < r.weights[-1]


def w3_variants(orc, ids):
    """(bm25, factors, wqf, stats) of the W3 queries."""
    tfs = [orc.termfreq(ids[n]) for n in B.W3_SET]
    out = [((1.0, 1.0, 0.5, 0.5), f, None, None) for f in B.W3_FACTORS]
    out.append(((1.2, 7.0, 0.75, 0.5), None, B.W3_WQF, None))
    out.append(((1.2, 1.0, 0.75, 0.5), None, None, B.reversed_stats(tfs, orc.total_length)))
    return out


def test_w3_weight_order_opposes_termfreq_order(bound_oracle):
    """get_maxpart, recomputed with the oracle's formula, is not non-increasing in ascending-termfreq order: a skip
    that assumed 'later leaves weigh less' would drop documents."""
    ids, orc = bound_oracle
    order = sorted(B.W3_SET, key=lambda n: orc.termfreq(ids[n]))
    assert order == list(B.W3_SET)
    for bm25, fac, wqf, stats in w3_variants(orc, ids):
        mp = [weigh(orc, ids[n], bm25, fac[j] if fac else 1.0, wqf[j] if wqf else 1,
                    (stats[0], stats[1], stats[2][j]) if stats else None)[2] for j, n in enumerate(B.W3_SET)]
        assert any(mp[j] < mp[j + 1] for j in range(len(mp) - 1)), (bm25, fac, wqf, stats)
        assert fac is None or mp[-1] == max(mp)
    # the heaviest h_freq postings (wdf 20 with l_mid, 21 alone) make the top of the MSet under the first factors
    r = top(orc, ids, B.W3_SET, 100, (1.0, 1.0, 0.5, 0.5), factors=B.W3_FACTORS[0])
    hd, hw = orc.postings(ids["h_freq"])
    heavy = set(hd[hw >= 20].tolist())
    ld = set(orc.postings(ids["l_mid"])[0].tolist())
    got = set(r.docids.tolist())
    assert got <= heavy and got & ld and got - ld


def test_w4_block_bound_is_attained(bound_oracle):
    """Under b = 1 and min_normlen below doclen_lb * len_factor, a top-k document of length doclen_lb holding its
    block's largest wdf weighs exactly the block bound sumpart(tw, block max, doclen_lb)."""
    ids, orc = bound_oracle
    bm25 = (2.0, 1.0, 1.0, 0.0)
    d, w = orc.postings(ids["w_att"])
    bmax = dict(zip(d.tolist(), block_max(w).tolist()))
    tw, lf, _ = weigh(orc, ids["w_att"], bm25)
    assert bm25[3] < orc.doclen_lb * lf
    for names in B.W4_SETS:
        r = top(orc, ids, names, 10, bm25, factors=B.w4_factors(names))
        hit = [y for x, y in zip(r.docids.tolist(), r.weights.tolist())
               if x in bmax and y == sumpart(bm25, tw, lf, bmax[x], orc.doclen_lb)]
        assert hit, names


def stack_depth(prog):
    depth = best = 0
    for x in prog:
        depth += 1 if x >= 0 else -1
        best = max(best, depth)
    return best


def test_w5_sixteen_leaves_fill_the_or_program(bound_oracle):
    """Geometric termfreqs make OrContext's heap build a caterpillar: the 16-leaf postfix program has 31 entries
    and reaches stack depth 16."""
    ids, orc = bound_oracle
    tfs = [orc.termfreq(ids[n]) for n in B.G_NAMES]
    assert tfs == [B.g_df(k) for k in range(B.G_LEAVES)]
    prog = O.or_program(tfs)
    assert len(prog) == 2 * B.G_LEAVES - 1 and stack_depth(prog) == B.G_LEAVES


@pytest.mark.skipif(not O.have_reference(), reason="oracle/_ref not built")
def test_oracle_clamps_bm25_parameters_like_the_reference(tmp_path):
    """BM25Weight's constructor clamps k1, k3 < 0 to 0 and b to [0, 1]; the oracle weighs out-of-range
    parameters the same way (compiled reference, query lines with a BM25 clause)."""
    ndocs, vocab = 3000, 400
    info = O.ref_build(str(tmp_path / "db"), ndocs, vocab)
    assert info is not None
    orc = O.Index.synthetic(ndocs, vocab)
    cases = [("OR", [3, 17, 40], (1.2, 1.0, 1.5, 0.5)), ("OR", [5, 9], (1.2, 1.0, -0.5, 0.5)),
             ("AND", [1, 2], (-1.0, 1.0, 0.5, 0.5)), ("OR", [2, 30, 7], (1.2, -2.0, 0.75, 0.5)),
             ("TERM", [4], (-1.0, -2.0, 1.5, 0.0))]
    lines = [O.query_line(op, [orc.name(t) for t in ts], 0, 20, ndocs, bm25=p) for op, ts, p in cases]
    _, refs = O.ref_query([str(tmp_path / "db")], lines, str(tmp_path / "q"))
    for (op, ts, p), ref in zip(cases, refs):
        m = orc.match(O.Query(op=O.OP_AND if op == "AND" else O.OP_OR, terms=ts, maxitems=20, check_at_least=ndocs,
                              bm25=p))
        assert m.docids.tolist() == ref.docids, (op, ts, p)
        assert m.weights.tolist() == ref.weights, (op, ts, p)
        assert m.max_possible == ref.max_possible and m.max_attained == ref.max_attained, (op, ts, p)
