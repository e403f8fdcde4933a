"""Pins the corpus of tests/test_gpu_percent.py with the oracle and numpy alone (no GPU): an edit to
tests/percent_corpus.py that took a witness away would leave the GPU tests passing without testing the percentage
scale they are for."""
import shutil
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import percent_corpus as P

ALL = P.NDOCS


@pytest.fixture(scope="module")
def pct():
    tmp = tempfile.mkdtemp(prefix="xgm_pct_")
    path, names, nvals, vals, ties = P.write_percent_corpus(tmp)
    orc = O.Index.load_flat(path)
    orc.set_slot0(nvals, vals)
    yield {n: i for i, n in enumerate(names)}, orc, ties
    shutil.rmtree(tmp, ignore_errors=True)


def leaves_of(orc, ids, names, did):
    return sum(int(did in set(orc.postings(ids[n])[0].tolist())) for n in names)


def scale(subqs, nsub, max_w):
    return subqs / nsub / max_w * 100.0


def test_corpus_shape(pct):
    ids, orc, ties = pct
    assert orc.doccount == P.NDOCS and orc.lastdocid == P.LASTDOCID
    assert P.LASTDOCID % 32 and P.LASTDOCID % 256
    bm = {n: orc.termfreq(ids[n]) >= P.BITMAP_MIN for n in ids}
    assert not bm["g0"] and not bm["g1"] and all(bm[n] for n in ids if n not in ("g0", "g1"))
    for names in P.W1_OR_SETS.values():
        assert {orc.termfreq(ids[n]) for n in names} == {P.OR_TF}
    assert [orc.termfreq(ids[n]) for n in ("y25", "y5a", "y5b")] == [P.Y25_TF, P.Y5_TF, P.Y5_TF]
    # the idfs of the optional leaves: log(25) and log(5), and the first is exactly twice the second
    x25 = (P.NDOCS - P.Y25_TF + 0.5) / (P.Y25_TF + 0.5)
    x5 = (P.NDOCS - P.Y5_TF + 0.5) / (P.Y5_TF + 0.5)
    assert (x25, x5) == (25.0, 5.0) and np.log(x25) == 2 * np.log(x5)
    dl = orc.doclen()
    d, w = orc.postings(ids["z_bool"])
    assert (w == 0).all() and set(np.concatenate(list(ties.values())).tolist()) <= set(d.tolist())
    assert not set(orc.postings(ids["z_not"])[0].tolist()) & set(np.concatenate(list(ties.values())).tolist())
    total = np.zeros(orc.lastdocid + 1, np.int64)
    for t in range(orc.nterms):
        d, w = orc.postings(t)
        total[d] += w
    assert (total <= dl).all()


def w1_queries(ids, ties):
    """(tie key, leaf names, oracle query kwargs) of every W1 shape: the OR sets alone, in a reversed leaf order,
    among fillers, under FILTER / AND_NOT, under a value range (which counts as one more matching subquery); the
    AND_MAYBE sets."""
    out = []
    for key, names in P.W1_OR_SETS.items():
        fac = list(P.W1_FACTORS)
        out.append((key, names, dict(op=O.OP_OR, terms=[ids[n] for n in names], factors=fac)))
        out.append((key, names, dict(op=O.OP_OR, terms=[ids[n] for n in names[::-1]], factors=fac[::-1])))
        out.append((key, names, dict(op=O.OP_OR, terms=[ids[n] for n in names], factors=fac,
                                     filter_terms=[ids["z_bool"]])))
        out.append((key, names, dict(op=O.OP_OR, terms=[ids[n] for n in names], factors=fac,
                                     not_terms=[ids["z_not"]])))
        out.append((key, names, dict(op=O.OP_OR, terms=[ids[n] for n in names], factors=fac,
                                     filter=O.FILTER_MULTI_RANGE, range_lo=P.RANGE[0], range_hi=P.RANGE[1])))
    for wide in P.WIDE_SETS:
        key = "fewer" if wide[0] == "fa" else "more"
        out.append((key, wide, dict(op=O.OP_OR, terms=[ids[n] for n in wide], factors=P.wide_factors(wide))))
    for key, (base, maybe) in P.W1_MAYBE_SETS.items():
        kw = dict(op=O.OP_AND, terms=[ids[n] for n in base], maybe_terms=[ids[n] for n in maybe])
        out.append(("maybe_" + key, base + maybe, kw))
    return out


def test_w1_ties_at_the_best_weight_have_different_leaf_counts(pct):
    """The best weight is shared bit for bit by the tie documents (those a filter lets through) and no other; the
    lowest of them matches a number of leaves that no other tie document matches, so a percentage scale taken from
    any other tie document (the highest docid, the last one logged) is not the reference's."""
    ids, orc, ties = pct
    seen = set()
    for key, names, kw in w1_queries(ids, ties):
        r = orc.match(O.Query(maxitems=ALL, check_at_least=ALL, **kw))
        top = r.docids[r.weights == r.max_attained].tolist()
        tie = ties[key].tolist()
        assert top == sorted(top) and set(top) <= set(tie) and len(top) >= 3, (key, kw)
        assert top[0] == tie[0], (key, kw)
        counted = [n for n in names if n not in ("r_few", "r_more", "r_wide")]
        base = len(names) - len(counted)
        extra = 1 if kw.get("filter") else 0
        counts = [base + leaves_of(orc, ids, counted, d) + extra for d in top]
        assert all(c != counts[0] for c in counts[1:]), (key, counts)
        nsub = len(names) + (1 if kw.get("filter_weighted") else 0)
        assert r.percent_scale_factor == scale(counts[0], nsub, r.max_attained), (key, kw)
        assert r.percent_scale_factor != scale(counts[-1], nsub, r.max_attained)
        seen.add((key, counts[0] < counts[-1]))
    # both orders: the lowest tie docid has fewer leaves than the others, and more
    assert {s[1] for s in seen} == {True, False}


SORTS = [(O.SORT_VAL, False), (O.SORT_VAL, True), (O.SORT_VAL_REL, False), (O.SORT_VAL_REL, True),
         (O.SORT_REL_VAL, False), (O.SORT_REL_VAL, True)]


def test_w2_best_document_is_outside_value_sorted_msets(pct):
    """Sorted by value (missing values last), the tie documents are past k = 100 in either direction: two have no
    value, the others a value in the middle of hundreds.  Relevance then value puts them first, so there they are
    skipped by `first`.  The percentage scale is still that of the lowest tie docid."""
    ids, orc, ties = pct
    for key, names, kw in w1_queries(ids, ties):
        full = orc.match(O.Query(maxitems=ALL, check_at_least=ALL, **kw))
        for sort_by, rev in SORTS:
            sk = dict(sort_by=sort_by, sort_slot=0, sort_reverse=rev, sort_keymaker=True,
                      sort_missing=P.missing_key(rev))
            for k, first in ((1, 0), (10, 0), (100, 0), (10, 7)):
                if sort_by == O.SORT_REL_VAL:
                    first = max(first, P.NTIE)
                r = orc.match(O.Query(maxitems=k, first=first, **sk, **kw))
                assert not set(r.docids.tolist()) & set(ties[key].tolist()), (key, sort_by, rev, k, first)
                assert r.percent_scale_factor == full.percent_scale_factor
                assert r.max_attained == full.max_attained


def test_w3_value_sorted_tie_overflows_the_raise_log(pct):
    """Under k1 = 0 the f set's best weight is shared by every fa document and the fb + fc ties: far more than the
    64 entries the raise log holds."""
    ids, orc, _ = pct
    names = P.W1_OR_SETS["fewer"]
    r = orc.match(O.Query(op=O.OP_OR, terms=[ids[n] for n in names], factors=list(P.W1_FACTORS),
                          bm25=(0.0, 1.0, 0.5, 0.5), maxitems=ALL, check_at_least=ALL))
    assert int((r.weights == r.max_attained).sum()) > 8 * 64


def test_w4_pruned_queries_have_a_best_document_with_few_leaves(pct):
    """The large relevance-ordered W4 queries are topped by pa's heavy documents, which match one leaf of the OR and
    no optional leaf of the AND_MAYBE: a scale taken from nweighted would be wrong.  Few documents share a weight."""
    ids, orc, _ = pct
    heavy = None
    for names in P.W4_OR_SETS:
        r = orc.match(O.Query(op=O.OP_OR, terms=[ids[n] for n in names], factors=P.W4_OR_FACTORS[len(names)],
                              maxitems=10, check_at_least=0))
        assert r.ub > 20000
        assert leaves_of(orc, ids, names, int(r.docids[0])) == 1
        assert r.percent_scale_factor == scale(1, len(names), r.max_attained)
        heavy = set(r.docids[:P.HEAVY].tolist())
        # few documents share a weight, so that value-sorted runs over these lists keep a short raise log
        full = orc.match(O.Query(op=O.OP_OR, terms=[ids[n] for n in names], factors=P.W4_OR_FACTORS[len(names)],
                                 maxitems=ALL, check_at_least=ALL))
        assert int(np.unique(full.weights, return_counts=True)[1].max()) <= 8
    base, maybe = P.W4_MAYBE
    r = orc.match(O.Query(op=O.OP_AND, terms=[ids[n] for n in base], maybe_terms=[ids[n] for n in maybe],
                          factors=P.W4_MAYBE_FACTORS, maxitems=10, check_at_least=ALL))
    assert r.exact > 5000 and set(r.docids[:P.HEAVY].tolist()) == heavy
    assert r.percent_scale_factor == scale(2, 4, r.max_attained)


def test_w5_count_only_queries_keep_a_percentage_scale(pct):
    """With `first` at the largest possible match count the MSet is empty, yet the reference computes the scale of
    its best document (every match went through ProtoMSet)."""
    ids, orc, ties = pct
    for key, names, kw in w1_queries(ids, ties):
        ub = orc.match(O.Query(maxitems=10, **kw)).ub
        full = orc.match(O.Query(maxitems=ALL, check_at_least=ALL, **kw))
        for cal in (1, ALL):
            r = orc.match(O.Query(first=ub, maxitems=10, check_at_least=cal, **kw))
            assert len(r.docids) == 0 and r.exact == full.exact
            assert r.percent_scale_factor == full.percent_scale_factor > 0
