"""Value-range filters on OR bases and sparse slots against the compiled reference's fixtures.

OP_FILTER(base, range) runs in the reference as a MultiAndPostList of [base, range], so the match bounds fold in
the range's termfreqs: (0, value_freq, value_freq) for Xapiand's MultipleValueRange source (range.cc:457-464), and
for a stock OP_VALUE_RANGE max value_freq and min value_freq when the range covers the slot's values, 0 otherwise
(valuerangepostlist.cc:40-54,145-148).  On an OR base the upper bound is then at most value_freq, and the lower
bound is usually 0, however many documents the OR tree alone must match.

  orvalues_5k, orvalues_sparse_5k  MultipleValueRange on Xapiand slots (value_freq 4279, and about half the
                                   documents), on OR bases of 2..5 and 6..16 leaves, single terms and ANDs
  vrbounds_5k                      stock OP_VALUE_RANGE on AND and OR bases

Every query is checked against the fixture bit for bit: docids, weights, percentages, max_possible and
max_attained, the order of the sort keys, and lb / est / ub exactly unless MSET_BOUNDS_APPROX licenses less; the
upper bound always.  Each OR route runs six copies of the fixture as one batch: the or3 kernel (default), the
general kernel (XGM_OR_KERNEL=1) and an index without membership bitmaps (XGM_BITMAP_K=0)."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.golden_util import load, sortable_key_to_int
from tests.percent_corpus import device_slot
from tests.util import assert_matches_oracle, bits
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

MAX_TOPK = 128
MV_TAGS = ("orvalues_5k", "orvalues_sparse_5k")


def device_index(fx):
    """The fixture's corpus with its slots as numeric keys, each value plus one (tests.percent_corpus.device_slot):
    the same order as the serialised bytes Xapiand stores, whose parsing multivalue_5k's device test covers.  Slot 0
    holds each document's 1..3 values, slot 1 one value, both thinned by the fixture's sparse rule."""
    orc = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    orc.make_sparse(*fx["sparse"])
    nvals, vals, val1 = orc.values()
    voff0 = np.zeros(len(nvals) + 1, np.uint64)
    voff0[1:] = np.cumsum(nvals.astype(np.uint64))
    keys0 = np.concatenate([vals[d, :nvals[d]] for d in range(len(nvals))]).astype(np.uint64) + 1
    has1 = (val1 % fx["sparse"][1] != 0) & (np.arange(len(val1)) > 0)
    voff1, keys1 = device_slot(has1.astype(np.uint8), val1[:, None])
    terms = [(orc.name(t),) + tuple(orc.postings(t)) for t in range(orc.nterms)]
    return xgm.Index.from_postings(orc.doclen(), terms, value_slots={0: (voff0, keys0), 1: (voff1, keys1)})


def mv_query(q):
    kw = dict(first=q["first"], maxitems=q["maxitems"], check_at_least=q["check_at_least"],
              filter=xgm.FILTER_MULTI_RANGE, filter_slot=q["mvr"][0], range_lo=q["mvr"][1] + 1,
              range_hi=q["mvr"][2] + 1)
    if "keysort" in q:
        slot, rev = q["keysort"]
        kw.update(sort_by=xgm.SORT_VAL_REL, sort_slot=slot, sort_reverse=bool(rev), sort_use_max=bool(rev),
                  sort_missing_key=0 if rev else 2 ** 64 - 1)
    return xgm.Query(xgm.OP_OR if q["op"] == "OR" else xgm.OP_AND, [f"T{t:06d}" for t in q["terms"]], **kw)


def check_bounds(m, q, ctx):
    assert m.matches_upper_bound == q["ub"], f"{ctx}: ub {m.matches_upper_bound} vs {q['ub']}"
    if m.flags & xgm.MSET_BOUNDS_APPROX:
        assert m.matches_lower_bound <= q["lb"], f"{ctx}: lb {m.matches_lower_bound} > {q['lb']}"
        assert m.matches_lower_bound <= m.matches_estimated_raw <= m.matches_upper_bound, f"{ctx}: lb/est/ub"
        return False
    assert (m.matches_lower_bound, m.get_matches_estimated()) == (q["lb"], q["est"]), \
        f"{ctx}: lb/est {(m.matches_lower_bound, m.get_matches_estimated())} vs {(q['lb'], q['est'])}"
    return True


def check_result(m, q, ctx):
    """Everything but the bounds, bit for bit against the fixture."""
    assert m.status == 0, f"{ctx}: status {m.status}"
    assert list(m.docids) == q["docids"], f"{ctx}: docids"
    assert [bits(w) for w in m.weights] == [bits(w) for w in q["weights"]], f"{ctx}: weights"
    assert bits(m.max_possible) == bits(q["max_possible"]), f"{ctx}: max_possible"
    assert bits(m.max_attained) == bits(q["max_attained"]), f"{ctx}: max_attained"
    assert [O.convert_to_percent(w, m.percent_scale_factor) for w in m.weights] == q["percents"], f"{ctx}: percentages"


def run_mv(ix, fx, route):
    """The fixture's queries six times over in one batch (at least 256 queries): every copy must give the
    reference's MSet."""
    qs = fx["queries"] * 6
    assert len(qs) >= 256
    res = xgm.Searcher(ix, max_batch=len(qs), max_topk=MAX_TOPK).search([mv_query(q) for q in qs])
    exact = {"OR": 0, "AND": 0}
    for i, (q, m) in enumerate(zip(qs, res)):
        ctx = f"{fx['tag']}/{route}[{i}] {q['op']} {q['terms']} mvr={q['mvr']} keysort={q.get('keysort')} " \
              f"first={q['first']} k={q['maxitems']} cal={q['check_at_least']}"
        check_result(m, q, ctx)
        if "keysort" in q:  # the device keys in the order of the reference's key bytes
            keys = [bytes.fromhex(k) for k in q.get("sort_keys", [])]
            mine = [int(k) for k in m.sort_keys]
            rev = bool(q["keysort"][1])
            for a in range(len(keys) - 1):
                # reverse key bytes are complemented: ascending bytes = descending values
                assert (keys[a] < keys[a + 1]) == ((mine[a] > mine[a + 1]) if rev else (mine[a] < mine[a + 1])), ctx
                assert (keys[a] == keys[a + 1]) == (mine[a] == mine[a + 1]), ctx
        exact[q["op"]] += check_bounds(m, q, ctx)
    n_or = sum(q["op"] == "OR" for q in qs)
    print(f"{fx['tag']}/{route}: exact bounds on {exact['OR']} of {n_or} OR and {exact['AND']} of {len(qs) - n_or} AND")
    # a Xapiand range's source is restated exactly: only pruning on the device may loosen the bounds
    assert 4 * exact["AND"] >= 3 * (len(qs) - n_or), f"{fx['tag']}/{route}: AND bounds flagged"
    assert 4 * exact["OR"] >= n_or, f"{fx['tag']}/{route}: only {exact['OR']} of {n_or} OR queries with exact bounds"


@pytest.fixture(scope="module", params=MV_TAGS)
def mv(request):
    fx = load(request.param)
    return fx, device_index(fx)


@pytest.mark.parametrize("route", ["or3", "general"])
def test_range_source_on_or_bases_matches_reference(mv, route, monkeypatch):
    fx, ix = mv
    if route == "general":
        monkeypatch.setenv("XGM_OR_KERNEL", "1")
    run_mv(ix, fx, route)


def test_range_source_on_or_bases_without_bitmaps(mv, monkeypatch):
    fx, _ = mv
    monkeypatch.setenv("XGM_BITMAP_K", "0")
    ix = device_index(fx)
    assert ix.info().nbitmaps == 0
    run_mv(ix, fx, "no-bitmap")


def test_pruned_filtered_or_keeps_its_upper_bound(monkeypatch):
    """Relevance-ordered ORs of the most frequent term and a rarer one under a MultipleValueRange on a slot half the
    documents have, 400 to a batch on a 200k-document corpus, so that MaxScore skips work items of the frequent leaf
    once the thresholds have risen (MSET_COUNT_LOWER_BOUND): the upper bound stays the reference's
    min(OR max, value_freq), the lower bound and the exact count stay below the oracle's (which the orvalues fixtures
    pin to the reference), docids and weights stay exact."""
    ndocs = 200000
    orc = O.Index.synthetic(ndocs, 3000)
    nvals = np.zeros(orc.lastdocid + 1, np.uint8)
    nvals[2::2] = 1
    vals = np.zeros((orc.lastdocid + 1, 3), np.uint64)
    vals[:, 0] = (np.arange(orc.lastdocid + 1, dtype=np.uint64) * 7919) % 1000000
    orc.set_slot0(nvals, vals)
    terms = [(orc.name(t),) + tuple(orc.postings(t)) for t in range(orc.nterms)]
    ix = xgm.Index.from_postings(orc.doclen(), terms, value_slots={0: device_slot(nvals, vals)})
    pairs = []
    for t in range(20, 120):
        for k in (1, 10):
            for first in (0, 2):
                # device keys are the values plus one (device_slot)
                pairs.append((xgm.Query(xgm.OP_OR, [0, t], first=first, maxitems=k, filter=xgm.FILTER_MULTI_RANGE,
                                        filter_slot=0, range_lo=1, range_hi=1000001),
                               O.Query(op=O.OP_OR, terms=[0, t], first=first, maxitems=k, filter=O.FILTER_MULTI_RANGE,
                                       range_lo=0, range_hi=1000000)))
    refs = [orc.match(o) for _, o in pairs]
    vf = int(nvals.sum())
    assert sum(r.ub == vf for r in refs) > 0  # the range's value_freq is below some ORs' own maximum
    skipped = 0
    for route in ("or3", "general"):
        if route == "general":
            monkeypatch.setenv("XGM_OR_KERNEL", "1")
        res = xgm.Searcher(ix, max_batch=len(pairs), max_topk=MAX_TOPK).search([x for x, _ in pairs])
        for i, (m, (x, _), ref) in enumerate(zip(res, pairs, refs)):
            assert_matches_oracle(m, ref, f"pruned/{route}[{i}] {list(x.terms)} first={x.first} k={x.maxitems}")
            skipped += bool(m.flags & xgm.MSET_COUNT_LOWER_BOUND)
    print(f"pruned: {skipped} of {2 * len(pairs)} skipped a work item")
    assert skipped > 0, "no filtered OR skipped a work item"


def test_stock_value_range_bounds_match_reference():
    """Stock OP_VALUE_RANGE on AND and OR bases: lower and upper bounds exact (the estimate, which folds in the
    range's string-fraction estimate, is licensed by MSET_BOUNDS_APPROX); a range covering every value of a slot
    all documents have is the all-documents list, which is no matching subquery for the percentages."""
    fx = load("vrbounds_5k")
    ix = xgm.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    qs = fx["queries"]
    xs = []
    for q in qs:
        kw = dict(first=q["first"], maxitems=q["maxitems"], check_at_least=q["check_at_least"],
                  filter=xgm.FILTER_VALUE_RANGE, filter_slot=0, range_lo=q["vr"][1], range_hi=q["vr"][2])
        if "sort" in q:
            kw.update(sort_by=xgm.SORT_VAL_REL, sort_slot=q["sort"][0], sort_reverse=bool(q["sort"][1]))
        xs.append(xgm.Query(xgm.OP_AND if q["op"] == "AND" else xgm.OP_OR, q["terms"], **kw))
    res = xgm.Searcher(ix, max_batch=len(xs), max_topk=MAX_TOPK).search(xs)
    exact_lb = 0
    for i, (q, m) in enumerate(zip(qs, res)):
        ctx = f"vrbounds[{i}] {q['op']} {q['terms']} vr={q['vr']} sort={q.get('sort')} first={q['first']} " \
              f"k={q['maxitems']} cal={q['check_at_least']}"
        check_result(m, q, ctx)
        check_bounds(m, q, ctx)
        exact_lb += m.matches_lower_bound == q["lb"]
        if "sort" in q:
            keys = [sortable_key_to_int(k) for k in q.get("sort_keys", [])]
            mine = list(m.sort_keys)
            for a in range(len(keys) - 1):
                assert (keys[a] < keys[a + 1]) == (mine[a] < mine[a + 1]), ctx
                assert (keys[a] == keys[a + 1]) == (mine[a] == mine[a + 1]), ctx
    assert 4 * exact_lb >= 3 * len(qs), f"only {exact_lb} of {len(qs)} exact lower bounds"
