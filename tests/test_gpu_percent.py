"""percent_scale_factor and max_attained against the oracle, bit for bit, on every matching route, whatever the
approximation flags say (tests/percent_corpus.py; tests/test_percent_corpus.py pins the witnesses).

The scale needs the number of subqueries matching the FIRST document in docid order that attains the best weight.
In relevance order that is the first result; sorted by value the kernels' raise log has to supply it, and a
count-only query (nothing returned) keeps its one best-ranked document for it.  The corpus has bit-exact ties at the best weight between documents with
different numbers of matching leaves (W1), keeps them out of value-sorted MSets (W2), has a tie too large for the
raise log (W3, declined), large pruned queries whose best document matches few leaves (W4), and count-only queries
(W5) that run right after a batch which left sort keys in their result slots.

Routes (one searcher each; the environment picks the kernels):
  single        one leaf: xgm_and_kernel
  maybe_bm3     OP_AND_MAYBE over a two-list base with bitmaps: xgm_and_bm3_kernel
  maybe_and     the same with XGM_BITMAP_K=0: xgm_and_kernel
  or_tile       OR of <= 5 bitmap leaves: relevance order on the tile kernel + xgm_or3_kernel<1>, the value
                sorts on xgm_or3_kernel<0>
  or3           XGM_OR_TILE=0: xgm_or3_kernel<0>
  or_general    XGM_OR_KERNEL=1: xgm_or_kernel
  wide          6..13 leaves, two without a bitmap: xgm_or_kernel
  wide_nobm     the same with XGM_BITMAP_K=0
  or_filter     OR under OP_FILTER (a boolean term); or_not: under OP_AND_NOT; or_range: under a value range,
                which counts as one more matching subquery
  range_src     an AND with the weighted value-range source (one more weighted subquery)
"""
import os
import shutil
import tempfile
import time

import pytest

from oracle import oracle as O
from tests import percent_corpus as P
from tests.flatfile import write_flat
from tests.util import assert_matches_oracle, bits
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

MAX_TOPK = 128
ALL = P.NDOCS
# (maxitems, first, check_at_least): k in {1, 10, 100}, check_at_least in {0, k + 1, all}, first > 0 on some
ARGS = ((1, 0, 0), (10, 0, 11), (100, 0, ALL), (10, 7, 0), (1, 3, 5), (100, 0, 101))
SORTS = ((xgm.SORT_REL, False), (xgm.SORT_VAL, False), (xgm.SORT_VAL, True), (xgm.SORT_VAL_REL, False),
         (xgm.SORT_VAL_REL, True), (xgm.SORT_REL_VAL, False), (xgm.SORT_REL_VAL, True))
K1_0 = (0.0, 1.0, 0.5, 0.5)


@pytest.fixture(scope="module")
def pct():
    tmp = tempfile.mkdtemp(prefix="xgm_pct_")
    doclen, terms, nvals, vals, ties = P.build()
    path = os.path.join(tmp, "percent.flat")
    write_flat(path, doclen, terms)
    orc = O.Index.load_flat(path)
    orc.set_slot0(nvals, vals)
    slot = {0: P.device_slot(nvals, vals)}
    yield dict(ids={t[0]: i for i, t in enumerate(terms)}, orc=orc, ties=ties, doclen=doclen, terms=terms, slot=slot)
    shutil.rmtree(tmp, ignore_errors=True)


def device_index(pct):
    return xgm.Index.from_postings(pct["doclen"], pct["terms"], value_slots=pct["slot"])


def shape(names, op=xgm.OP_OR, factors=None, maybe=(), filter_terms=(), not_terms=(), value_range=None, bm25=None,
          tie=None):
    return dict(names=tuple(names), op=op, factors=factors, maybe=tuple(maybe), filter_terms=tuple(filter_terms),
                not_terms=tuple(not_terms), value_range=value_range, bm25=bm25, tie=tie)


def or_w1(**kw):
    out = []
    for key, names in P.W1_OR_SETS.items():
        out.append(shape(names, factors=list(P.W1_FACTORS), tie=key, **kw))
        out.append(shape(names[::-1], factors=list(P.W1_FACTORS)[::-1], tie=key, **kw))
    return out


def or_w4(**kw):
    return [shape(n, factors=list(P.W4_OR_FACTORS[len(n)]), **kw) for n in P.W4_OR_SETS]


def maybe_shapes():
    out = [shape(base, op=xgm.OP_AND, maybe=maybe, tie="maybe_" + key) for key, (base, maybe) in P.W1_MAYBE_SETS.items()]
    base, maybe = P.W4_MAYBE
    out.append(shape(base, op=xgm.OP_AND, maybe=maybe, factors=list(P.W4_MAYBE_FACTORS)))
    return out


W3 = shape(P.W1_OR_SETS["fewer"], factors=list(P.W1_FACTORS), bm25=K1_0)


def route_shapes(route):
    """(env, shapes, whether the route's queries vary their number of matching subqueries)."""
    wide = [shape(n, factors=P.wide_factors(n), tie="fewer" if n[0] == "fa" else "more") for n in P.WIDE_SETS]
    wide.append(shape(P.W4_OR_SETS[1] + P.G_NAMES[:2], factors=list(P.W4_OR_FACTORS[4]) + [P.FILLER_FACTOR] * 2))
    return {
        "single": ({}, [shape([n], op=xgm.OP_AND) for n in ("fa", "pa", "y25")], False),
        "maybe_bm3": ({}, maybe_shapes(), True),
        "maybe_and": ({"XGM_BITMAP_K": "0"}, maybe_shapes(), True),
        "or_tile": ({}, or_w1() + or_w4() + [W3], True),
        "or3": ({"XGM_OR_TILE": "0"}, or_w1() + or_w4() + [W3], True),
        "or_general": ({"XGM_OR_KERNEL": "1"}, or_w1() + or_w4() + [W3], True),
        "wide": ({}, wide, True),
        "wide_nobm": ({"XGM_BITMAP_K": "0"}, wide, True),
        "or_filter": ({}, or_w1(filter_terms=["z_bool"]) + or_w4(filter_terms=["z_bool"]), True),
        "or_not": ({}, or_w1(not_terms=["z_not"]) + or_w4(not_terms=["z_not"]), True),
        "or_range": ({}, or_w1(value_range="plain") + or_w4(value_range="plain"), True),
        "range_src": ({}, [shape(n, op=xgm.OP_AND, value_range="weighted")
                           for n in (("r_few", "r_wide"), ("pa", "w_all"), ("fa",))], False),
    }[route]


def pair(ids, s, sort, k, first, cal):
    """The same query for the CUDA path (term names, device keys = value + 1) and the oracle (term ids, values)."""
    sort_by, rev = sort
    kw = dict(first=first, maxitems=k, check_at_least=cal, factors=s["factors"], bm25=s["bm25"], sort_by=sort_by,
              sort_reverse=rev)
    xkw, okw = {}, {}
    if s["value_range"]:
        lo, hi = P.RANGE
        xkw = dict(filter=xgm.FILTER_MULTI_RANGE, filter_slot=0, range_lo=lo + 1, range_hi=hi + 1)
        okw = dict(filter=O.FILTER_MULTI_RANGE, range_lo=lo, range_hi=hi)
        if s["value_range"] == "weighted":
            xkw.update(filter_weighted=True, filter_factor=0.5)
            okw.update(filter_weighted=True, filter_factor=0.5)
    x = xgm.Query(s["op"], list(s["names"]), filter_terms=list(s["filter_terms"]), not_terms=list(s["not_terms"]),
                  maybe_terms=list(s["maybe"]), sort_slot=0, sort_missing_key=P.missing_key(rev), **xkw, **kw)
    o = O.Query(op=s["op"], terms=[ids[n] for n in s["names"]], filter_terms=[ids[n] for n in s["filter_terms"]],
                not_terms=[ids[n] for n in s["not_terms"]], maybe_terms=[ids[n] for n in s["maybe"]], sort_slot=0,
                sort_keymaker=True, sort_missing=P.missing_key(rev), **okw, **kw)
    return x, o


_refs = {}


def oracle(orc, o):
    """Oracle MSets are the same on every route: computed once per query."""
    key = repr(o)
    if key not in _refs:
        _refs[key] = orc.match(o)
    return _refs[key]


def tf_max(orc, o):
    return oracle(orc, O.Query(**dict(o.__dict__, first=0, maxitems=10, check_at_least=0, sort_by=O.SORT_REL))).ub


def check(m, ref, ctx):
    assert_matches_oracle(m, ref, ctx)
    assert [O.convert_to_percent(w, m.percent_scale_factor) for w in m.weights] == \
        [O.convert_to_percent(w, ref.percent_scale_factor) for w in ref.weights], ctx


def leaf_count(orc, ids, names, did):
    return sum(int(did in set(orc.postings(ids[n])[0].tolist())) for n in names)


def assert_w1_needs_the_lowest_docid(orc, ids, ties, s, o):
    """The tie at the best weight: the scale of its highest docid (what a wrong tie-break would return, and the last
    entry a docid-ordered log would hold) is not the reference's."""
    full = oracle(orc, O.Query(**dict(o.__dict__, first=0, maxitems=ALL, check_at_least=ALL, sort_by=O.SORT_REL)))
    top = full.docids[full.weights == full.max_attained].tolist()
    assert len(top) >= 3 and top[0] == int(ties[s["tie"]][0]), (s["names"], top)
    counted = list(s["names"]) + list(s["maybe"])
    cnt = [leaf_count(orc, ids, counted, d) for d in top]
    assert cnt[0] != cnt[-1] and cnt.count(cnt[0]) == 1, (s["names"], cnt)
    extra = 1 if s["value_range"] else 0
    nsub = len(counted) + (1 if s["value_range"] == "weighted" else 0)
    wrong = (cnt[-1] + extra) / nsub / full.max_attained * 100.0
    assert bits(wrong) != bits(full.percent_scale_factor)


def run(searcher, orc, pairs, ctx):
    res = searcher.search([x for x, _ in pairs])
    for i, (m, (x, o)) in enumerate(zip(res, pairs)):
        yield m, x, o, f"{ctx}[{i}] {list(x.terms)} F{list(x.filter_terms)} N{list(x.not_terms)} M{list(x.maybe_terms)} " \
                       f"fac={x.factors} bm25={x.bm25} sort={x.sort_by}/{int(x.sort_reverse)} k={x.maxitems} " \
                       f"first={x.first} cal={x.check_at_least} range={x.filter}/{x.filter_weighted}"


ROUTES = ["single", "maybe_bm3", "maybe_and", "or_tile", "or3", "or_general", "wide", "wide_nobm", "or_filter",
          "or_not", "or_range", "range_src"]


@pytest.mark.parametrize("route", ROUTES)
def test_percent_scale_matches_oracle(pct, route, monkeypatch):
    t0 = time.time()
    ids, orc = pct["ids"], pct["orc"]
    env, shapes, varies = route_shapes(route)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ix = device_index(pct)
    if env.get("XGM_BITMAP_K") == "0":
        assert ix.info().nbitmaps == 0
    for s in shapes:
        if s["tie"]:
            assert_w1_needs_the_lowest_docid(orc, ids, pct["ties"], s, pair(ids, s, SORTS[0], 10, 0, 0)[1])
    main = [(s, pair(ids, s, sort, k, first, cal)) for s in shapes for sort in SORTS for k, first, cal in ARGS]
    if route == "or_general":
        # MaxScore skips a leaf's items once the thresholds have risen: enough earlier work for that to happen
        w4 = [s for s in shapes if "pz" in s["names"]][0]
        main += [(w4, pair(ids, w4, SORTS[0], k, first, 0)) for k in range(1, 101) for first in (0, 2)]
    # count-only (first at the largest possible match count), and before them, at the same positions, a value
    # sort with results: a stale read of those slots' sort keys would show in the percentage scale
    count_only, dirty = [], []
    for s in shapes:
        for sort in SORTS:
            for cal in (1, ALL):
                o = pair(ids, s, sort, 10, 0, 0)[1]
                count_only.append((s, pair(ids, s, sort, 10, tf_max(orc, o), cal)))
                dirty.append((s, pair(ids, s, (xgm.SORT_VAL, False), 10, 0, 0)))
    searcher = xgm.Searcher(ix, max_batch=max(len(main), len(dirty)), max_topk=MAX_TOPK)
    # served, best document not among the results (raise log or count-only), pruned, skipped
    cells = {(sort, co): [0, 0, 0, 0] for sort in SORTS for co in (False, True)}
    declined = 0
    for batch, name in ((main, "main"), (dirty, "dirty"), (count_only, "count_only")):
        got = list(run(searcher, orc, [p for _, p in batch], f"{route}/{name}"))
        for (s, _), (m, x, o, ctx) in zip(batch, got):
            ref = oracle(orc, o)
            if s is W3 and x.sort_by != xgm.SORT_REL and name != "count_only":
                # more matches tie at the best weight than the raise log holds: declined, never guessed (a
                # count-only query ranks its matches by relevance and needs no raise log)
                assert m.status == xgm.E_UNIMPLEMENTED, ctx
                declined += 1
                continue
            check(m, ref, ctx)
            if name == "dirty":
                continue
            c = cells[((x.sort_by, x.sort_reverse), name == "count_only")]
            c[0] += 1
            c[1] += varies and (x.sort_by != xgm.SORT_REL or name == "count_only")
            c[2] += bool(m.flags & xgm.MSET_BOUNDS_APPROX)
            c[3] += bool(m.flags & xgm.MSET_COUNT_LOWER_BOUND)
    for (sort, co), (n, logged, pruned, skipped) in sorted(cells.items()):
        print(f"{route} sort={sort[0]}/{int(sort[1])} count_only={co}: {n} served, {logged} from outside the results, "
              f"{pruned} pruned, {skipped} with a skipped item")
    for sort in SORTS:
        logged = cells[(sort, False)][1] + cells[(sort, True)][1]
        # a single leaf and an AND with a range source match one fixed number of subqueries
        assert not varies or logged > 0, f"{route} sort={sort}: no query needed a document outside its results"
    rel = cells[(SORTS[0], False)]
    assert rel[2] > 0, f"{route}: no relevance-ordered query was pruned"
    if route == "or_general":
        assert rel[3] > 0, f"{route}: no query skipped a work item"
    assert declined > 0 or all(s is not W3 for s in shapes)
    print(f"{route}: {len(main) + len(dirty) + len(count_only)} queries, {declined} declined, {time.time() - t0:.1f} s")


def test_raise_log_overflow_declines_only_that_query(pct):
    """W3 (a value-sorted OR whose best weight more than 64 matches share) comes back XGM_E_UNIMPLEMENTED, and the
    W1 queries around it in the same batch are answered exactly."""
    ids, orc = pct["ids"], pct["orc"]
    ix = device_index(pct)
    w3 = [pair(ids, W3, sort, 10, 0, cal) for sort in SORTS[1:] for cal in (0, ALL)]
    others = [pair(ids, s, sort, 10, 0, 0) for s in or_w1() + maybe_shapes() for sort in SORTS]
    mixed = [p for i, p in enumerate(others) if i % 3] + w3 + [p for i, p in enumerate(others) if not i % 3]
    res = xgm.Searcher(ix, max_batch=len(mixed), max_topk=MAX_TOPK).search([x for x, _ in mixed])
    for i, (m, (x, o)) in enumerate(zip(res, mixed)):
        if any(x is y for y, _ in w3):
            assert m.status == xgm.E_UNIMPLEMENTED, f"w3[{i}]"
            full = oracle(orc, O.Query(**dict(o.__dict__, maxitems=ALL, check_at_least=ALL, sort_by=O.SORT_REL)))
            assert int((full.weights == full.max_attained).sum()) > 64
        else:
            check(m, oracle(orc, o), f"mixed[{i}] {list(x.terms)} sort={x.sort_by}/{int(x.sort_reverse)}")
