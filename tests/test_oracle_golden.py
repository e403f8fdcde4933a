"""CPU tests: the C restatement (oracle/xgm_oracle.c) against golden vectors produced by the
compiled reference itself (tests/golden/*.json).  This is what pins the oracle."""
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests.golden_util import load, sortable_key_to_int


def bits(x):
    return struct.pack("<d", float(x))


def o_query(q, stats=None, first=None, maxitems=None):
    kw = dict(op=O.OP_AND if q["op"] == "AND" else O.OP_OR, terms=q["terms"],
              first=q["first"] if first is None else first,
              maxitems=q["maxitems"] if maxitems is None else maxitems, check_at_least=q["check_at_least"], stats=stats)
    if "vr" in q:
        kw.update(filter=O.FILTER_VALUE_RANGE_MIN, range_lo=q["vr"][1], range_hi=q["vr"][2])
    if "sort" in q:
        mode = {0: O.SORT_VAL_REL, 1: O.SORT_VAL, 2: O.SORT_REL_VAL}[q.get("sort_mode", 0)]
        kw.update(sort_by=mode, sort_slot=q["sort"][0], sort_reverse=bool(q["sort"][1]))
    for g in ("filter_terms", "not_terms", "maybe_terms", "factors", "wqf", "bm25"):
        if q.get(g):
            kw[g] = q[g]
    return O.Query(**kw)


def check(m, q, ctx, counts=True):
    assert list(m.docids) == q["docids"], f"{ctx}: docids"
    assert all(bits(a) == bits(b) for a, b in zip(m.weights, q["weights"])), f"{ctx}: weights not bit-equal"
    assert bits(m.max_attained) == bits(q["max_attained"]), f"{ctx}: max_attained"
    if counts:
        assert bits(m.max_possible) == bits(q["max_possible"]), f"{ctx}: max_possible"
        assert (m.lb, O.round_estimate(m.lb, m.ub, m.est), m.ub) == (q["lb"], q["est"], q["ub"]), f"{ctx}: bounds"
    if "percents" in q:  # MSetIterator::get_percent of the reference ← percent_scale_factor (protomset.h:466-471)
        mine = [O.convert_to_percent(w, m.percent_scale_factor) for w in m.weights]
        assert mine == q["percents"], f"{ctx}: percentages"


@pytest.mark.parametrize("tag", ["c1_1k_100", "mid_20k"])
def test_oracle_matches_reference_single_db(tag):
    fx = load(tag)
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"{tag}[{i}] {q['op']} {q['terms']}")


def test_oracle_matches_reference_filter_andnot_andmaybe():
    """SURVEY.md §8(f)-1: OP_FILTER with boolean terms, OP_AND_NOT, OP_AND_MAYBE around an AND base
    (api/queryinternal.cc:2208-2283, matcher/andnotpostlist.cc, andmaybepostlist.cc) — docids, weights,
    bounds, max_possible and max_attained bit-equal with the compiled reference."""
    fx = load("ops_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    shapes = set()
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"ops[{i}] {q}")
        shapes.add((bool(q["filter_terms"]), bool(q["not_terms"]), bool(q["maybe_terms"])))
    assert len(shapes) >= 7  # every combination of the three groups is present


def test_oracle_matches_reference_groups_around_or_base():
    """The same three groups around an OR base (a free-text OR restricted by boolean terms): the MultiAndPostList
    of [OrPostList tree, filter], AndNotPostList and AndMaybePostList above it — orops_6k fixture."""
    fx = load("orops_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    shapes = set()
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"orops[{i}] {q}")
        shapes.add((bool(q["filter_terms"]), bool(q["not_terms"]), bool(q["maybe_terms"])))
    assert len(shapes) >= 7


def test_oracle_matches_reference_scale_weight():
    """OP_SCALE_WEIGHT factors on the leaves (QueryScaleWeight::postlist api/queryinternal.cc:1075-1080 →
    Weight::init_ factor), incl. factor 0 = unweighted leaf that is not a counted subquery."""
    fx = load("scale_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"scale[{i}] {q['op']} {q['terms']} x {q['factors']}")


def test_oracle_matches_reference_wqf():
    """Within-query frequency > 1: Weight::init_'s wqf and BM25Weight::init's (k3+1)*wqf/(k3+wqf) factor."""
    fx = load("wqf_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"wqf[{i}] {q['op']} {q['terms']} wqf {q['wqf']}")


def test_oracle_matches_reference_sort_modes():
    """Enquire::set_sort_by_value / set_sort_by_relevance_then_value / set_sort_by_value_then_relevance:
    comparators of msetcmp.cc:54-98 and the ProtoMSet paths they select (early_reject, min_weight)."""
    fx = load("sortmodes_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    seen = set()
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"sortmodes[{i}] {q}")
        seen.add(q["sort_mode"])
    assert seen == {0, 1, 2}


def test_oracle_matches_reference_bm25_parameters():
    """BM25Weight with non-default k1 / k3 / b / min_normlen (k2 = 0), incl. the k1 = 0 and b = 0 branches of
    BM25Weight::init (bm25weight.cc:46-130) and get_maxpart."""
    fx = load("bm25_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"])
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"bm25[{i}] {q['op']} {q['terms']} {q['bm25']}")


def test_oracle_matches_reference_count_regimes():
    """check_at_least between k+1 and the match count, k = 1, first > 0, value sorts: where ProtoMSet's
    min_weight lags behind the k-th best weight (protomset.h:377-398) and the count rule has its third term
    (tests/test_protomset_count_model.py)."""
    fx = load("regimes_6k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    for i, q in enumerate(fx["queries"]):
        check(ix.match(o_query(q)), q, f"regimes[{i}] {q}")


def test_oracle_matches_reference_twophase_shards():
    fx = load("shard4_20k")
    n = fx["nshards"]
    shards = [O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], nshards=n, shard=s) for s in range(n)]
    coll = sum(s.doccount for s in shards)
    tlen = sum(s.total_length for s in shards)
    for i, q in enumerate(fx["queries"]):
        gtf = [sum(s.termfreq(t) for s in shards) for t in q["terms"]]
        parts = []
        for si, s in enumerate(shards):
            # DocMatcher asks every shard for first=0, maxitems=first+maxitems (handler.cc:1511-1512)
            m = s.match(o_query(q, stats=(coll, tlen, gtf), first=0, maxitems=q["first"] + q["maxitems"]))
            m.docids = ((m.docids.astype(np.uint64) - 1) * n + si + 1).astype(np.uint32)  # unshard_docids
            parts.append(m)
        merged = O.merge(parts, q["first"], q["maxitems"])
        ctx = f"shard4[{i}] {q}"
        assert list(merged.docids) == q["docids"], ctx
        assert all(bits(a) == bits(b) for a, b in zip(merged.weights, q["weights"])), ctx
        assert bits(merged.max_attained) == bits(q["max_attained"]), ctx
        assert bits(merged.max_possible) == bits(q["max_possible"]), ctx
        assert (merged.lb, O.round_estimate(merged.lb, merged.ub, merged.est), merged.ub) == (q["lb"], q["est"], q["ub"]), ctx


def test_oracle_matches_reference_value_filter_and_sort():
    fx = load("values_5k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    for i, q in enumerate(fx["queries"]):
        m = ix.match(o_query(q))
        ctx = f"values[{i}] {q}"
        # bounds of a value-range AND depend on ValueRangePostList's string-fraction estimate
        # (valuerangepostlist.cc:70-130), not restated: exact only when check_at_least covers the db
        check(m, q, ctx, counts=False)
        if q["check_at_least"] >= fx["ndocs"] and len(q["docids"]) < q["maxitems"]:
            assert m.lb == q["lb"] and m.ub == q["ub"], ctx
        if "sort" in q:
            keys = [sortable_key_to_int(k) for k in q.get("sort_keys", [])]
            mine = list(m.sortvals)
            # same order relation between consecutive items
            for a in range(len(keys) - 1):
                assert (keys[a] < keys[a + 1]) == (mine[a] < mine[a + 1]) and (keys[a] == keys[a + 1]) == (mine[a] == mine[a + 1]), ctx


def test_and_order_and_or_program_shapes():
    assert O.and_order([5, 3, 9]) == [1, 0, 2]
    # OR tree of OrContext::postlist: leaves with the smallest termfreq are merged first
    prog = O.or_program([100, 10, 1])
    assert prog.count(-1) == 2 and sorted(x for x in prog if x >= 0) == [0, 1, 2]
    assert O.or_program([7]) == [0]


def test_round_estimate_examples():
    # values observed from the reference (tests/golden): est 925 within [676,1000] → 900
    assert O.round_estimate(676, 1000, 925) == 900
    assert O.round_estimate(9998, 19159, 18081) == 18000
    assert O.round_estimate(5, 5, 5) == 5


def mv_o_query(q):
    """multivalue_5k fixture → oracle query: Xapiand's MultipleValueRange / Multi_MultiValueKeyMaker shapes."""
    kw = dict(op=O.OP_OR if q.get("op") == "OR" else O.OP_AND, terms=q["terms"], first=q["first"],
              maxitems=q["maxitems"], check_at_least=q["check_at_least"])
    if "mvr" in q:
        kw.update(filter=O.FILTER_MULTI_RANGE, range_lo=q["mvr"][1], range_hi=q["mvr"][2], filter_weighted=bool(q["mvr"][3]))
    if "keysort" in q:
        slot, rev = q["keysort"]
        kw.update(sort_by=O.SORT_VAL_REL, sort_slot=1 if slot == 1 else (2 if rev else 0), sort_reverse=bool(rev),
                  sort_keymaker=True, sort_missing=0 if rev else 2 ** 64 - 1)
    return O.Query(**kw)


def test_oracle_matches_xapiand_multivalue_classes():
    """SURVEY.md §8 rows a15 / a16 pinned against Xapiand's REAL code: the fixture comes from
    src/multivalue/range.cc (MultipleValueRange as OP_FILTER right side and as weighted OP_AND child),
    src/multivalue/keymaker.cc (Multi_MultiValueKeyMaker with a SerialiseKey, forward and reverse, documents
    without a value) and src/serialise_list.h / src/sortable_serialise.cc slot encodings, compiled from the
    reference by oracle/build_ref.sh.  Docids, weights, bounds, max_possible / max_attained, percentages."""
    fx = load("multivalue_5k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    ix.make_sparse(*fx["sparse"])
    kinds = set()
    for i, q in enumerate(fx["queries"]):
        m = ix.match(mv_o_query(q))
        check(m, q, f"mv[{i}] {q['terms']} mvr={q.get('mvr')} keysort={q.get('keysort')}")
        kinds.add((q.get("mvr", [0, 0, 0, -1])[3], tuple(q.get("keysort", ()))))
        check_keysort_order(m, q, i)
    assert len(kinds) >= 10


def check_keysort_order(m, q, ctx):
    """Same order relation between consecutive sort keys (byte strings vs the oracle's scale)."""
    if "keysort" not in q:
        return
    keys = [bytes.fromhex(k) for k in q.get("sort_keys", [])]
    mine = list(m.sortvals)
    rev = bool(q["keysort"][1])
    for a in range(len(keys) - 1):
        # reverse keys are complemented: ascending bytes = descending values
        assert (keys[a] < keys[a + 1]) == ((mine[a] > mine[a + 1]) if rev else (mine[a] < mine[a + 1])), ctx
        assert (keys[a] == keys[a + 1]) == (mine[a] == mine[a + 1]), ctx


def range_kind(lo, hi):
    return "nothing" if lo >= 2000000 else "all" if (lo, hi) == (0, 1000000) else "narrow" if hi - lo <= 10000 else "wide"


@pytest.mark.parametrize("tag", ["orvalues_5k", "orvalues_sparse_5k"])
def test_oracle_matches_reference_range_source_on_or_bases(tag):
    """OP_FILTER(base, MultipleValueRange) on OR bases of 2..5 and 6..16 leaves, single terms and ANDs: the reference
    runs it as a MultiAndPostList of [base, source] whose termfreqs fold in the source's (0, value_freq, value_freq)
    (range.cc:457-464), so the upper bound is at most value_freq and the lower bound is usually 0.  Docids, weights,
    sort keys, percentages and all three bounds bit-equal with the compiled reference."""
    fx = load(tag)
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    ix.make_sparse(*fx["sparse"])
    vf = int((ix.values()[0] != 0).sum())
    shapes, clipped = set(), 0
    for i, q in enumerate(fx["queries"]):
        m = ix.match(mv_o_query(q))
        ctx = f"{tag}[{i}] {q['op']} {q['terms']} mvr={q['mvr']} keysort={q.get('keysort')}"
        check(m, q, ctx)
        check_keysort_order(m, q, ctx)
        base = "single" if len(q["terms"]) == 1 else q["op"] + ("-wide" if len(q["terms"]) > 5 else "")
        shapes.add((base, range_kind(*q["mvr"][1:3])))
        if q["op"] == "OR":  # the reference's bound lies below the OR tree's own
            whole = ix.match(O.Query(op=O.OP_OR, terms=q["terms"], maxitems=0))
            clipped += q["ub"] == vf < whole.ub
    assert len(shapes) == 16, sorted(shapes)
    assert clipped >= 3, clipped


def test_oracle_matches_reference_value_range_bounds():
    """Stock OP_VALUE_RANGE on AND and OR bases: the range's termfreq max is value_freq and its min value_freq when it
    covers the slot's value bounds, 0 otherwise (valuerangepostlist.cc:40-54,145-148), so the lower and upper
    bounds are exact; the estimate folds in the range's string-fraction estimate, which is not restated.  A range
    covering every value of a slot all documents have is the all-documents list: no matching subquery for the
    percentages."""
    fx = load("vrbounds_5k")
    ix = O.Index.synthetic(fx["ndocs"], fx["vocab"], fx["seed"], values=True)
    covering = 0
    for i, q in enumerate(fx["queries"]):
        m = ix.match(o_query(q))
        ctx = f"vrbounds[{i}] {q}"
        check(m, q, ctx, counts=False)
        assert bits(m.max_possible) == bits(q["max_possible"]), f"{ctx}: max_possible"
        assert (m.lb, m.ub) == (q["lb"], q["ub"]), f"{ctx}: bounds"
        covering += q["vr"][1:] == [0, 1000000] and q["lb"] > 0
    assert covering >= 5, covering
