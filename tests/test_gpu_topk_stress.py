"""Tie masses against the oracle: the second matching pass, the overflow pool and the radix select of the top-k
kernel, pool exhaustion, and the top-k kernel's size classes with tied weights.

A bucket of the pruning histogram cannot separate equal weights (or equal sort keys), so more than keep_cap
matches tied at the top always overflow the top-k kernel's shared memory: the query is matched a second time
into a slice of the overflow pool and the exact top-k is found by a radix select over (key, ~docid).  The
corpus (tests/tie_corpus.py) is built so that every query set here has such a mass."""
import shutil
import tempfile

import pytest

from oracle import oracle as O
from tests import tie_corpus as T
from tests.util import assert_matches_oracle, assert_mset_equal
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ties():
    tmp = tempfile.mkdtemp(prefix="xgm_ties_")
    path, names = T.write_tie_corpus(tmp)
    yield path, {n: i for i, n in enumerate(names)}, xgm.Index.load_flat(path), O.Index.load_flat(path)
    shutil.rmtree(tmp, ignore_errors=True)


def pair(ids, op, terms, factors=None, **kw):
    """The same query for the CUDA path (by term name) and the oracle (by term id)."""
    x = xgm.Query(xgm.OP_AND if op == "AND" else xgm.OP_OR, list(terms), factors=factors, **kw)
    o = O.Query(op=O.OP_AND if op == "AND" else O.OP_OR, terms=[ids[t] for t in terms], factors=factors, **kw)
    return x, o


def run(searcher, orc, pairs, ctx):
    res = searcher.search([x for x, _ in pairs])
    refs = [orc.match(o) for _, o in pairs]
    for i, (m, ref, (x, _)) in enumerate(zip(res, refs, pairs)):
        assert_matches_oracle(m, ref, ctx=f"{ctx}[{i}] op={x.op} {x.terms} first={x.first} k={x.maxitems} "
                                          f"cal={x.check_at_least} sort={x.sort_by}/{int(x.sort_reverse)}")
    return res, refs, searcher.last_stats()


def top_tie(orc, o):
    """Matches sharing the best weight, by the oracle (the radix select's precondition)."""
    r = orc.match(O.Query(op=o.op, terms=o.terms, factors=o.factors, maxitems=T.NDOCS, check_at_least=T.NDOCS))
    return int((r.weights == r.weights.max()).sum()) if len(r.weights) else 0


def route_pairs(ids, specs):
    out = []
    for op, terms, factors in specs:
        for k in (1, 10, 100):
            for cal in (0, k + 1, 5000, T.NDOCS):
                out.append(pair(ids, op, terms, factors, maxitems=k, check_at_least=cal))
        out.append(pair(ids, op, terms, factors, first=7, maxitems=10))
    return out


@pytest.mark.parametrize("route", ["single", "and2", "and3", "and_nobitmap", "or", "or_tile_off", "or_wide",
                                   "and_zero"])
def test_tie_mass_takes_the_second_pass_and_matches_oracle(ties, route, monkeypatch):
    """Single term (xgm_and_kernel), 2- and 3-term AND (xgm_and_bm3_kernel), the same ANDs without membership
    bitmaps (block galloping), relevance-ordered OR of 2-5 leaves (bitmap-union tile + xgm_or3_kernel<1>, and
    xgm_or3_kernel<0> alone), OR of 6 leaves (xgm_or_kernel), AND with all factors 0 (every match weighs 0)."""
    path, ids, ix, orc = ties
    specs = {"and_nobitmap": T.TIE_ROUTES["and2"] + T.TIE_ROUTES["and3"],
             "or_tile_off": T.TIE_ROUTES["or"]}.get(route, T.TIE_ROUTES.get(route))
    if route == "and_nobitmap":
        monkeypatch.setenv("XGM_BITMAP_K", "0")
        ix = xgm.Index.load_flat(path)
        assert ix.info().nbitmaps == 0
    if route == "or_tile_off":
        monkeypatch.setenv("XGM_OR_TILE", "0")
    for op, terms, factors in specs:
        assert top_tie(orc, pair(ids, op, terms, factors)[1]) > T.KEEP_CAP, terms
    pairs = route_pairs(ids, specs)
    s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=256)
    res, _, stats = run(s, orc, pairs, route)
    print(f"{route}: {len(pairs)} queries, second_pass_queries={stats.second_pass_queries}")
    assert stats.second_pass_queries > 0
    assert all(m.status == 0 for m in res)


def test_large_k_and_the_c_abi_maximum(ties):
    """maxitems 1000 on every route, and first + maxitems = 4096 (the C-ABI's largest top-k) with first > 0: the
    top-k kernel then holds 8192 survivors and the tie mass of f_flat still exceeds that."""
    _, ids, ix, orc = ties
    pairs = [pair(ids, op, terms, fac, maxitems=1000, check_at_least=cal)
             for specs in T.TIE_ROUTES.values() for op, terms, fac in specs[:1] for cal in (0, 1001)]
    pairs.append(pair(ids, "AND", ["f_flat"], first=96, maxitems=4000))
    pairs.append(pair(ids, "AND", ["t01", "t02"], first=1, maxitems=4095, check_at_least=T.NDOCS))
    pairs.append(pair(ids, "OR", ["t01", "t02", "t03"], first=4095, maxitems=1))
    assert top_tie(orc, pairs[-3][1]) > 8192
    s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=xgm.MAX_TOPK)
    res, _, stats = run(s, orc, pairs, "large_k")
    print(f"large_k: {len(pairs)} queries, second_pass_queries={stats.second_pass_queries}")
    assert stats.second_pass_queries > 0
    assert len(res[-3].docids) == 4000


def test_value_sort_tie_mass():
    """SORT_VAL and SORT_VAL_REL, forward and reverse, smallest and largest value, on a slot 90 % of the documents
    lack: the documents without a value share one key and fill the pool; the radix select runs over the five-word
    (value, weight, ~docid) key.  Also OR with a value sort (xgm_or3_kernel<0>)."""
    orc = O.Index.synthetic(T.VALUE_NDOCS, T.VALUE_VOCAB, values=True)
    voff, keys = T.value_slot_arrays(orc)
    terms = [(orc.name(t),) + tuple(orc.postings(t)) for t in range(orc.nterms)]
    ix = xgm.Index.from_postings(orc.doclen(), terms, value_slots={0: (voff, keys)})
    xq, oq = [], []
    for op, sets in ((xgm.OP_AND, T.VALUE_AND_SETS), (xgm.OP_OR, T.VALUE_OR_SETS)):
        for ts in sets:
            for sort_by in (xgm.SORT_VAL, xgm.SORT_VAL_REL):
                for rev in (False, True):
                    for use_max in (False, True):
                        for k, cal in ((10, 0), (100, T.VALUE_NDOCS)):
                            kw = dict(maxitems=k, check_at_least=cal, sort_by=sort_by, sort_reverse=rev)
                            xq.append(xgm.Query(op, ts, sort_slot=0, sort_use_max=use_max,
                                                sort_missing_key=T.missing_key(rev), **kw))
                            oq.append(O.Query(op=op, terms=ts, sort_slot=2 if use_max else 0, sort_keymaker=True,
                                              sort_missing=T.missing_key(rev), **kw))
    for ts in T.VALUE_AND_SETS:  # the radix select's precondition: a tie mass above keep_cap at the top key
        for rev in (False, True):
            r = orc.match(O.Query(op=O.OP_AND, terms=ts, maxitems=T.VALUE_NDOCS, sort_by=O.SORT_VAL, sort_slot=0,
                                  sort_reverse=rev, sort_keymaker=True, sort_missing=T.missing_key(rev)))
            assert int((r.sortvals == T.missing_key(rev)).sum()) > T.KEEP_CAP
            assert r.sortvals[0] == T.missing_key(rev)
    # every query here overflows with ~25k matches in its pool slice; the default pool (2^20 entries at this
    # corpus size) holds a few dozen such slices per batch, and a query that finds it full is declined
    s = xgm.Searcher(ix, max_batch=16, max_topk=256)
    second = []
    for a in range(0, len(xq), 16):
        res = s.search(xq[a:a + 16])
        second.append(s.last_stats().second_pass_queries)
        for i, (m, q) in enumerate(zip(res, oq[a:a + 16]), a):
            ref = orc.match(q)
            ctx = f"vsort[{i}] {xq[i]}"
            assert_matches_oracle(m, ref, ctx)
            assert list(m.sort_keys) == list(ref.sortvals), ctx
    print(f"value sort: {len(xq)} queries in batches of 16, second_pass_queries per batch={second}")
    assert all(n > 0 for n in second)


def test_pool_exhaustion_declines_only_that_query(ties, monkeypatch):
    """An overflow pool smaller than one tie mass: that query is declined (XGM_E_UNIMPLEMENTED, so the caller
    runs it elsewhere), never answered wrongly, and the rest of its batch is unaffected."""
    _, ids, ix, orc = ties
    monkeypatch.setenv("XGM_POOL_ENTRIES", "1000")
    pairs = [pair(ids, "AND", ["f_flat"], maxitems=10)]
    for n in T.EDGE_SIZES[:9]:  # up to 1025 matches: none of these needs the pool
        pairs.append(pair(ids, "AND", list(T.edge_names(n)), maxitems=10, check_at_least=n // 2))
    pairs += [pair(ids, "AND", ["r_rare"], maxitems=10), pair(ids, "AND", ["r_rare", "t01"], maxitems=10),
              pair(ids, "OR", ["r_rare", "t08"], maxitems=10)]
    assert top_tie(orc, pairs[0][1]) > 1000
    s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=64)
    res = s.search([x for x, _ in pairs])
    assert res[0].status == xgm.E_UNIMPLEMENTED
    assert s.last_stats().second_pass_queries == 0
    for i, (m, (x, o)) in enumerate(zip(res[1:], pairs[1:]), 1):
        assert_matches_oracle(m, orc.match(o), ctx=f"pool[{i}] {x.terms}")


def edge_pairs(ids, n, max_topk):
    out = []
    for k in (10, n - 1, n, n + 1):
        if k > max_topk:
            continue
        for cal in (0, (k + 1 + n) // 2 if k + 1 < n else n + 3):
            out.append(pair(ids, "AND", list(T.edge_names(n)), maxitems=k, check_at_least=cal))
    return out


@pytest.mark.parametrize("max_topk", [256, 2050])
def test_size_class_edges_with_ties(ties, max_topk):
    """2-term ANDs whose intersection is exactly N documents of three distinct weights, N at either side of the
    top-k kernel's size classes (64: one warp; 256: the pair pass; 1024: the merge sort, beyond it the histogram
    cut; 2048: keep_cap).  Up to 1024 matches the set is never pruned, so the bounds and the match count must be
    the oracle's exactly and no flag may be set.  Run as one batch (>= 64 queries: the one-warp kernel takes the
    smallest sets) and one batch per N."""
    _, ids, ix, orc = ties
    s = xgm.Searcher(ix, max_batch=256, max_topk=max_topk)
    all_pairs = [p for n in T.EDGE_SIZES for p in edge_pairs(ids, n, max_topk)]
    batches = [all_pairs * 2] + [edge_pairs(ids, n, max_topk) for n in T.EDGE_SIZES]
    assert len(batches[0]) >= 64 and all(len(b) < 64 for b in batches[1:])
    for b, pairs in enumerate(batches):
        res, refs, _ = run(s, orc, pairs, f"edges/{max_topk}/{b}")
        for m, ref, (x, o) in zip(res, refs, pairs):
            if ref.exact <= 1024:
                ctx = f"edges N={ref.exact} k={x.maxitems} cal={x.check_at_least}"
                assert m.flags == 0, ctx
                assert_mset_equal(m, ref, ctx, check_counts=True)
