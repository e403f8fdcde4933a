"""How a batch's work is cut up must not change its results: range-major work lists with many document ranges,
driver blocks per work item, the OR kernels' routing knobs, and the batch sizes at which the planner switches
code paths (driver blocks per item at 16 and 256 queries, the one-warp top-k kernel from 64, range-major lists
from 256, planning on helper threads from 512).  Everything is compared with the oracle."""
import random

import pytest

from oracle import oracle as O
from tests.util import assert_matches_oracle, bits
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

ND, V = 30000, 20000


@pytest.fixture(scope="module")
def corpus():
    return xgm.Index.synthetic(ND, V, values=True), O.Index.synthetic(ND, V, values=True)


def pair(op, terms, **kw):
    """The same query for the CUDA path and the oracle.  sort_use_max=True is the oracle's slot 2."""
    use_max = kw.pop("sort_use_max", False)
    x = xgm.Query(op, list(terms), sort_slot=0, sort_use_max=use_max, **kw)
    o = O.Query(op=op, terms=list(terms), sort_slot=2 if use_max else 0, **kw)
    return x, o


def bitmap_ands(rng, n):
    """All-bitmap ANDs (every term among the 1500 most frequent), a third of them with FILTER / AND_NOT /
    AND_MAYBE groups."""
    out = []
    for i in range(n):
        pool = rng.sample(range(1000), 9)
        nb = rng.choice([2, 2, 3, 4])
        kw = dict(first=rng.choice([0, 0, 3]), maxitems=rng.choice([1, 10, 100]), check_at_least=rng.choice([0, 0, ND]))
        if i % 3 == 0:
            kw.update(filter_terms=pool[4:4 + rng.choice([0, 1])], not_terms=pool[5:5 + rng.choice([0, 1, 2])],
                      maybe_terms=pool[7:7 + rng.choice([1, 2])])
        out.append(pair(xgm.OP_AND, pool[:nb], **kw))
    return out


def run(ix, orc, pairs, ctx, max_topk=128):
    s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=max_topk)
    res = s.search([x for x, _ in pairs])
    for i, (m, (x, o)) in enumerate(zip(res, pairs)):
        ref = orc.match(o)
        assert_matches_oracle(m, ref, ctx=f"{ctx}[{i}] op={x.op} {x.terms} F{x.filter_terms} N{x.not_terms} "
                                          f"M{x.maybe_terms} k={x.maxitems}")
        if x.sort_by != xgm.SORT_REL:
            assert list(m.sort_keys) == list(ref.sortvals), f"{ctx}[{i}] sort keys"
    return res, s.last_stats()


@pytest.mark.parametrize("bpi", [1, 3, 32])
@pytest.mark.parametrize("range_bits", [8, 11, 14])
def test_range_major_work_lists(corpus, monkeypatch, range_bits, bpi):
    """300 all-bitmap ANDs at 2^range_bits documents per range (118, 15 or 2 ranges over 30k docids) and 1, 3 or
    32 driver blocks per item: blocks straddle range edges, items of odd length and of one block test how the
    bitmap kernel pairs driver blocks.  One query weighs every match 0 (factors 0), a tie mass that takes the
    second matching pass over the range-major items."""
    ix, orc = corpus
    pairs = bitmap_ands(random.Random(100 + range_bits), 300)
    pairs.append(pair(xgm.OP_AND, [0, 1], factors=[0.0, 0.0], maxitems=10))
    pairs.append(pair(xgm.OP_AND, [0, 2, 5], factors=[0.0, 0.0, 0.0], maxitems=100, check_at_least=ND))
    monkeypatch.setenv("XGM_BPI", str(bpi))
    _, one = run(ix, orc, pairs, "one range")  # the default range width covers the whole corpus
    monkeypatch.setenv("XGM_RANGE_BITS", str(range_bits))
    res, split = run(ix, orc, pairs, f"ranges 2^{range_bits} bpi {bpi}")
    print(f"range_bits={range_bits} bpi={bpi}: work_items {one.work_items} in one range, {split.work_items} split; "
          f"second_pass_queries={split.second_pass_queries}")
    # a range cuts an item short where it ends; with one block per item there is nothing to cut
    assert split.work_items > one.work_items if bpi > 1 else split.work_items == one.work_items
    assert split.second_pass_queries >= 2 and res[-2].status == 0 and res[-1].status == 0


def or_pairs(rng, n):
    out = []
    for _ in range(n):
        ts = rng.sample(range(600), rng.choice([2, 3, 4, 5]))
        out.append(pair(xgm.OP_OR, ts, first=rng.choice([0, 0, 4]), maxitems=rng.choice([1, 10, 100]),
                        check_at_least=rng.choice([0, 0, ND])))
    return out


@pytest.mark.parametrize("knob", [None, ("XGM_OR_TILE", "0"), ("XGM_OR_KERNEL", "1")])
def test_or_route_knobs(corpus, monkeypatch, knob):
    """Relevance-ordered OR of 2-5 bitmap leaves: by default the bitmap-union tile kernel then xgm_or3_kernel<1>;
    XGM_OR_TILE=0 keeps them in xgm_or3_kernel<0>; XGM_OR_KERNEL=1 sends them to the general xgm_or_kernel."""
    ix, orc = corpus
    if knob:
        monkeypatch.setenv(*knob)
    run(ix, orc, or_pairs(random.Random(200), 150), f"or {knob}")


def probes():
    """40 fixed queries: ANDs, ORs, term groups, value sorts (smallest / largest value, both directions)."""
    rng = random.Random(300)
    out = []
    for i in range(10):
        out.append(pair(xgm.OP_AND, rng.sample(range(400), rng.choice([1, 2, 3])), maxitems=rng.choice([10, 100]),
                        check_at_least=rng.choice([0, ND])))
    for i in range(10):  # counting the whole match set keeps MaxScore from skipping segments: exact counts
        out.append(pair(xgm.OP_OR, rng.sample(range(2000), rng.choice([2, 3, 5, 7])), maxitems=rng.choice([10, 100]),
                        check_at_least=ND))
    for i in range(10):
        pool = rng.sample(range(500), 8)
        out.append(pair(xgm.OP_AND, pool[:2], filter_terms=pool[2:3], not_terms=pool[3:3 + i % 3],
                        maybe_terms=pool[5:5 + 1 + i % 2], maxitems=10, check_at_least=rng.choice([0, ND])))
    for i in range(10):
        out.append(pair(xgm.OP_AND, rng.sample(range(300), 2), maxitems=rng.choice([10, 50]),
                        sort_by=xgm.SORT_VAL_REL if i % 2 else xgm.SORT_VAL, sort_reverse=bool(i % 4 >= 2),
                        sort_use_max=i >= 5, check_at_least=rng.choice([0, ND])))
    return out


def filler(n, seed):
    rng = random.Random(seed)
    return [pair(xgm.OP_AND, rng.sample(range(800), rng.choice([2, 3])), maxitems=10) for _ in range(n)]


def fingerprint(m, value_sort):
    """Every field of an MSet; sort keys only where the order has them."""
    return (m.status, m.flags, m.docids.tobytes(), m.weights.tobytes(),
            m.sort_keys.tobytes() if value_sort else b"", m.matches_lower_bound,
            m.matches_estimated_raw, m.matches_upper_bound, m.exact_matches, bits(m.max_possible),
            bits(m.max_attained), bits(m.percent_scale_factor))


def test_batch_size_thresholds_do_not_change_results(corpus):
    """The 40 probes in batches of 1, 15, 16, 63, 64, 255, 256, 511 and 512 queries (seeded filler around them):
    every probe's MSet is byte-identical at every batch size and equals the oracle's."""
    ix, orc = corpus
    ps = probes()
    s = xgm.Searcher(ix, max_batch=512, max_topk=128)
    seen = {}
    for B in (1, 15, 16, 63, 64, 255, 256, 511, 512):
        per = max(1, B // 4)
        for a in range(0, len(ps), per):
            chunk = ps[a:a + per]
            batch = chunk + filler(B - len(chunk), seed=B * 1000 + a)
            res = s.search([x for x, _ in batch])
            for j, m in enumerate(res[:len(chunk)]):
                seen.setdefault(a + j, {})[B] = fingerprint(m, ps[a + j][0].sort_by != xgm.SORT_REL)
                if B == 1:
                    x, o = ps[a + j]
                    ref = orc.match(o)
                    assert_matches_oracle(m, ref, ctx=f"probe {a + j} {x}")
                    if x.sort_by != xgm.SORT_REL:
                        assert list(m.sort_keys) == list(ref.sortvals), f"probe {a + j} sort keys"
    for i, by_size in seen.items():
        first = by_size[1]
        for B, fp in by_size.items():
            assert fp == first, f"probe {i} {ps[i][0]}: batch of {B} differs from a batch of 1"
    # the pairs either side of a threshold really take different paths
    launches = {}
    for B in (63, 64, 255, 256):
        s.search([x for x, _ in filler(B, seed=7)])  # filler(64) extends filler(63) by one query
        launches[B] = s.last_stats().kernel_launches
    print(f"kernel_launches by batch size: {launches}")
    assert launches[64] > launches[63] and launches[256] > launches[255]
