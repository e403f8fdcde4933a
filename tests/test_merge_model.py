"""CPU tests: the library's host merge (xgm_merge_msets) against tests/merge_model.merge_ref, a plain restatement
of Matcher::merge_mset + MSet::Internal::merge_stats, on seeded random shards and on the inputs where a merge
goes wrong: ties everywhere, weights one ulp apart, equal sort keys over different weights, empty parts, `first`
past the merged size and parts that tie on max_attained."""
import math
import random
import struct

import numpy as np
import pytest

from tests.merge_model import SORT_REL, SORT_REL_VAL, SORT_VAL, SORT_VAL_REL, Part, merge_ref, msetcmp
from xapiand_b200 import xgm

ORDERS = [(SORT_REL, False), (SORT_VAL_REL, False), (SORT_VAL_REL, True), (SORT_VAL, False), (SORT_VAL, True),
          (SORT_REL_VAL, False), (SORT_REL_VAL, True)]


def bits(x):
    return struct.pack("<d", float(x))


def sort_part(docids, weights, keys, sort_by, reverse):
    """A shard's MSet order: the merge order over local docids (unshard is monotone within a shard)."""
    import functools
    before = msetcmp(sort_by, reverse)
    items = sorted(zip(weights, docids, keys),
                   key=functools.cmp_to_key(lambda a, b: -1 if before(a, b) else (1 if before(b, a) else 0)))
    return [d for _, d, _ in items], [w for w, _, _ in items], [k for _, _, k in items]


def make_part(rng, n, draw_w, draw_k, sort_by, reverse, maxdoc=60):
    docids = rng.sample(range(1, maxdoc + 1), n)
    d, w, k = sort_part(docids, [draw_w() for _ in range(n)], [draw_k() for _ in range(n)], sort_by, reverse)
    mp = max(w, default=0.0)
    return Part(d, w, k, lb=n, est=n + rng.randrange(0, 5), ub=n + rng.randrange(5, 50),
                max_possible=mp * (1.0 + rng.random()), max_attained=mp, percent_scale_factor=rng.random())


def host_merge(parts, first, maxitems, sort_by, reverse):
    n = len(parts)
    ms = [xgm.MSet(xgm.unshard(np.asarray(p.docids, np.uint32), i, n), np.asarray(p.weights, np.float64),
                   np.asarray(p.keys, np.uint64), 0, p.lb, p.est, p.ub, p.max_possible, p.max_attained,
                   p.percent_scale_factor, len(p.docids), 0) for i, p in enumerate(parts)]
    return xgm.merge_msets(ms, first, maxitems, sort_by, reverse)


def assert_same(got, ref, sort_by, ctx):
    assert list(got.docids) == ref.docids, f"{ctx}: docids\n got {list(got.docids)}\n ref {ref.docids}"
    assert [bits(w) for w in got.weights] == [bits(w) for w in ref.weights], f"{ctx}: weights"
    if sort_by != SORT_REL:
        assert list(got.sort_keys) == ref.keys, f"{ctx}: sort keys"
    assert (got.matches_lower_bound, got.matches_estimated_raw, got.matches_upper_bound) == (ref.lb, ref.est, ref.ub), ctx
    assert bits(got.max_possible) == bits(ref.max_possible), f"{ctx}: max_possible"
    assert bits(got.max_attained) == bits(ref.max_attained), f"{ctx}: max_attained"
    assert bits(got.percent_scale_factor) == bits(ref.percent_scale_factor), f"{ctx}: percent_scale_factor"


def test_merge_ref_by_hand():
    """The model on an example worked out by hand: two shards, docid 2 of shard 1 is global 4, and the tie at 2.0
    goes to the smaller global docid; the percentage scale comes from the shard with the larger max_attained."""
    a = Part([3, 1], [2.0, 1.0], lb=2, est=2, ub=2, max_possible=5.0, max_attained=2.0, percent_scale_factor=0.5)
    b = Part([2, 5], [2.0, 1.5], lb=2, est=3, ub=9, max_possible=4.0, max_attained=2.0, percent_scale_factor=0.25)
    c = Part([1], [3.0], lb=1, est=1, ub=1, max_possible=3.0, max_attained=3.0, percent_scale_factor=0.125)
    m = merge_ref([a, b], 0, 10)
    assert m.docids == [4, 5, 10, 1] and m.weights == [2.0, 2.0, 1.5, 1.0]
    assert (m.lb, m.est, m.ub, m.max_possible, m.max_attained, m.percent_scale_factor) == (4, 5, 11, 5.0, 2.0, 0.5)
    m = merge_ref([a, b, c], 1, 2)
    assert m.docids == [5, 7] and m.percent_scale_factor == 0.125


@pytest.mark.parametrize("sort_by,reverse", ORDERS)
def test_host_merge_matches_model_random(sort_by, reverse):
    rng = random.Random(1000 + 10 * sort_by + reverse)
    for it in range(300):
        nparts = rng.choice([1, 2, 3, 5, 8, 16])
        wset = [rng.uniform(0, 10) for _ in range(rng.choice([1, 3, 50]))]
        kset = [rng.randrange(0, 1 << 64) for _ in range(rng.choice([1, 2, 4, 40]))]
        parts = [make_part(rng, rng.choice([0, 1, 5, 20, 40]), lambda: rng.choice(wset), lambda: rng.choice(kset),
                           sort_by, reverse) for _ in range(nparts)]
        total = sum(len(p.docids) for p in parts)
        first = rng.choice([0, 0, 1, 7, total, total + 3])
        maxitems = rng.choice([0, 1, 10, 1000])
        assert_same(host_merge(parts, first, maxitems, sort_by, reverse),
                    merge_ref(parts, first, maxitems, sort_by, reverse), sort_by, f"random[{it}] {sort_by}/{reverse}")


def ulp_neighbours(base, spread):
    out = [base]
    lo = hi = base
    for _ in range(spread):
        lo, hi = math.nextafter(lo, -math.inf), math.nextafter(hi, math.inf)
        out += [lo, hi]
    return out


ADVERSARIAL = ["all_equal", "ulp", "keys_equal_weights_up", "keys_equal_weights_down", "empty_parts",
               "first_past_end", "max_attained_tie"]


@pytest.mark.parametrize("case", ADVERSARIAL)
@pytest.mark.parametrize("sort_by,reverse", ORDERS)
def test_host_merge_matches_model_adversarial(case, sort_by, reverse):
    rng = random.Random(2000 + 100 * ADVERSARIAL.index(case) + 10 * sort_by + reverse)
    ulps = ulp_neighbours(2.5, 2)
    for it in range(40):
        nparts = rng.choice([2, 3, 4, 7])
        draw_w = lambda: rng.uniform(0, 5)  # noqa: E731
        draw_k = lambda: rng.randrange(0, 1000)  # noqa: E731
        sizes = [rng.choice([1, 5, 20] if case not in ("all_equal", "ulp") else [5, 20]) for _ in range(nparts)]
        if case == "all_equal":
            draw_w, draw_k = (lambda: 1.25), (lambda: 7)
        elif case == "ulp":
            draw_w = lambda: rng.choice(ulps)  # noqa: E731
            draw_k = lambda: rng.choice([3, 4])  # noqa: E731
        elif case.startswith("keys_equal"):  # one key, weights rising or falling with the docid
            draw_k = lambda: 42  # noqa: E731
        elif case == "empty_parts":
            sizes = [0 if p % 2 == 0 else s for p, s in enumerate(sizes)]
        parts = [make_part(rng, s, draw_w, draw_k, sort_by, reverse) for s in sizes]
        if case.startswith("keys_equal"):
            up = case.endswith("up")
            for p in parts:
                ws = sorted(p.weights, reverse=not up)
                p.docids, p.weights, p.keys = sort_part(sorted(p.docids), ws, p.keys, sort_by, reverse)
            assert len({w for p in parts for w in p.weights}) > 1
        if case == "max_attained_tie":
            for i, p in enumerate(parts):
                p.max_attained, p.percent_scale_factor = 9.0, 0.1 * (i + 1)
        total = sum(sizes)
        first = total + rng.choice([0, 1, 100]) if case == "first_past_end" else rng.choice([0, 2])
        maxitems = rng.choice([1, 10, 1000])
        ref = merge_ref(parts, first, maxitems, sort_by, reverse)
        if case == "all_equal" or case == "ulp":  # equal items in different parts really are there
            seen = {}
            for i, p in enumerate(parts):
                for w, k in zip(p.weights, p.keys):
                    seen.setdefault((w, k), set()).add(i)
            assert any(len(v) > 1 for v in seen.values())
        if case == "first_past_end":
            assert ref.docids == []
        if case == "max_attained_tie":
            assert ref.percent_scale_factor == 0.1
        assert_same(host_merge(parts, first, maxitems, sort_by, reverse), ref, sort_by, f"{case}[{it}] {sort_by}/{reverse}")
