"""Shared helpers for the parity tests: seeded query generators and result comparison."""
import random
import struct

import numpy as np


def bits(x: float) -> bytes:
    return struct.pack("<d", float(x))


def gen_queries(rng: random.Random, n, topranks, ndocs, ops=("AND",), ks=(3,), maxitems=(100,), first=(0,),
                check_all=False):
    out = []
    for _ in range(n):
        op = rng.choice(ops)
        k = rng.choice(ks)
        terms = rng.sample(range(topranks), k)
        out.append(dict(op=op, terms=terms, first=rng.choice(first), maxitems=rng.choice(maxitems),
                        check_at_least=ndocs if check_all else 0))
    return out


def assert_matches_oracle(got, ref, ctx=""):
    """assert_mset_equal, except that what an approximation flag licenses is checked in its weaker form:
    with BOUNDS_APPROX (1) lb <= ref.lb and lb <= est <= ub; with COUNT_LOWER_BOUND (2) exact <= ref.exact.
    The upper bound is always exact."""
    approx = bool(got.flags & 1)
    assert_mset_equal(got, ref, ctx, check_counts=not approx)
    assert got.matches_upper_bound == ref.ub, f"{ctx}: ub {got.matches_upper_bound} vs {ref.ub}"
    if got.flags & 2:
        assert got.exact_matches <= ref.exact, f"{ctx}: exact {got.exact_matches} > {ref.exact}"
    else:
        assert got.exact_matches == ref.exact, f"{ctx}: exact {got.exact_matches} vs {ref.exact}"
    if approx:
        assert got.matches_lower_bound <= ref.lb, f"{ctx}: lb {got.matches_lower_bound} > {ref.lb}"
        assert got.matches_lower_bound <= got.matches_estimated_raw <= got.matches_upper_bound, f"{ctx}: lb/est/ub"


def assert_mset_equal(got, ref, ctx="", check_counts=True):
    """got: xgm.MSet, ref: oracle MSet. docids in order, weights bit-exact."""
    assert got.status == 0, f"{ctx}: status {got.status}"
    assert list(got.docids) == list(ref.docids), f"{ctx}: docids differ\n got {list(got.docids)[:10]}\n ref {list(ref.docids)[:10]}"
    gw = np.asarray(got.weights, np.float64)
    rw = np.asarray(ref.weights, np.float64)
    assert gw.tobytes() == rw.tobytes(), f"{ctx}: weights differ (max rel {np.max(np.abs(gw-rw)/np.maximum(rw,1e-300)) if len(gw) else 0})"
    assert bits(got.max_possible) == bits(ref.max_possible), f"{ctx}: max_possible {got.max_possible} vs {ref.max_possible}"
    assert bits(got.max_attained) == bits(ref.max_attained), f"{ctx}: max_attained {got.max_attained} vs {ref.max_attained}"
    if check_counts:
        assert (got.matches_lower_bound, got.matches_estimated_raw, got.matches_upper_bound) == (ref.lb, ref.est, ref.ub), \
            f"{ctx}: bounds {(got.matches_lower_bound, got.matches_estimated_raw, got.matches_upper_bound)} vs {(ref.lb, ref.est, ref.ub)}"
        assert got.exact_matches == ref.exact, f"{ctx}: exact {got.exact_matches} vs {ref.exact}"
        assert bits(got.percent_scale_factor) == bits(ref.percent_scale_factor), f"{ctx}: percent scale"
