"""Range-major bitmap ANDs whose queries share their driver list (the rarest required term): the planner packs up to
XGM_BM_RUN (6) of them into a run, and the AND kernel decodes the run's driver blocks once per range and probes them
for every query of the run.  A driver with far more queries than a run holds, runs of 1, 2 and 6 queries, term groups
and value ranges mixed inside runs, and tie masses that take the second matching pass while the other queries of their
run do not are compared with the oracle."""
import random

import pytest

from tests.test_gpu_work_split import bitmap_ands, corpus, pair, run  # noqa: F401  (corpus is a fixture)
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

RUN = 6  # queries per run (XGM_BM_RUN)
PROBES = range(30)  # more frequent than every driver below, so that the driver stays the rarest required term


def shared_driver(rng, driver, n, mixed=False):
    """n ANDs led by `driver`, each with its own probe terms; mixed: FILTER / AND_NOT / AND_MAYBE groups and value
    ranges over slot 0 in turn, so that neighbouring lanes of one flush hold queries with different tests."""
    out = []
    for i in range(n):
        t = rng.sample(PROBES, 4)
        kw = dict(maxitems=rng.choice([1, 10, 100]), check_at_least=rng.choice([0, 0, 30000]))
        if mixed:
            k = i % 5
            if k == 1:
                kw.update(filter_terms=t[2:3])
            elif k == 2:
                kw.update(not_terms=[rng.randrange(100, 600)])
            elif k == 3:
                kw.update(maybe_terms=t[2:4])
            elif k == 4:
                lo = rng.randrange(0, 900000)
                kw.update(filter=xgm.FILTER_MULTI_RANGE, range_lo=lo, range_hi=lo + rng.choice([50000, 300000]))
        out.append(pair(xgm.OP_AND, [driver] + t[:rng.choice([1, 2])], **kw))
    return out


def tie_run(rng):
    """Term 0 is the only term more frequent than term 1, so every AND led by term 1 is [1, 0] with more or less
    around it.  Two of them weigh every match 0 (a tie mass that overflows the first pass); the others carry AND_NOT,
    AND_MAYBE and value-range tests and keep their ordinary weights."""
    out = [pair(xgm.OP_AND, [1, 0], factors=[0.0, 0.0], maxitems=10),
           pair(xgm.OP_AND, [1, 0], maxitems=10),
           pair(xgm.OP_AND, [1, 0], not_terms=[rng.randrange(100, 600)], maxitems=100),
           pair(xgm.OP_AND, [1, 0], maybe_terms=[5, 9], maxitems=10),
           pair(xgm.OP_AND, [1, 0], filter=xgm.FILTER_MULTI_RANGE, range_lo=100000, range_hi=200000, maxitems=10),
           pair(xgm.OP_AND, [1, 0], factors=[0.0, 0.0], maxitems=100, check_at_least=30000)]
    return out


@pytest.mark.parametrize("bpi", [None, 1, 32])
@pytest.mark.parametrize("range_bits", [8, 14, 17])
def test_driver_runs(corpus, monkeypatch, range_bits, bpi):
    """40 ANDs led by one driver (7 runs), runs of 6, 2 and 1 queries, 12 ANDs with mixed tests led by one driver
    and two runs that hold two tie masses, among 250 other all-bitmap ANDs, at 118, 2 and 1 document ranges over
    the 30k docids and the default, 1 and 32 driver blocks per item (32: the widest block field of a queued
    candidate)."""
    ix, orc = corpus
    rng = random.Random(700 + range_bits)
    pairs = (bitmap_ands(rng, 250) + shared_driver(rng, 60, 40) + shared_driver(rng, 61, RUN)
             + shared_driver(rng, 62, 2) + shared_driver(rng, 63, 1) + shared_driver(rng, 64, 12, mixed=True)
             + tie_run(rng))
    rng.shuffle(pairs)
    monkeypatch.setenv("XGM_RANGE_BITS", str(range_bits))
    if bpi is not None:
        monkeypatch.setenv("XGM_BPI", str(bpi))
    res, st = run(ix, orc, pairs, f"driver runs, ranges 2^{range_bits} bpi {bpi}")
    print(f"range_bits={range_bits} bpi={bpi}: work_items {st.work_items}, second_pass_queries={st.second_pass_queries}")
    ties = [i for i, (x, _) in enumerate(pairs) if x.factors is not None and x.terms == [1, 0]]
    assert st.second_pass_queries >= 2 and all(res[i].status == 0 for i in ties)
