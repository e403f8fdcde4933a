"""Range-major bitmap ANDs whose queries share their probe list (the second-rarest required term): the planner
groups them per range and the AND kernel hands a group to the warps of one CTA, which take its items from a
shared cursor.  Groups larger than a CTA's warp count, FILTER / AND_NOT groups and tie masses that take the second
matching pass over the grouped list are compared with the oracle."""
import random

import pytest

from tests.test_gpu_work_split import ND, bitmap_ands, corpus, pair, run  # noqa: F401  (corpus is a fixture)
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

PROBE = 2  # a frequent term: every rarer driver probes its bitmap


def shared_probe_ands(rng, n):
    """n two-term ANDs of a rarer driver and PROBE, a third of them with FILTER / AND_NOT groups of more frequent
    terms, so that PROBE stays the probe list."""
    out = []
    for i in range(n):
        kw = dict(maxitems=rng.choice([1, 10, 100]), check_at_least=rng.choice([0, 0, ND]))
        if i % 3 == 0:
            kw.update(filter_terms=[rng.choice([0, 1])], not_terms=rng.sample([3, 4, 6], rng.choice([1, 2])))
        out.append(pair(xgm.OP_AND, [rng.randrange(20, 1000), PROBE], **kw))
    return out


@pytest.mark.parametrize("range_bits", [8, 14, 17])
def test_shared_probe_groups(corpus, monkeypatch, range_bits):
    """40 ANDs probing one list (more than a CTA has warps) among 300 others, and two zero-weight tie masses that
    probe it too, at 118, 2 and 1 document ranges over the 30k docids."""
    ix, orc = corpus
    rng = random.Random(500 + range_bits)
    pairs = bitmap_ands(rng, 300) + shared_probe_ands(rng, 40)
    rng.shuffle(pairs)
    pairs.append(pair(xgm.OP_AND, [5, PROBE], factors=[0.0, 0.0], maxitems=10))
    pairs.append(pair(xgm.OP_AND, [0, PROBE, 5], factors=[0.0, 0.0, 0.0], maxitems=100, check_at_least=ND))
    monkeypatch.setenv("XGM_RANGE_BITS", str(range_bits))
    res, st = run(ix, orc, pairs, f"shared probe, ranges 2^{range_bits}")
    assert st.second_pass_queries >= 2 and res[-2].status == 0 and res[-1].status == 0
