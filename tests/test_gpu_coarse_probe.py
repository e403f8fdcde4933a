"""The bitmap AND kernel's coarse probe: for an AND whose second list (terms[1]) is sparse, a driver posting is first
tested against a bit per 8 docids and only then against the membership bitmap.  A corpus where every driver posting
of long stretches shares its 8-docid group with a member of the probe list, but is not one, docids on 8-, 32-, 256-docid
and range boundaries, runs mixing queries of both probe routes with term groups and value ranges, tie masses that take
the second matching pass, and runs of every length up to XGM_BM_RUN are compared with the oracle."""
import os
import random
import shutil
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.flatfile import write_flat
from tests.test_gpu_work_split import corpus, pair, run  # noqa: F401  (corpus is a fixture)
from tests.util import assert_matches_oracle
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

RUN = 6  # queries per run (XGM_BM_RUN)
COARSE_MAX = 0.1  # the planner's largest coarse pass rate for the coarse route
LAST = 1000077  # the last 256-docid group is partial
BOUNDS = [1, 2, 7, 8, 9, 31, 32, 33, 255, 256, 257, 2047, 2048, 16383, 16384, 16385, 131071, 131072, 131073,
          262143, 262144, 262145, LAST - 1, LAST]


def coarse_route(tf, lastdocid):
    return pass_rate(tf, lastdocid) <= COARSE_MAX


def pass_rate(tf, lastdocid):
    return 1.0 - (1.0 - tf / lastdocid) ** 8


def make_corpus(tmp):
    rng = np.random.default_rng(11)
    every = np.arange(1, LAST + 1, dtype=np.uint32)
    # stretch of misses: the probe list holds the multiples of 64 in [1024, 60000), the driver one docid 1..7 above
    # each, in the same 8-docid group: every coarse test passes and every fine test must reject
    base = np.arange(1024, 60000, 64, dtype=np.uint32)
    near = base + rng.integers(1, 8, size=len(base)).astype(np.uint32)
    hits = np.sort(rng.choice(np.arange(60000, 100000, dtype=np.uint32), 300, replace=False))  # true matches
    tie_b = np.sort(rng.choice(np.arange(100000, 300000, dtype=np.uint32), 3600, replace=False))
    tie_d = np.sort(rng.choice(tie_b, 3400, replace=False))  # matches of the tie mass
    bnd = np.array(BOUNDS, np.uint32)
    beside = np.setdiff1d(np.concatenate([bnd - 1, bnd + 1]), np.concatenate([bnd, [0]]))  # misses next to the hits
    beside = beside[beside <= LAST]
    sets = {
        "a_drv": np.unique(np.concatenate([near, hits, tie_d, bnd, beside])),
        "b_sparse": np.unique(np.concatenate([base, hits, tie_b, bnd])),
        "c_dense": np.unique(np.concatenate([np.sort(rng.choice(every, 300000, replace=False)), bnd])),
        "d_filt": np.sort(rng.choice(every, 100000, replace=False)),
        "e_not": np.sort(rng.choice(every, 10000, replace=False)),
        "f_maybe": np.sort(rng.choice(every, 50000, replace=False)),
        "g_drv": np.unique(np.concatenate([np.sort(rng.choice(every, 2500, replace=False)), hits, bnd])),
    }
    terms = [(n, d.astype(np.uint32), rng.integers(1, 6, size=len(d)).astype(np.uint32)) for n, d in sorted(sets.items())]
    total = np.zeros(LAST + 1, np.uint64)
    for _, d, w in terms:
        total[d] += w
    doclen = (total + rng.integers(1, 300, size=LAST + 1).astype(np.uint64)).astype(np.uint32)
    doclen[0] = 0
    path = os.path.join(tmp, "coarse.flat")
    write_flat(path, doclen, terms)
    return path, [t[0] for t in terms], sets


@pytest.fixture(scope="module")
def crafted():
    tmp = tempfile.mkdtemp(prefix="xgm_coarse_")
    path, names, sets = make_corpus(tmp)
    yield xgm.Index.load_flat(path), O.Index.load_flat(path), names, sets
    shutil.rmtree(tmp, ignore_errors=True)


def test_crafted_corpus_takes_both_routes(crafted):
    _, _, _, sets = crafted
    # b_sparse stays on the coarse route with a wide margin (pass rate ~0.04), and above the bitmap threshold
    assert pass_rate(len(sets["b_sparse"]), LAST) <= COARSE_MAX / 2 and len(sets["b_sparse"]) >= LAST // 256
    assert not coarse_route(len(sets["c_dense"]), LAST)
    assert len(sets["a_drv"]) < len(sets["b_sparse"]) and len(sets["g_drv"]) < len(sets["b_sparse"])


def crafted_queries(names):
    """RUN * 2 + RUN - 1 ANDs led by a_drv (runs of RUN, RUN and RUN - 1 queries) and one led by g_drv (a run of 1);
    the probe list is b_sparse (coarse route) or c_dense (fine route) in turn, with term groups and a tie mass."""
    ix_of = {n: i for i, n in enumerate(names)}

    def q(terms, **kw):
        x = xgm.Query(xgm.OP_AND, list(terms), **kw)
        okw = dict(kw)
        for g in ("filter_terms", "not_terms", "maybe_terms"):
            if g in okw:
                okw[g] = [ix_of[t] for t in okw[g]]
        o = O.Query(op=O.OP_AND, terms=[ix_of[t] for t in terms], **okw)
        return x, o

    ex = dict(maxitems=100, check_at_least=LAST)
    a = [q(["a_drv", "b_sparse"], **ex),
         q(["a_drv", "c_dense"], **ex),
         q(["a_drv", "b_sparse", "c_dense"], maxitems=10),
         q(["a_drv", "b_sparse"], factors=[0.0, 0.0], maxitems=10),  # 3700 tied matches: second pass
         q(["a_drv", "c_dense"], filter_terms=["d_filt"], maxitems=10),
         q(["a_drv", "b_sparse"], not_terms=["e_not"], maybe_terms=["f_maybe"], maxitems=10),
         q(["a_drv", "c_dense"], not_terms=["e_not"], maxitems=1, check_at_least=LAST),
         q(["a_drv", "b_sparse"], filter_terms=["c_dense"], maxitems=100)]
    a += [q(["a_drv", "b_sparse" if i % 2 else "c_dense"], first=i + 1, maxitems=10) for i in range(3 * RUN - 1 - len(a))]
    assert len(a) == 3 * RUN - 1
    return a + [q(["g_drv", "b_sparse"], **ex)]


@pytest.mark.parametrize("order", ["level", 8, 14, 17])
def test_coarse_probe_crafted(crafted, monkeypatch, order):
    """The crafted ANDs alone (level order), and padded with 250 single-term queries to a range-major batch at
    2^8, 2^14 and 2^17 docids per range."""
    ix, orc, names, sets = crafted
    pairs = crafted_queries(names)
    if order != "level":
        rng = random.Random(order)
        pad = [rng.choice(names) for _ in range(250)]
        pairs += [(xgm.Query(xgm.OP_AND, [t], maxitems=10), O.Query(op=O.OP_AND, terms=[names.index(t)], maxitems=10))
                  for t in pad]
        monkeypatch.setenv("XGM_RANGE_BITS", str(order))
    s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=128)
    res = s.search([x for x, _ in pairs])
    for i, (m, (x, o)) in enumerate(zip(res, pairs)):
        assert_matches_oracle(m, orc.match(o), ctx=f"coarse {order}[{i}] {x.terms} F{x.filter_terms} N{x.not_terms} "
                                                   f"M{x.maybe_terms}")
    # the coarse-hit / fine-miss stretch adds no match: the count is the true intersection
    want = len(np.intersect1d(sets["a_drv"], sets["b_sparse"]))
    assert res[0].status == 0 and res[0].exact_matches == want == orc.match(pairs[0][1]).exact
    st = s.last_stats()
    print(f"order={order}: work_items {st.work_items}, second_pass_queries {st.second_pass_queries}")
    assert st.second_pass_queries >= 1 and res[3].status == 0


def test_coarse_probe_mixed_runs(corpus, monkeypatch):
    """Synthetic corpus: ANDs led by one driver whose probe term is on either side of the coarse threshold, with
    FILTER / AND_NOT / AND_MAYBE groups and value ranges, at 2^8, 2^14 and 2^17 docids per range."""
    ix, orc = corpus
    nd = ix.info().lastdocid
    tf = {t: len(orc.postings(t)[0]) for t in range(0, 2000)}
    # sparse: well inside the coarse route (half the threshold), with a bitmap
    sparse = [t for t in range(40, 2000) if pass_rate(tf[t], nd) <= COARSE_MAX / 2 and tf[t] >= nd // 256][:40]
    dense = [t for t in range(1, 40) if not coarse_route(tf[t], nd)]
    assert len(sparse) >= 20 and len(dense) >= 5
    driver = next(t for t in range(sparse[-1] + 1, 2000) if tf[t] < tf[sparse[-1]])  # rarer than every probe term
    rng = random.Random(900)
    pairs = []
    for i in range(4 * RUN):
        probe = rng.choice(sparse if i % 2 == 0 else dense)
        kw = dict(maxitems=rng.choice([1, 10, 100]), check_at_least=rng.choice([0, 30000]))
        k = i % 4
        if k == 1:
            kw.update(filter_terms=[rng.choice(dense)])
        elif k == 2:
            kw.update(not_terms=[rng.choice(sparse)], maybe_terms=[rng.choice(dense)])
        elif k == 3:
            lo = rng.randrange(0, 900000)
            kw.update(filter=xgm.FILTER_MULTI_RANGE, range_lo=lo, range_hi=lo + 300000)
        pairs.append(pair(xgm.OP_AND, [driver, probe], **kw))
    pairs += [pair(xgm.OP_AND, [rng.choice(sparse + dense)], maxitems=10) for _ in range(256 - len(pairs))]
    for rb in (8, 14, 17):
        monkeypatch.setenv("XGM_RANGE_BITS", str(rb))
        run(ix, orc, pairs, f"coarse mixed 2^{rb}")
