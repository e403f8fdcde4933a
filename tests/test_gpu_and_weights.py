"""The AND kernels' weight sums against the oracle on a corpus where a slightly wrong sum changes the result bits
(tests/and_corpus.py; tests/test_and_corpus.py pins the witnesses): FILTER terms and factor-0 leaves over wdf-0
postings, the weighted range source at every place of the sum, AND_MAYBE trees of 9..15 optional leaves, wdfs that
differ from their neighbours at block and group edges, and several AND_NOT lists.

Every witness query runs under k1 x b x min_normlen (and k3 with wqf and factors, 0 among them) on every AND route:
  level        fewer than 256 queries a batch: xgm_and_bm3_kernel (fine and coarse probes of terms[1]) where every
               list but the driver has a bitmap, xgm_and_kernel for the rest and for single-term bases
  no_bitmap    XGM_BITMAP_K=0: every query on xgm_and_kernel, every probe by decoding blocks
  mid_bitmap   XGM_BITMAP_K=MID_BITMAP_K: p_coarse loses its bitmap, so one query mixes both kinds of probe
  rb{8,14,17}_bpi{1,32}
               one range-major batch at 2^8, 2^14 and 2^17 docids per range, 1 and 32 driver blocks per item"""
import shutil
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import and_corpus as A
from tests.percent_corpus import device_slot
from tests.util import assert_matches_oracle
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

MAX_TOPK = 128
ALL = A.NDOCS
# (maxitems, first, check_at_least): a top-100 MSet holds every CORE match
ARGS = ((100, 0, 0), (10, 0, 11), (1, 0, ALL), (10, 5, 0))


@pytest.fixture(scope="module")
def corpus():
    tmp = tempfile.mkdtemp(prefix="xgm_andw_")
    path, built = A.write_and_corpus(tmp)
    doclen, terms, doccount, nvals, vals, _ = built
    orc = O.Index.load_flat(path)
    orc.set_slot0(nvals, vals)
    yield dict(orc=orc, ids={t[0]: i for i, t in enumerate(terms)}, doclen=doclen, terms=terms, doccount=doccount,
               slot={0: device_slot(nvals, vals)})
    shutil.rmtree(tmp, ignore_errors=True)


def device_index(c):
    return xgm.Index.from_postings(c["doclen"], c["terms"], doccount=c["doccount"], value_slots=c["slot"])


def pair(c, s, cell, maxitems, first, cal):
    o = A.oracle_query(c["ids"], s, cell, maxitems=maxitems, first=first, check_at_least=cal)
    kw = dict(first=first, maxitems=maxitems, check_at_least=cal, factors=o.factors, wqf=o.wqf, bm25=o.bm25)
    if s["src"] is not None:  # device keys are the values plus one
        kw.update(filter=xgm.FILTER_MULTI_RANGE, filter_slot=0, range_lo=1, range_hi=A.VALUE_MAX + 1,
                  filter_weighted=True, filter_factor=s["src"])
    x = xgm.Query(xgm.OP_AND, list(s["names"]), filter_terms=list(s["filter_terms"]), not_terms=list(s["not_terms"]),
                  maybe_terms=list(s["maybe"]), **kw)
    return x, o


def witness_pairs(c):
    return [pair(c, s, cell, *a) for s in A.witness_specs() for cell in A.WEIGHTINGS for a in ARGS]


_refs = {}


def oracle(orc, o):
    key = repr(o)
    if key not in _refs:
        _refs[key] = orc.match(o)
    return _refs[key]


def check(c, pairs, res, route):
    for i, ((x, o), m) in enumerate(zip(pairs, res)):
        ctx = (f"{route}[{i}] {list(x.terms)} F{list(x.filter_terms)} N{list(x.not_terms)} M{len(x.maybe_terms)} "
               f"src={x.filter_factor if x.filter_weighted else None} fac={x.factors} wqf={x.wqf} bm25={x.bm25} "
               f"k={x.maxitems} first={x.first} cal={x.check_at_least}")
        assert not np.isnan(m.weights).any() and not np.isnan(m.max_attained), ctx
        assert_matches_oracle(m, oracle(c["orc"], o), ctx)


LEVEL = {"level": {}, "no_bitmap": {"XGM_BITMAP_K": "0"}, "mid_bitmap": {"XGM_BITMAP_K": str(A.MID_BITMAP_K)}}


@pytest.mark.parametrize("route", sorted(LEVEL))
def test_and_weights_level_order(corpus, monkeypatch, route):
    for k, v in LEVEL[route].items():
        monkeypatch.setenv(k, v)
    ix = device_index(corpus)
    if route == "no_bitmap":
        assert ix.info().nbitmaps == 0
    pairs = witness_pairs(corpus)
    res = xgm.Searcher(ix, max_batch=255, max_topk=MAX_TOPK).search([x for x, _ in pairs])
    check(corpus, pairs, res, route)


@pytest.mark.parametrize("bpi", [1, 32])
@pytest.mark.parametrize("range_bits", [8, 14, 17])
def test_and_weights_range_major(corpus, monkeypatch, range_bits, bpi):
    monkeypatch.setenv("XGM_RANGE_BITS", str(range_bits))
    monkeypatch.setenv("XGM_BPI", str(bpi))
    pairs = witness_pairs(corpus)
    assert len(pairs) >= 256
    res = xgm.Searcher(device_index(corpus), max_batch=len(pairs), max_topk=MAX_TOPK).search([x for x, _ in pairs])
    check(corpus, pairs, res, f"rb{range_bits}_bpi{bpi}")


class _CudaArray:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2}


def test_replay_gives_the_submitted_msets(corpus, monkeypatch):
    """A range-major batch of the witness queries (one weighting) with tie masses that take the second matching pass,
    submitted once and replayed three times: the device results (weights, docids, counts) equal the submitted
    MSets bit for bit every time."""
    import torch
    monkeypatch.setenv("XGM_RANGE_BITS", "14")
    c = corpus
    cells = ("k1=1.2 b=0.5 mnl=0.5", "k1=0.0 b=1.0 mnl=0.0")
    pairs = [pair(c, s, cell, *a) for s in A.witness_specs() for cell in cells for a in ARGS]
    # every match weighs 0: thousands of tied matches overflow the first pass
    ties = [A.spec(("p_big", "p_huge"), factors=(0.0, 0.0)), A.spec(("z_freq", "p_huge"), factors=(0.0, 0.0))]
    pairs += [pair(c, s, "k1=1.2 b=0.5 mnl=0.5", 10, 0, 0) for s in ties]
    assert len(pairs) >= 256
    nq = len(pairs)
    s = xgm.Searcher(device_index(c), max_batch=nq, max_topk=MAX_TOPK)
    res = s.search([x for x, _ in pairs])
    assert s.last_stats().second_pass_queries >= 1
    check(c, pairs, res, "replay submit")
    wptr, dptr, cptr, stride = s.device_results()
    for r in range(3):
        s.replay()
        torch.cuda.synchronize()
        w = torch.as_tensor(_CudaArray(wptr, (nq * stride,), "<f8"), device="cuda").cpu().numpy().reshape(nq, stride)
        d = torch.as_tensor(_CudaArray(dptr, (nq * stride,), "<u4"), device="cuda").view(torch.int32).cpu().numpy()
        n = torch.as_tensor(_CudaArray(cptr, (nq * 8,), "<u4"), device="cuda").view(torch.int32).cpu().numpy()
        d = d.view(np.uint32).reshape(nq, stride)
        for i, m in enumerate(res):
            k = int(n[8 * i])
            assert k == m.first + len(m.docids) or k == len(m.docids), (r, i, k, len(m.docids))
            got_d, got_w = d[i, k - len(m.docids):k], w[i, k - len(m.docids):k]
            assert got_d.tobytes() == m.docids.tobytes() and got_w.tobytes() == m.weights.tobytes(), (r, i)
