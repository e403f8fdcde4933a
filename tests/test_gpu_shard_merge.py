"""The multi-shard merge against tests/merge_model.merge_ref (Matcher::merge_mset + merge_stats restated).

Every multi-GPU answer passes through xgm_merge_kernel: the per-shard top-k records of an all-gather, laid out
[part][query][rank], unsharded (backends/multi.h:66-70) and merged under (weight desc, docid asc).  Here it runs
  * on built inputs: 1 to 64 parts, k from 1 to the largest the kernel's shared memory allows (past the 48 KiB
    opt-in), stride > k, parts holding 0, < k, k and > k records, tie masses across all parts, ties in pairs of
    parts, weights one ulp apart; through both entry points (three arrays, whole result slabs);
  * on sharded search: 2, 3 and 8 shards of a corpus whose size none of them divides, global statistics passed
    per query and through QueryBatch.set_global_stats, every matching route, term group, range filter, value sort
    and factor-0 tie mass, and rare terms absent from some shards.  Each shard is answered by the oracle with the
    same statistics and the shards are merged by merge_ref; the library's host merge (xgm_merge_msets) is checked
    the same way for every sort order and first > 0;
  * with one shard that lost a query (its overflow pool could not take a tie mass): the merged count of that
    query is UINT32_MAX and the rest of the batch is unchanged."""
import math
import random
import struct

import numpy as np
import pytest

from oracle import oracle as O
from tests.merge_model import SORT_REL, Part, merge_ref, rel_top
from tests.test_gpu_work_split import bitmap_ands, or_pairs, probes
from tests.util import assert_matches_oracle
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

SMEM_LIMIT = 200 * 1024  # xgm_merge_topk_device*: nparts * k * 12 bytes of shared memory at most
RES_LOST, RES_APPROX, RES_PENDING, RES_SKIPPED, RES_SECOND_PASS = 1, 2, 4, 8, 16  # XgmDevResult.flags
LOST_COUNT = 0xFFFFFFFF
SENT_W, SENT_D = -7.0, 0x7EEEEEEE  # what the merge must not overwrite


def bits(x):
    return struct.pack("<d", float(x))


def _torch():
    import torch
    return torch


def merge_arrays(W, D, C, nparts, nq, stride, k):
    """xgm_merge_topk_device over three gathered arrays; returns (counts u32[nq], docids u32[nq,k], weights)."""
    torch = _torch()
    ow = torch.full((nq * k,), SENT_W, dtype=torch.float64, device="cuda")
    od = torch.full((nq * k,), SENT_D, dtype=torch.int32, device="cuda")
    on = torch.full((nq,), 0x55555555, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = xgm.lib().xgm_merge_topk_device(W.data_ptr(), D.data_ptr(), C.data_ptr(), nparts, nq, stride, k,
                                         ow.data_ptr(), od.data_ptr(), on.data_ptr(), None)
    assert st == 0, xgm.lib().xgm_last_error()
    torch.cuda.synchronize()
    return (on.cpu().numpy().view(np.uint32), od.cpu().numpy().view(np.uint32).reshape(nq, k),
            ow.cpu().numpy().reshape(nq, k))


def merge_slabs(G, slab_bytes, off_d, off_c, nparts, nq, stride, k):
    """xgm_merge_topk_device_slab over nparts slabs of slab_bytes each."""
    torch = _torch()
    ow = torch.full((nq * k,), SENT_W, dtype=torch.float64, device="cuda")
    od = torch.full((nq * k,), SENT_D, dtype=torch.int32, device="cuda")
    on = torch.full((nq,), 0x55555555, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = xgm.lib().xgm_merge_topk_device_slab(G.data_ptr(), slab_bytes, off_d, off_c, nparts, nq, stride, k,
                                              ow.data_ptr(), od.data_ptr(), on.data_ptr(), None)
    assert st == 0, xgm.lib().xgm_last_error()
    torch.cuda.synchronize()
    return (on.cpu().numpy().view(np.uint32), od.cpu().numpy().view(np.uint32).reshape(nq, k),
            ow.cpu().numpy().reshape(nq, k))


def merge_both(slabs, slab_bytes, off_d, off_c, nq, stride, k, rows=None):
    """Both entry points over the same per-part slabs (uint8 tensors): the three-array layout is cut out of the
    slabs.  The two must agree byte for byte, sentinels included, on the queries `rows` (default all): the merge
    is defined for relevance-ordered parts only, and parts in value order put records on the same rank."""
    torch = _torch()
    n = len(slabs)
    W = torch.cat([s[:nq * stride * 8].view(torch.float64) for s in slabs])
    D = torch.cat([s[off_d:off_d + nq * stride * 4].view(torch.int32) for s in slabs])
    C = torch.cat([s[off_c:off_c + nq * 32].view(torch.int32) for s in slabs])
    a = merge_arrays(W, D, C, n, nq, stride, k)
    b = merge_slabs(torch.cat(slabs), slab_bytes, off_d, off_c, n, nq, stride, k)
    rows = slice(None) if rows is None else rows
    assert np.array_equal(a[0][rows], b[0][rows]) and np.array_equal(a[1][rows], b[1][rows])
    assert a[2][rows].tobytes() == b[2][rows].tobytes()
    return a


def check_row(on, od, ow, qi, docids, weights, ctx):
    c = int(on[qi])
    assert c == len(docids), f"{ctx}: count {c} vs {len(docids)}"
    assert list(od[qi, :c]) == list(docids), f"{ctx}: docids\n got {list(od[qi, :c])[:12]}\n ref {list(docids)[:12]}"
    assert ow[qi, :c].tobytes() == np.asarray(weights, np.float64).tobytes(), f"{ctx}: weights"
    assert (od[qi, c:] == SENT_D).all() and (ow[qi, c:] == SENT_W).all(), f"{ctx}: written beyond the count"


# ------------------------------------------------------------------------------------------------------------
# 1. the merge kernel on built inputs
# ------------------------------------------------------------------------------------------------------------

NPARTS = [1, 2, 3, 5, 7, 8, 16, 33, 64]


def kmax(nparts):
    return SMEM_LIMIT // (12 * nparts)


def k_values(nparts):
    return sorted({k for k in (1, 2, 31, 128) if k <= kmax(nparts)} | {kmax(nparts)})


CELLS = [(p, k, s) for p in NPARTS for k in k_values(p) for s in ("k", "k+37")]
W_TIE, W_PAIRS, W_ULP, W_RANDOM = range(4)


def build_inputs(nparts, nq, k, stride, seed):
    """[part][query][rank] weights / local docids, each (part, query) sorted by (weight desc, docid asc), and the
    32-byte records.  Query q uses weight pattern q % 4 (W_*); every 16th query has one part LOST or PENDING.  Ranks at
    or beyond a part's n hold NaN weights and docid 0xffffffff, which the merge must never read."""
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    shape = (nparts, nq, stride)
    tie = torch.full(shape, 1.0, dtype=torch.float64, device="cuda")
    pairs = torch.randint(1, 5, ((nparts + 1) // 2, nq, stride), generator=g, device="cuda").double()
    pairs = pairs.repeat_interleave(2, dim=0)[:nparts]
    base = torch.tensor(3.0, dtype=torch.float64)
    ulps = [base]
    for direction in (math.inf, -math.inf):
        x = base
        for _ in range(2):
            x = torch.nextafter(x, torch.tensor(direction, dtype=torch.float64))
            ulps.append(x)
    ulps = torch.stack(ulps).cuda()
    # one value per (part, query): parts one ulp apart or equal, every part a tie mass of its own
    ulp = ulps[torch.randint(0, len(ulps), shape[:2], generator=g, device="cuda")].unsqueeze(-1).expand(shape)
    rnd = torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) * 20.0
    pat = (torch.arange(nq, device="cuda") % 4).view(1, nq, 1)
    w = torch.where(pat == W_TIE, tie, torch.where(pat == W_PAIRS, pairs, torch.where(pat == W_ULP, ulp, rnd)))
    # distinct local docids in [1, 2 * stride]: the parts' unsharded docids interleave
    d = torch.rand((nparts, nq, 2 * stride), generator=g, device="cuda").argsort(-1)[..., :stride].to(torch.int32) + 1
    d = d.sort(-1).values
    order = torch.sort(w, dim=-1, descending=True, stable=True).indices
    w, d = w.gather(-1, order), d.gather(-1, order)
    # per-part record count: 0, below k, k, above k (up to stride)
    kind = torch.randint(0, 4, (nparts, nq), generator=g, device="cuda")
    below = torch.randint(1, max(k, 2), (nparts, nq), generator=g, device="cuda").clamp(max=max(k - 1, 0))
    above = torch.randint(k, stride + 1, (nparts, nq), generator=g, device="cuda").clamp(min=min(k + 1, stride))
    n = torch.where(kind == 0, 0, torch.where(kind == 1, below, torch.where(kind == 2, k, above)))
    invalid = torch.arange(stride, device="cuda").view(1, 1, stride) >= n.unsqueeze(-1)
    w = w.masked_fill(invalid, float("nan"))
    d = d.masked_fill(invalid, -1)
    info = torch.zeros((nparts, nq, 8), dtype=torch.int32, device="cuda")
    info[..., 0] = n.to(torch.int32)
    benign = torch.tensor([0, RES_APPROX, RES_SKIPPED, RES_SECOND_PASS, RES_APPROX | RES_SKIPPED], device="cuda")
    info[..., 3] = benign[torch.randint(0, len(benign), (nparts, nq), generator=g, device="cuda")].to(torch.int32)
    lost_q = torch.arange(15, nq, 16, device="cuda")
    lost_p = torch.randint(0, nparts, (len(lost_q),), generator=g, device="cuda")
    lost_f = torch.tensor([RES_LOST, RES_PENDING], device="cuda")[torch.arange(len(lost_q), device="cuda") % 2]
    info[lost_p, lost_q, 3] |= lost_f.to(torch.int32)
    return w.contiguous(), d.contiguous(), info.contiguous(), lost_q.cpu().numpy()


def slab_layout(nq, stride):
    """Offsets of the slab entry point, padded beyond the minimum (8-byte aligned)."""
    off_d = nq * stride * 8 + 24
    off_c = (off_d + nq * stride * 4 + 7) // 8 * 8 + 40
    return off_c + nq * 32 + 56, off_d, off_c


def to_slabs(w, d, info, nq, stride):
    torch = _torch()
    nbytes, off_d, off_c = slab_layout(nq, stride)
    slabs = []
    for p in range(w.shape[0]):
        s = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device="cuda")
        s[:nq * stride * 8].view(torch.float64).copy_(w[p].reshape(-1))
        s[off_d:off_d + nq * stride * 4].view(torch.int32).copy_(d[p].reshape(-1))
        s[off_c:off_c + nq * 32].view(torch.int32).copy_(info[p].reshape(-1))
        slabs.append(s)
    return slabs, nbytes, off_d, off_c


@pytest.mark.parametrize("nparts,k,stride_kind", CELLS)
def test_merge_kernel_on_built_inputs(nparts, k, stride_kind):
    stride = k if stride_kind == "k" else k + 37
    nq = max(64, min(4096, (1 << 19) // (nparts * stride)))
    w, d, info, lost_q = build_inputs(nparts, nq, k, stride, seed=nparts * 100003 + k * 7 + stride)
    slabs, nbytes, off_d, off_c = to_slabs(w, d, info, nq, stride)
    on, od, ow = merge_both(slabs, nbytes, off_d, off_c, nq, stride, k)
    W, D = w.cpu().numpy(), d.cpu().numpy().view(np.uint32)
    cnt = info[..., 0].cpu().numpy().astype(np.int64)
    lost = set(lost_q.tolist())
    # the cell really holds what it is meant to test
    if k == kmax(nparts) or nparts * k * 12 > 48 * 1024:
        assert nparts * k * 12 > 48 * 1024, "meant to cross the 48 KiB shared-memory opt-in"
    if k > 1:
        assert ((cnt > 0) & (cnt < k)).any()
    assert (cnt == 0).any() and (cnt == k).any()
    if stride > k:
        assert (cnt > k).any()
    cross_ties = ulp_pairs = 0
    for qi in range(nq):
        ctx = f"{nparts} parts k={k} stride={stride} q{qi} pattern {qi % 4}"
        if qi in lost:
            assert on[qi] == LOST_COUNT, f"{ctx}: a lost part must void the query"
            assert (od[qi] == SENT_D).all() and (ow[qi] == SENT_W).all(), f"{ctx}: records of a lost query"
            continue
        docids, weights = rel_top(D[:, qi], W[:, qi], cnt[:, qi], k)
        check_row(on, od, ow, qi, docids, weights, ctx)
        if nparts > 1 and qi < 256:
            vals = [set(W[p, qi, :min(cnt[p, qi], k)].tolist()) for p in range(nparts)]
            seen = set()
            for v in vals:
                cross_ties += bool(seen & v)
                seen |= v
            if qi % 4 == W_ULP:
                ws = sorted(seen)
                ulp_pairs += any(math.nextafter(a, math.inf) == b for a, b in zip(ws, ws[1:]))
    if nparts > 1:
        assert cross_ties > 0 and ulp_pairs > 0


def test_merge_entry_points_reject_bad_arguments():
    torch = _torch()
    L = xgm.lib()
    nq, stride, k = 4, 8, 8
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p, o = buf.data_ptr(), out.data_ptr()

    def arrays(nparts, nq, stride, k):
        return L.xgm_merge_topk_device(p, p, p, nparts, nq, stride, k, o, o, o, None)

    def slab(slab_bytes, off_d, off_c, nparts, nq, stride, k):
        return L.xgm_merge_topk_device_slab(p, slab_bytes, off_d, off_c, nparts, nq, stride, k, o, o, o, None)

    nbytes, off_d, off_c = slab_layout(nq, stride)
    assert arrays(2, nq, stride, k) == xgm.OK and slab(nbytes, off_d, off_c, 2, nq, stride, k) == xgm.OK
    torch.cuda.synchronize()
    assert arrays(2, nq, stride, stride + 1) == xgm.E_INVALID  # k > stride
    assert slab(nbytes, off_d, off_c, 2, nq, stride, stride + 1) == xgm.E_INVALID
    assert arrays(65, nq, stride, 1) == xgm.E_INVALID  # more than 64 parts
    assert slab(nbytes, off_d, off_c, 65, nq, stride, 1) == xgm.E_INVALID
    big = kmax(2) + 1  # 2 * big * 12 bytes is over the limit
    assert arrays(2, nq, big, big) == xgm.E_INVALID
    nb2, od2, oc2 = slab_layout(nq, big)
    assert slab(nb2, od2, oc2, 2, nq, big, big) == xgm.E_INVALID
    assert arrays(2, nq, kmax(2), kmax(2)) == xgm.OK  # the limit itself is allowed
    torch.cuda.synchronize()
    for bad in ((nbytes + 4, off_d, off_c), (nbytes, off_d + 4, off_c), (nbytes, off_d, off_c + 4)):
        assert slab(*bad, 2, nq, stride, k) == xgm.E_INVALID, bad  # misaligned
    assert slab(nbytes, nq * stride * 8 - 8, off_c, 2, nq, stride, k) == xgm.E_INVALID  # docids overlap weights
    assert slab(nbytes, off_d, off_d + nq * stride * 4 - 8, 2, nq, stride, k) == xgm.E_INVALID
    assert slab(off_c + nq * 32 - 8, off_d, off_c, 2, nq, stride, k) == xgm.E_INVALID  # slab too small
    assert slab(nbytes, off_d, off_c, 2, nq + 1, stride, k) == xgm.E_INVALID  # too small for nq * stride
    assert arrays(0, nq, stride, k) == xgm.E_INVALID and arrays(2, nq, stride, 0) == xgm.E_INVALID


# ------------------------------------------------------------------------------------------------------------
# 2. sharded search on every route
# ------------------------------------------------------------------------------------------------------------

ND, V = 30001, 20000  # divisible by none of 2, 3, 8
K = 128  # searcher max_topk, slab stride and device-merge k


def name(t):
    return f"T{t:06d}"


def spec_of(x):
    """A query of tests/test_gpu_work_split's generators (term ids) as a plain dict."""
    return dict(op=x.op, terms=list(x.terms), first=x.first, maxitems=x.maxitems, check_at_least=x.check_at_least,
                filter_terms=list(x.filter_terms), not_terms=list(x.not_terms), maybe_terms=list(x.maybe_terms),
                sort_by=x.sort_by, sort_reverse=x.sort_reverse, sort_use_max=x.sort_use_max, factors=x.factors,
                filter=x.filter, range_lo=x.range_lo, range_hi=x.range_hi, filter_weighted=x.filter_weighted,
                filter_factor=x.filter_factor)


def spec(op, terms, **kw):
    base = spec_of(xgm.Query(op, list(terms)))
    base.update(kw)
    return base


def all_terms(sp):
    return sp["terms"] + sp["filter_terms"] + sp["not_terms"] + sp["maybe_terms"]


def x_query(sp, stats=None, first=None, maxitems=None):
    kw = dict(sp)
    op, terms = kw.pop("op"), kw.pop("terms")
    for g in ("filter_terms", "not_terms", "maybe_terms"):
        kw[g] = [name(t) for t in kw[g]]
    if first is not None:
        kw.update(first=first, maxitems=maxitems)
    return xgm.Query(op, [name(t) for t in terms], sort_slot=0, filter_slot=0, stats=stats, **kw)


def o_query(sp, stats=None, first=None, maxitems=None):
    kw = dict(sp)
    use_max = kw.pop("sort_use_max")
    if first is not None:
        kw.update(first=first, maxitems=maxitems)
    return O.Query(sort_slot=2 if use_max else 0, stats=stats, **kw)


def lacking_terms(os_):
    """Terms of the corpus that some shard does not hold."""
    return [t for t in range(V) if min(o.termfreq(t) for o in os_) == 0 and max(o.termfreq(t) for o in os_) > 0]


def query_mix(n, rng, lacking):
    """(spec, tag) pairs over every route; the tags say what a query is there for.  `lacking`: terms some shard
    does not hold."""
    out = [(spec_of(x), "and_bitmap") for x, _ in bitmap_ands(rng, 60)]
    for _ in range(25):  # general AND: a term with a membership bitmap and one without
        out.append((spec(xgm.OP_AND, [rng.randrange(0, 300), rng.randrange(3000, 8000)], maxitems=rng.choice([10, 100]),
                         first=rng.choice([0, 0, 2]), check_at_least=rng.choice([0, ND])), "and_general"))
    for _ in range(15):
        out.append((spec(xgm.OP_AND, [rng.randrange(0, 5000)], maxitems=rng.choice([1, 10, 100]),
                         first=rng.choice([0, 5])), "single"))
    out += [(spec_of(x), "or") for x, _ in or_pairs(rng, 40)]
    for _ in range(10):
        out.append((spec(xgm.OP_OR, rng.sample(range(3000), rng.choice([6, 8])), maxitems=rng.choice([10, 100]),
                         check_at_least=ND), "or_wide"))
    for i in range(20):  # FILTER and AND_NOT around OR bases
        pool = rng.sample(range(600), 8)
        out.append((spec(xgm.OP_OR, pool[:rng.choice([2, 3, 4])], filter_terms=pool[5:5 + i % 2],
                         not_terms=pool[6:6 + 1 + (i // 2) % 2], maxitems=rng.choice([10, 50]),
                         check_at_least=rng.choice([0, ND])), "or_groups"))
    out += [(spec_of(x), "probe") for x, _ in probes()]
    for i in range(20):  # value ranges: filter on AND and OR bases, the weighted source on AND bases
        lo = rng.randrange(0, 900000)
        kw = dict(filter=xgm.FILTER_MULTI_RANGE, range_lo=lo, range_hi=lo + rng.choice([20000, 200000]),
                  maxitems=rng.choice([10, 100]), check_at_least=rng.choice([0, ND]))
        if i % 4 == 3:
            out.append((spec(xgm.OP_OR, rng.sample(range(200), 3), **kw), "range_or"))
        else:
            if i % 2:
                kw.update(filter_weighted=True, filter_factor=rng.choice([1.0, 2.5]))
            out.append((spec(xgm.OP_AND, rng.sample(range(200), 2), **kw), "range_and"))
    for i in range(12):  # relevance-then-value and the other value sorts with first > 0
        out.append((spec(xgm.OP_AND, rng.sample(range(300), 2), first=rng.choice([1, 7]), maxitems=20,
                         sort_by=[xgm.SORT_REL_VAL, xgm.SORT_VAL, xgm.SORT_VAL_REL][i % 3], sort_reverse=bool(i % 2),
                         sort_use_max=i >= 6), "sort"))
    # factor-0 tie masses: every match weighs 0, so the merged order is the interleaved docid order
    out.append((spec(xgm.OP_AND, [0], factors=[0.0], maxitems=100), "zero"))
    out.append((spec(xgm.OP_AND, [0, 1], factors=[0.0, 0.0], maxitems=10, first=3), "zero"))
    out.append((spec(xgm.OP_AND, [0, 2, 5], factors=[0.0, 0.0, 0.0], maxitems=100, check_at_least=ND), "zero"))
    for _ in range(20):  # rare terms, absent from some shards
        rare = [rng.choice(lacking), rng.randrange(9000, V)]
        out.append((spec(xgm.OP_OR, rare + [rng.randrange(0, 50)], maxitems=100), "rare"))
        out.append((spec(xgm.OP_OR, rare, maxitems=10), "rare"))
        out.append((spec(xgm.OP_AND, [rng.randrange(0, 20), rare[0]], maxitems=10), "rare"))
    # declined by its shape (AND_MAYBE around an OR base) on every shard alike
    out.append((spec(xgm.OP_OR, [3, 4], maybe_terms=[5], maxitems=10), "declined"))
    return out


_SHARDS = {}


def shards(n):
    if n not in _SHARDS:
        xs = [xgm.Index.synthetic(ND, V, values=True, nshards=n, shard=s) for s in range(n)]
        os_ = [O.Index.synthetic(ND, V, values=True, nshards=n, shard=s) for s in range(n)]
        _SHARDS.clear()  # one corpus at a time on the device
        _SHARDS[n] = (xs, os_)
    return _SHARDS[n]


def global_stats(xs, os_, specs):
    """Phase 1 of the two-phase search: collection size, total length and each term's termfreq summed over the
    shards (the termfreq of a term a shard lacks is 0 there)."""
    infos = [x.info() for x in xs]
    coll, tlen = sum(i.doccount for i in infos), sum(i.total_length for i in infos)
    assert coll == ND and tlen == sum(o.total_length for o in os_)
    gtf = []
    for sp in specs:
        ts = all_terms(sp)
        tf = sum(x.term_freqs([name(t) for t in ts]).astype(np.int64) for x in xs)
        assert list(tf) == [sum(o.termfreq(t) for o in os_) for t in ts]
        gtf.append([int(v) for v in tf])
    return coll, tlen, gtf


def run_shard(ix, specs, coll, tlen, gtf, via_batch):
    """One shard's search of the batch with the global statistics, either per query (stats=) or through
    QueryBatch.set_global_stats, for ranks [0, first + maxitems) as the two-phase scheme asks every shard; returns
    the MSets and a copy of the device result slab."""
    torch = _torch()
    s = xgm.Searcher(ix, max_batch=len(specs), max_topk=K)
    if via_batch:
        batch = xgm.QueryBatch([x_query(sp, first=0, maxitems=sp["first"] + sp["maxitems"]) for sp in specs])
        batch.attach_global_stats()
        m = np.zeros((len(specs), xgm.MAX_TERMS), np.uint32)
        for i, tf in enumerate(gtf):
            m[i, :len(tf)] = tf
        batch.set_global_stats(coll, tlen, m)
    else:
        batch = xgm.QueryBatch([x_query(sp, stats=(coll, tlen, gtf[i]), first=0, maxitems=sp["first"] + sp["maxitems"])
                                for i, sp in enumerate(specs)])
    res = s.search(batch)
    base, nbytes, off_d, off_c, stride = s.device_slab()
    assert stride == K

    class _A:  # the slab as a torch tensor (copied before the searcher goes)
        __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(base), False), "version": 2}
    slab = torch.as_tensor(_A(), device="cuda").clone()
    torch.cuda.synchronize()
    s.close()
    return res, slab, (nbytes, off_d, off_c)


def same_results(a, b, slab_a, slab_b, layout, specs):
    """Two runs of one shard are the same: the slab's records and result prefixes, and every MSet field.  Whether a
    pruned run flags its bounds approximate (and then reports only the guaranteed part of the match count) depends
    on when the running threshold rose during the match, which can differ between two runs of one batch, and so can
    whether MaxScore skipped whole segments: those flags and the counts they license are compared only where neither
    run set them."""
    nbytes, off_d, off_c = layout
    nq = len(specs)
    ra = slab_a[off_c:off_c + nq * 32].cpu().numpy()
    rb = slab_b[off_c:off_c + nq * 32].cpu().numpy()
    ua, ub = ra.view(np.uint32).reshape(nq, 8), rb.view(np.uint32).reshape(nq, 8)
    racy = np.uint32(RES_APPROX | RES_SKIPPED)
    exact_cols = [0, 4, 5, 6, 7]  # n, max_w, max_subqs, pad
    assert np.array_equal(ua[:, exact_cols], ub[:, exact_cols]), "result records differ"
    assert np.array_equal(ua[:, 3] & ~racy, ub[:, 3] & ~racy), "record flags differ"
    plain = ((ua[:, 3] | ub[:, 3]) & racy) == 0
    assert np.array_equal(ua[plain][:, [1, 2]], ub[plain][:, [1, 2]]), "match counts differ"
    wa, wb = slab_a[:nq * K * 8].cpu().numpy(), slab_b[:nq * K * 8].cpu().numpy()
    da, db = slab_a[off_d:off_d + nq * K * 4].cpu().numpy(), slab_b[off_d:off_d + nq * K * 4].cpu().numpy()
    cnt = ra.view(np.uint32).reshape(nq, 8)[:, 0]
    for i in range(nq):
        c = int(min(cnt[i], K))
        assert wa[i * K * 8:(i * K + c) * 8].tobytes() == wb[i * K * 8:(i * K + c) * 8].tobytes(), i
        assert da[i * K * 4:(i * K + c) * 4].tobytes() == db[i * K * 4:(i * K + c) * 4].tobytes(), i
    for i, (x, y) in enumerate(zip(a, b)):
        keyed = specs[i]["sort_by"] != SORT_REL  # a relevance order leaves the keys unset
        approx = (x.flags | y.flags) & xgm.MSET_BOUNDS_APPROX
        lower = (x.flags | y.flags) & xgm.MSET_COUNT_LOWER_BOUND

        def fingerprint(m):
            return (m.status, m.flags | approx | lower, m.docids.tobytes(), m.weights.tobytes(),
                    m.sort_keys.tobytes() if keyed else b"", None if approx else m.matches_lower_bound,
                    None if approx else m.matches_estimated_raw, m.matches_upper_bound, None if lower else m.exact_matches,
                    bits(m.max_possible), bits(m.max_attained), bits(m.percent_scale_factor))
        assert fingerprint(x) == fingerprint(y), f"query {i}"


def check_sharded(n, tagged, env=None, monkeypatch=None, unsharded=None):
    xs, os_ = shards(n)
    specs = [sp for sp, _ in tagged]
    tags = [t for _, t in tagged]
    nq = len(specs)
    coll, tlen, gtf = global_stats(xs, os_, specs)
    per_shard, slabs, layout = [], [], None
    for s in range(n):
        if env:
            for k_, v in env.items():
                monkeypatch.setenv(k_, v)
        res, slab, layout_s = run_shard(xs[s], specs, coll, tlen, gtf, via_batch=False)
        res2, slab2, _ = run_shard(xs[s], specs, coll, tlen, gtf, via_batch=True)
        same_results(res, res2, slab, slab2, layout_s, specs)
        assert layout is None or layout == layout_s
        layout = layout_s
        per_shard.append(res)
        slabs.append(slab)
    # each shard against the oracle's answer for that shard with the same statistics
    orefs = [[None] * nq for _ in range(n)]
    absent = 0
    for i, sp in enumerate(specs):
        nt, nm = len(sp["terms"]), len(sp["maybe_terms"])
        ost = (coll, tlen, gtf[i][:nt], gtf[i][len(gtf[i]) - nm:] if nm else None)
        absent += any(o.termfreq(t) == 0 for o in os_ for t in all_terms(sp))
        for s in range(n):
            m = per_shard[s][i]
            if tags[i] == "declined":
                assert m.status == xgm.E_UNIMPLEMENTED, f"shard {s} q{i}"
                continue
            ref = os_[s].match(o_query(sp, stats=ost, first=0, maxitems=sp["first"] + sp["maxitems"]))
            ctx = f"{n} shards, shard {s} q{i} {tags[i]} {sp}"
            assert_matches_oracle(m, ref, ctx)
            if sp["sort_by"] != SORT_REL:
                assert list(m.sort_keys) == list(ref.sortvals), f"{ctx}: sort keys"
            orefs[s][i] = ref
    # relevance order through the device merge (both entry points) == merge_ref over the oracle's shards
    rel = [i for i, sp in enumerate(specs) if sp["sort_by"] == SORT_REL]
    on, od, ow = merge_both(slabs, *layout, nq, K, K, rows=rel)
    merged_dev = 0
    for i, sp in enumerate(specs):
        if tags[i] == "declined":
            assert on[i] == 0, f"declined q{i}: count {on[i]}"
            continue
        if sp["sort_by"] != SORT_REL:
            continue
        ref = merge_ref([Part.of_oracle(orefs[s][i]) for s in range(n)], 0, K)
        check_row(on, od, ow, i, ref.docids, ref.weights, f"{n} shards device merge q{i} {tags[i]} {sp}")
        merged_dev += 1
    # every sort order and first > 0 through the host merge == merge_ref over the oracle's shards
    for i, sp in enumerate(specs):
        if tags[i] == "declined":
            continue
        parts = [per_shard[s][i] for s in range(n)]
        for s, m in enumerate(parts):
            m.docids = xgm.unshard(m.docids, s, n)
        got = xgm.merge_msets(parts, sp["first"], sp["maxitems"], sp["sort_by"], sp["sort_reverse"])
        ref = merge_ref([Part.of_oracle(orefs[s][i]) for s in range(n)], sp["first"], sp["maxitems"],
                        sp["sort_by"], sp["sort_reverse"])
        ctx = f"{n} shards host merge q{i} {tags[i]} {sp}"
        assert list(got.docids) == ref.docids, ctx
        assert [bits(w) for w in got.weights] == [bits(w) for w in ref.weights], f"{ctx}: weights"
        if sp["sort_by"] != SORT_REL:
            assert list(got.sort_keys) == ref.keys, f"{ctx}: sort keys"
        assert bits(got.max_possible) == bits(ref.max_possible), f"{ctx}: max_possible"
        assert bits(got.max_attained) == bits(ref.max_attained), f"{ctx}: max_attained"
        assert bits(got.percent_scale_factor) == bits(ref.percent_scale_factor), f"{ctx}: percent scale"
        assert got.matches_upper_bound == ref.ub, f"{ctx}: ub"
        if not any(m.flags & xgm.MSET_BOUNDS_APPROX for m in parts):
            assert (got.matches_lower_bound, got.matches_estimated_raw) == (ref.lb, ref.est), f"{ctx}: bounds"
        # against the unsharded corpus where every shard sums the leaves in the global order
        if unsharded is not None and tags[i] in ("and_general", "single", "zero", "rare") \
                and not sp["filter_terms"] and not sp["not_terms"] and not sp["maybe_terms"] and sp["op"] == xgm.OP_AND:
            gorder = O.and_order(gtf[i])
            if all(O.and_order([o.termfreq(t) for t in sp["terms"]]) == gorder for o in os_):
                whole = unsharded.match(o_query(sp))
                assert list(got.docids) == list(whole.docids), f"{ctx}: unsharded docids"
                assert np.asarray(got.weights).tobytes() == whole.weights.tobytes(), f"{ctx}: unsharded weights"
    return merged_dev, absent


@pytest.fixture(scope="module")
def whole():
    return O.Index.synthetic(ND, V, values=True)


@pytest.mark.parametrize("n", [2, 3, 8])
def test_sharded_search_every_route_merges_like_the_oracle(n, whole):
    tagged = query_mix(n, random.Random(500 + n), lacking_terms(shards(n)[1]))
    merged_dev, absent = check_sharded(n, tagged, unsharded=whole)
    assert merged_dev > len(tagged) // 2
    assert absent > 0, "no query has a term some shard lacks"


@pytest.mark.parametrize("knob", [("XGM_OR_TILE", "0"), ("XGM_OR_KERNEL", "1")])
def test_sharded_or_routes_merge_like_the_oracle(knob, monkeypatch):
    """The OR queries of the mix again with the bitmap-union tile off (xgm_or3_kernel) and on the general OR
    kernel, over 3 shards."""
    tagged = [t for t in query_mix(3, random.Random(503), lacking_terms(shards(3)[1])) if t[1] in ("or", "or_wide", "or_groups", "rare", "range_or")]
    check_sharded(3, tagged, env=dict([knob]), monkeypatch=monkeypatch)


def test_lost_shard_voids_only_that_query(monkeypatch):
    """One shard's searcher has an overflow pool smaller than a factor-0 tie mass: that shard reports the query
    lost (XGM_E_UNIMPLEMENTED) and the device merge gives it count UINT32_MAX and no records; every other query of
    the batch merges exactly as with a full-size pool."""
    n = 3
    xs, os_ = shards(n)
    rng = random.Random(77)
    tagged = [(spec(xgm.OP_AND, rng.sample(range(400), 2), maxitems=10), "and") for _ in range(30)]
    tagged += [(spec(xgm.OP_OR, rng.sample(range(400), 3), maxitems=10), "or") for _ in range(10)]
    lost_q = 17
    tagged.insert(lost_q, (spec(xgm.OP_AND, [0], factors=[0.0], maxitems=10), "zero"))
    specs = [sp for sp, _ in tagged]
    coll, tlen, gtf = global_stats(xs, os_, specs)
    assert all(o.termfreq(0) > 1000 for o in os_)  # the tie mass cannot fit a pool of 1000 entries

    def merged(small_pool_shard):
        slabs, status = [], []
        for s in range(n):
            if s == small_pool_shard:
                monkeypatch.setenv("XGM_POOL_ENTRIES", "1000")
            res, slab, layout = run_shard(xs[s], specs, coll, tlen, gtf, via_batch=True)
            monkeypatch.delenv("XGM_POOL_ENTRIES", raising=False)
            slabs.append(slab)
            status.append([m.status for m in res])
        return merge_both(slabs, *layout, len(specs), K, K), status

    (on, od, ow), st = merged(1)
    (on0, od0, ow0), st0 = merged(None)
    assert st[1][lost_q] == xgm.E_UNIMPLEMENTED and st[0][lost_q] == 0 and st[2][lost_q] == 0
    assert all(v == 0 for row in st0 for v in row)
    assert on[lost_q] == LOST_COUNT and (od[lost_q] == SENT_D).all() and (ow[lost_q] == SENT_W).all()
    assert on0[lost_q] == n * 10  # the device merge keeps every record of the shards, up to K
    keep = [i for i in range(len(specs)) if i != lost_q]
    assert np.array_equal(on[keep], on0[keep]) and np.array_equal(od[keep], od0[keep])
    assert ow[keep].tobytes() == ow0[keep].tobytes()
    # the full-pool merge of the tie mass: the 10 smallest docids of the interleaved shards
    sp = specs[lost_q]
    parts = [Part.of_oracle(os_[s].match(o_query(sp, stats=(coll, tlen, gtf[lost_q]), first=0, maxitems=10)))
             for s in range(n)]
    ref = merge_ref(parts, 0, K)
    check_row(on0, od0, ow0, lost_q, ref.docids, ref.weights, "full pool")
