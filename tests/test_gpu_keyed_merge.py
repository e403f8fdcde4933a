"""The device merge under every sort order (xgm_merge_mset_device_slab) against tests/merge_model.merge_ref and the
library's host merge (xgm_merge_msets).

Xapiand merges the shards of every request with a `sort` under Multi_MultiValueKeyMaker's comparator
(Matcher::merge_mset with the request's sorter), so a multi-GPU answer to a value-sorted query needs the sort keys
in the result slab and a merge that compares them.  Here the merge runs
  * on built inputs: 1 to 64 parts, first + maxitems up to the largest the kernel's shared memory allows (past the
    48 KiB opt-in), stride = first + maxitems and more, first 0, 1, 7 and beyond the total; each query ordered by
    one of the four sort settings, forward or reverse, over keys that are all equal, a few shared values, one apart,
    random, or the missing-value keys 0 and 2**64 - 1, crossed with the weight patterns of the relevance tests (tie
    masses, pairs of parts, one-ulp neighbours); lost and pending parts and order bytes the kernel cannot know;
  * with NULL orders, where it must equal xgm_merge_topk_device_slab byte for byte;
  * on real slabs of 2, 3 and 8 shards of the synthetic corpus, every query merged under its own order, first and
    maxitems, against the oracle's shards."""
import random

import numpy as np
import pytest

from tests.merge_model import SORT_REL, SORT_REL_VAL, SORT_VAL, SORT_VAL_REL, Part, merge_ref
from tests.test_gpu_shard_merge import (K, LOST_COUNT, SENT_D, SENT_W, bits, build_inputs, global_stats,
                                        lacking_terms, o_query, query_mix, run_shard, shards, spec)
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

SMEM_LIMIT = 200 * 1024  # xgm_merge_mset_device_slab: nparts * (first + maxitems) * 20 bytes at most
SENT_K = 0x5A5A5A5A5A5A5A5A
U64 = (1 << 64) - 1
ORDERS = [(s, r) for s in (SORT_REL, SORT_VAL_REL, SORT_VAL, SORT_REL_VAL) for r in (False, True)]


def _torch():
    import torch
    return torch


def order_byte(sort_by, reverse):
    return sort_by | (4 if reverse else 0)


# ------------------------------------------------------------------------------------------------------------
# the comparator as a lexicographic sort, and the slabs
# ------------------------------------------------------------------------------------------------------------

def sort_columns(w, d, k, sort_by, reverse):
    """uint64 columns whose ascending lexicographic order is the merge order (weights are >= 0 here, so their bit
    patterns order them; weight descending = complemented bits)."""
    wdesc = ~w.astype(np.float64).view(np.uint64)
    kk = np.where(reverse, ~k, k)
    d = d.astype(np.uint64)
    zero = np.zeros_like(d)
    rel = sort_by == SORT_REL
    c1 = np.where(rel | (sort_by == SORT_REL_VAL), wdesc, kk)
    c2 = np.where(rel | (sort_by == SORT_VAL), d, np.where(sort_by == SORT_VAL_REL, wdesc, kk))
    c3 = np.where(rel | (sort_by == SORT_VAL), zero, d)
    return c1, c2, c3


def build_keyed(nparts, nq, m, stride, seed, first=None, relevance=False):
    """build_inputs' weights, docids and records (relevance patterns q % 4, lost and pending parts), with keys of
    pattern (q // 32) % 6, order ORDERS[(q // 4) % 8] and every (part, query) sorted under its query's order.
    With `first`, every third query keeps at most first // nparts records per part, so its total is <= first;
    with `relevance`, every query is ordered by relevance."""
    w, d, info, lost_q = build_inputs(nparts, nq, m, stride, seed)
    W, D, INFO = w.cpu().numpy(), d.cpu().numpy().view(np.uint32), info.cpu().numpy()
    n = INFO[..., 0].astype(np.int64)
    if first is not None:
        few = (np.arange(nq) % 3) == 2
        n[:, few] = np.minimum(n[:, few], first // nparts)
        INFO[..., 0] = n
    rng = np.random.default_rng(seed)
    shape = (nparts, nq, stride)
    # keys all equal, a few shared values, one apart, random, the missing-value keys 0 and 2**64 - 1
    few_vals = np.array([3, 1 << 63, (1 << 63) - 1, 1 << 40], np.uint64)
    pats = [np.full(shape, 1 << 33, np.uint64),
            few_vals[rng.integers(0, len(few_vals), shape)],
            np.uint64(1 << 62) + rng.integers(0, 3, shape).astype(np.uint64),
            rng.integers(0, U64, shape, dtype=np.uint64, endpoint=True),
            np.where(rng.random(shape) < 0.5, np.uint64(0), rng.integers(1, 5, shape).astype(np.uint64)),
            np.where(rng.random(shape) < 0.5, np.uint64(U64), np.uint64(U64 - 2) + rng.integers(0, 2, shape).astype(np.uint64))]
    q = np.arange(nq)
    kpat = (q // 32) % 6
    Kk = np.zeros(shape, np.uint64)
    for p_, arr in enumerate(pats):
        Kk[:, kpat == p_] = arr[:, kpat == p_]
    sort_by = np.array([0 if relevance else ORDERS[(i // 4) % 8][0] for i in range(nq)])
    reverse = np.array([False if relevance else ORDERS[(i // 4) % 8][1] for i in range(nq)])
    sb = np.broadcast_to(sort_by.reshape(1, nq, 1), shape)
    rv = np.broadcast_to(reverse.reshape(1, nq, 1), shape)
    c1, c2, c3 = sort_columns(np.nan_to_num(W), D, Kk, sb, rv)
    invalid = np.arange(stride).reshape(1, 1, stride) >= n[..., None]
    grp = np.broadcast_to(np.arange(nparts * nq).reshape(nparts, nq, 1), shape)
    idx = np.lexsort((c3.ravel(), c2.ravel(), c1.ravel(), invalid.ravel(), grp.ravel())).reshape(shape)
    idx = idx - (grp * stride)
    W = np.take_along_axis(W, idx, -1)
    D = np.take_along_axis(D, idx, -1)
    Kk = np.take_along_axis(Kk, idx, -1)
    W[invalid] = np.nan
    D[invalid] = 0xFFFFFFFF
    orders = (sort_by | np.where(reverse, 4, 0)).astype(np.uint8)
    return W, D, Kk, INFO, n, orders, lost_q


def slab4_layout(nq, stride):
    """weights | docids | records | keys, padded beyond the minimum (8-byte aligned)."""
    off_d = nq * stride * 8 + 24
    off_c = (off_d + nq * stride * 4 + 7) // 8 * 8 + 40
    off_k = off_c + nq * 32 + 56
    return off_k + nq * stride * 8 + 16, off_d, off_c, off_k


def to_slabs4(W, D, Kk, INFO, nq, stride):
    torch = _torch()
    nbytes, off_d, off_c, off_k = slab4_layout(nq, stride)
    raw = np.full((W.shape[0], nbytes), 0xAB, np.uint8)
    for p in range(W.shape[0]):
        raw[p, :nq * stride * 8] = W[p].reshape(-1).view(np.uint8)
        raw[p, off_d:off_d + nq * stride * 4] = D[p].reshape(-1).view(np.uint8)
        raw[p, off_c:off_c + nq * 32] = np.ascontiguousarray(INFO[p]).reshape(-1).view(np.uint8)
        raw[p, off_k:off_k + nq * stride * 8] = Kk[p].reshape(-1).view(np.uint8)
    return torch.from_numpy(raw.reshape(-1)).cuda(), (nbytes, off_d, off_c, off_k)


def merge_keyed(G, layout, orders, nparts, nq, stride, first, maxitems):
    """xgm_merge_mset_device_slab into sentinel-filled outputs: (counts, docids, weights, keys) on the host."""
    torch = _torch()
    nbytes, off_d, off_c, off_k = layout
    ow = torch.full((nq * maxitems,), SENT_W, dtype=torch.float64, device="cuda")
    od = torch.full((nq * maxitems,), SENT_D, dtype=torch.int32, device="cuda")
    ok = torch.full((nq * maxitems,), SENT_K, dtype=torch.int64, device="cuda")
    on = torch.full((nq,), 0x55555555, dtype=torch.int32, device="cuda")
    og = None if orders is None else torch.from_numpy(np.ascontiguousarray(orders, np.uint8)).cuda()
    torch.cuda.synchronize()
    st = xgm.lib().xgm_merge_mset_device_slab(G.data_ptr(), nbytes, off_d, off_c, off_k,
                                              None if og is None else og.data_ptr(), nparts, nq, stride, first,
                                              maxitems, ow.data_ptr(), od.data_ptr(), ok.data_ptr(), on.data_ptr(),
                                              None)
    assert st == 0, xgm.lib().xgm_last_error()
    torch.cuda.synchronize()
    return (on.cpu().numpy().view(np.uint32), od.cpu().numpy().view(np.uint32).reshape(nq, maxitems),
            ow.cpu().numpy().reshape(nq, maxitems), ok.cpu().numpy().view(np.uint64).reshape(nq, maxitems))


def expected(W, D, Kk, n, orders, void, first, maxitems):
    """Every query's merged ranks [first, first + maxitems) as sentinel-filled arrays, by one lexicographic sort of
    all records each part gives (min(n, first + maxitems))."""
    nparts, nq, stride = W.shape
    m = first + maxitems
    i = np.arange(stride).reshape(1, 1, stride)
    take = i < np.minimum(n, m)[..., None]
    take &= ~void.reshape(1, nq, 1)
    p, q, _ = np.nonzero(take)
    w, d, k = W[take], (D[take].astype(np.int64) - 1) * nparts + p + 1, Kk[take]
    sort_by, reverse = orders[q] & 3, (orders[q] >> 2) & 1 == 1
    c1, c2, c3 = sort_columns(w, d.astype(np.uint64), k, sort_by, reverse)
    o = np.lexsort((c3, c2, c1, q))
    q, w, d, k, sort_by = q[o], w[o], d[o], k[o], sort_by[o]
    start = np.searchsorted(q, np.arange(nq))
    rank = np.arange(len(q)) - start[q]
    total = np.bincount(q, minlength=nq)
    cnt = np.clip(total - first, 0, maxitems).astype(np.uint32)
    cnt[void] = LOST_COUNT
    ew = np.full((nq, maxitems), SENT_W)
    ed = np.full((nq, maxitems), SENT_D, np.uint32)
    ek = np.full((nq, maxitems), SENT_K, np.uint64)
    sel = (rank >= first) & (rank < m)
    ew[q[sel], rank[sel] - first] = w[sel]
    ed[q[sel], rank[sel] - first] = d[sel]
    keyed = sel & (sort_by != SORT_REL)
    ek[q[keyed], rank[keyed] - first] = k[keyed]
    return cnt, ed, ew, ek


def check_against_models(W, D, Kk, n, orders, qs, first, maxitems, got, ctx):
    """merge_ref and xgm_merge_msets on the queries qs, over the records each part gives."""
    on, od, ow, ok = got
    nparts = W.shape[0]
    m = first + maxitems
    for qi in qs:
        sort_by, reverse = int(orders[qi]) & 3, bool(orders[qi] & 4)
        cnt = [int(min(n[p, qi], m)) for p in range(nparts)]
        parts = [Part(D[p, qi, :c].tolist(), W[p, qi, :c].tolist(), Kk[p, qi, :c].tolist(), max_possible=1.0)
                 for p, c in enumerate(cnt)]
        ref = merge_ref(parts, first, maxitems, sort_by, reverse)
        c = int(on[qi])
        at = f"{ctx} q{qi} order {sort_by}{'r' if reverse else ''}"
        assert c == len(ref.docids), f"{at}: count {c} vs {len(ref.docids)}"
        assert od[qi, :c].tolist() == ref.docids, f"{at}: docids"
        assert [bits(x) for x in ow[qi, :c]] == [bits(x) for x in ref.weights], f"{at}: weights"
        if sort_by != SORT_REL:
            assert ok[qi, :c].tolist() == ref.keys, f"{at}: keys"
        msets = [xgm.MSet(xgm.unshard(D[p, qi, :cnt[p]], p, nparts), W[p, qi, :cnt[p]].copy(), Kk[p, qi, :cnt[p]].copy(),
                          0, 0, 0, 0, 1.0, 0.0, 0.0, 0, 0) for p in range(nparts)]
        host = xgm.merge_msets(msets, first, maxitems, sort_by, reverse)
        assert host.docids.tolist() == ref.docids and host.weights.tobytes() == ow[qi, :c].tobytes(), f"{at}: host merge"
        if sort_by != SORT_REL:
            assert host.sort_keys.tolist() == ref.keys, f"{at}: host merge keys"


# ------------------------------------------------------------------------------------------------------------
# 1. built inputs
# ------------------------------------------------------------------------------------------------------------

NPARTS = [1, 2, 3, 5, 8, 16, 33, 64]


def mmax(nparts):
    return SMEM_LIMIT // (20 * nparts)


def m_values(nparts):
    return sorted({m for m in (8, 31, 128) if m <= mmax(nparts)} | {mmax(nparts)})


CELLS = [(p, m, s) for p in NPARTS for m in m_values(p) for s in ("m", "m+37")]


@pytest.mark.parametrize("nparts,m,stride_kind", CELLS)
def test_keyed_merge_on_built_inputs(nparts, m, stride_kind):
    stride = m if stride_kind == "m" else m + 37
    nq = max(256, min(2048, (1 << 18) // (nparts * stride)))
    nq -= nq % 256
    if m == mmax(nparts) and nparts > 1:
        assert nparts * m * 20 > 48 * 1024, "meant to cross the 48 KiB shared-memory opt-in"
    firsts = sorted({0, 1, 7, m - 1} & set(range(m)))
    for first in firsts:
        maxitems = m - first
        W, D, Kk, INFO, n, orders, lost_q = build_keyed(nparts, nq, m, stride, seed=nparts * 7919 + m * 13 + stride + first,
                                                        first=first if first == m - 1 else None)
        bad = np.arange(7, nq, 64)  # order bytes naming no order: one per block of 64 queries
        orders[bad] = np.array([8, 0x10, 0xFF, 0x80, 0x0B], np.uint8)[np.arange(len(bad)) % 5]
        void = np.zeros(nq, bool)
        void[lost_q] = True
        void[bad] = True
        G, layout = to_slabs4(W, D, Kk, INFO, nq, stride)
        got = merge_keyed(G, layout, orders, nparts, nq, stride, first, maxitems)
        want = expected(W, D, Kk, n, orders, void, first, maxitems)
        ctx = f"{nparts} parts first={first} maxitems={maxitems} stride={stride}"
        for name_, g, e in zip(("counts", "docids", "weights", "keys"), got, want):
            bad_rows = np.nonzero((g.view(np.uint8).reshape(nq, -1) != e.view(np.uint8).reshape(nq, -1)).any(1))[0]
            assert len(bad_rows) == 0, f"{ctx}: {name_} differ on queries {bad_rows[:8].tolist()} " \
                                       f"(orders {orders[bad_rows[:8]].tolist()})"
        assert (got[0][void] == LOST_COUNT).all() and (got[0][~void] != LOST_COUNT).all(), ctx
        if first == m - 1:
            assert ((got[0] == 0) & ~void).any(), f"{ctx}: no query whose total is within first"
        keep = np.nonzero(~void)[0]
        sample = [q for q in keep[:256] if q % 3 != 1][:32]  # every order, weight and key pattern within 256 queries
        check_against_models(W, D, Kk, n, orders, sample, first, maxitems, got, ctx)


def test_null_orders_equal_the_relevance_entry_point():
    """NULL orders, first = 0: the same records, counts and sentinels as xgm_merge_topk_device_slab, and out_keys
    untouched.  The parts are in relevance order: parts in another order put records on the same rank."""
    torch = _torch()
    for nparts, k, stride in ((1, 31, 31), (3, 100, 137), (8, 128, 128), (64, 40, 77)):
        nq = 512
        W, D, Kk, INFO, n, orders, lost_q = build_keyed(nparts, nq, k, stride, seed=nparts + k, relevance=True)
        G, layout = to_slabs4(W, D, Kk, INFO, nq, stride)
        on, od, ow, ok = merge_keyed(G, layout, None, nparts, nq, stride, 0, k)
        nbytes, off_d, off_c, _ = layout
        rw = torch.full((nq * k,), SENT_W, dtype=torch.float64, device="cuda")
        rd = torch.full((nq * k,), SENT_D, dtype=torch.int32, device="cuda")
        rn = torch.full((nq,), 0x55555555, dtype=torch.int32, device="cuda")
        st = xgm.lib().xgm_merge_topk_device_slab(G.data_ptr(), nbytes, off_d, off_c, nparts, nq, stride, k,
                                                  rw.data_ptr(), rd.data_ptr(), rn.data_ptr(), None)
        assert st == 0
        torch.cuda.synchronize()
        assert on.tobytes() == rn.cpu().numpy().tobytes()
        assert od.tobytes() == rd.cpu().numpy().tobytes()
        assert ow.tobytes() == rw.cpu().numpy().tobytes()
        assert (ok == SENT_K).all()
        assert (on[lost_q] == LOST_COUNT).all()


def test_keyed_merge_rejects_bad_arguments():
    torch = _torch()
    L = xgm.lib()
    nq, stride = 4, 8
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    ords = torch.zeros(nq, dtype=torch.uint8, device="cuda")
    p, o, r = buf.data_ptr(), out.data_ptr(), ords.data_ptr()
    nbytes, off_d, off_c, off_k = slab4_layout(nq, stride)

    def call(nbytes=nbytes, off_d=off_d, off_c=off_c, off_k=off_k, nparts=2, nq=nq, stride=stride, first=0,
             maxitems=stride, g=p, ow=o, od=o, ok=o, on=o, orders=r):
        return L.xgm_merge_mset_device_slab(g, nbytes, off_d, off_c, off_k, orders, nparts, nq, stride, first,
                                            maxitems, ow, od, ok, on, None)

    assert call() == xgm.OK and call(orders=None) == xgm.OK and call(first=3, maxitems=5) == xgm.OK
    torch.cuda.synchronize()
    for kw in (dict(g=None), dict(ow=None), dict(od=None), dict(ok=None), dict(on=None)):
        assert call(**kw) == xgm.E_INVALID, kw  # null pointers
    assert call(maxitems=0) == xgm.E_INVALID
    assert call(first=1, maxitems=stride) == xgm.E_INVALID  # first + maxitems > stride
    assert call(first=0xFFFFFFFF, maxitems=2) == xgm.E_INVALID  # ... without wrapping around
    for kw in (dict(nbytes=nbytes + 4), dict(off_d=off_d + 4), dict(off_c=off_c + 4), dict(off_k=off_k + 4)):
        assert call(**kw) == xgm.E_INVALID, kw  # misaligned
    assert call(off_d=nq * stride * 8 - 8) == xgm.E_INVALID  # docids overlap weights
    assert call(off_c=off_d + nq * stride * 4 - 8) == xgm.E_INVALID  # records overlap docids
    assert call(off_k=off_c + nq * 32 - 8) == xgm.E_INVALID  # keys overlap records
    assert call(nbytes=off_k + nq * stride * 8 - 8) == xgm.E_INVALID  # no room for the keys
    assert call(nq=nq + 1) == xgm.E_INVALID  # too small for nq * stride
    assert call(nparts=65, stride=1, maxitems=1) == xgm.E_INVALID  # more than 64 parts
    big = mmax(2) + 1  # 2 * big * 20 bytes is over the limit
    nb2, od2, oc2, ok2 = slab4_layout(nq, big)
    assert call(nbytes=nb2, off_d=od2, off_c=oc2, off_k=ok2, stride=big, maxitems=big) == xgm.E_INVALID
    assert call(nbytes=nb2, off_d=od2, off_c=oc2, off_k=ok2, stride=big, first=1, maxitems=big - 1) == xgm.E_INVALID
    assert call(nbytes=nb2, off_d=od2, off_c=oc2, off_k=ok2, stride=big, maxitems=big - 1) == xgm.OK  # the limit itself
    assert call(nparts=0) == xgm.E_INVALID and call(nq=0) == xgm.E_INVALID
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------
# 2. real shards
# ------------------------------------------------------------------------------------------------------------

def sorted_mix(rng):
    """Value-sorted queries beyond query_mix's: every order in both directions on AND and OR bases, first > 0,
    the maximum value of a multi-valued slot, and factor-0 tie masses under value orders."""
    out = []
    for i in range(24):
        sort_by = [SORT_VAL, SORT_VAL_REL, SORT_REL_VAL][i % 3]
        op = xgm.OP_OR if i % 4 == 3 else xgm.OP_AND
        out.append((spec(op, rng.sample(range(400), 2 + (op == xgm.OP_OR)), sort_by=sort_by, sort_reverse=bool(i // 3 % 2),
                         sort_use_max=i >= 12, first=[0, 3, 17][i % 3], maxitems=[10, 40][i % 2]), "sort"))
    for i, sort_by in enumerate((SORT_VAL, SORT_VAL_REL, SORT_REL_VAL, SORT_REL_VAL)):
        out.append((spec(xgm.OP_AND, [0, 1 + i], factors=[0.0, 0.0], sort_by=sort_by, sort_reverse=bool(i % 2),
                         first=[0, 5][i % 2], maxitems=30), "zero_sorted"))
    return out


def merge_real(n, tagged):
    xs, os_ = shards(n)
    specs = [sp for sp, _ in tagged]
    tags = [t for _, t in tagged]
    nq = len(specs)
    coll, tlen, gtf = global_stats(xs, os_, specs)
    results, slabs, layout = [], [], None
    for s in range(n):
        res, slab, lay = run_shard(xs[s], specs, coll, tlen, gtf, via_batch=True)
        srch = xgm.Searcher(xs[s], max_batch=nq, max_topk=K)
        off_k = srch.device_slab_keys()
        srch.close()
        nbytes, off_d, off_c = lay
        assert off_k % 256 == 0 and off_k >= off_c + nq * 32 and off_k + nq * K * 8 <= nbytes
        assert layout is None or layout == (*lay, off_k)
        layout = (*lay, off_k)
        keys = slab[off_k:off_k + nq * K * 8].cpu().numpy().view(np.uint64).reshape(nq, K)
        for i, m in enumerate(res):  # the slab's keys are what xgm_search_wait returned
            if specs[i]["sort_by"] != SORT_REL and m.status == 0:
                assert keys[i, :m.size()].tolist() == m.sort_keys.tolist(), f"shard {s} q{i}: slab keys"
        results.append(res)
        slabs.append(slab)
    torch = _torch()
    G = torch.cat(slabs)
    orders = torch.tensor([order_byte(sp["sort_by"], sp["sort_reverse"]) for sp in specs], dtype=torch.uint8,
                          device="cuda")
    orefs = [[None] * nq for _ in range(n)]
    for i, sp in enumerate(specs):
        if tags[i] == "declined":
            continue
        nt, nm = len(sp["terms"]), len(sp["maybe_terms"])
        ost = (coll, tlen, gtf[i][:nt], gtf[i][len(gtf[i]) - nm:] if nm else None)
        for s in range(n):
            orefs[s][i] = os_[s].match(o_query(sp, stats=ost, first=0, maxitems=sp["first"] + sp["maxitems"]))
    checked = keyed = 0
    for first, maxitems in sorted({(sp["first"], sp["maxitems"]) for sp in specs}):
        counts, docids, weights, keys = xgm.merge_device_slabs(G, *layout, orders, n, nq, K, first, maxitems)
        on = counts.cpu().numpy().view(np.uint32)
        od = docids.cpu().numpy().view(np.uint32)
        ow = weights.cpu().numpy()
        ok = keys.cpu().numpy().view(np.uint64)
        for i, sp in enumerate(specs):
            if (sp["first"], sp["maxitems"]) != (first, maxitems):
                continue
            ctx = f"{n} shards q{i} {tags[i]} {sp}"
            if tags[i] == "declined":
                assert on[i] == 0, ctx
                continue
            for s in range(n):
                assert results[s][i].status == 0, ctx
            ref = merge_ref([Part.of_oracle(orefs[s][i]) for s in range(n)], first, maxitems, sp["sort_by"],
                            sp["sort_reverse"])
            c = int(on[i])
            assert c == len(ref.docids), f"{ctx}: count {c} vs {len(ref.docids)}"
            assert od[i, :c].tolist() == ref.docids, f"{ctx}: docids"
            assert [bits(x) for x in ow[i, :c]] == [bits(x) for x in ref.weights], f"{ctx}: weights"
            parts = [results[s][i] for s in range(n)]
            for s, m in enumerate(parts):
                m.docids = xgm.unshard(m.docids, s, n)
            host = xgm.merge_msets(parts, first, maxitems, sp["sort_by"], sp["sort_reverse"])
            for s, m in enumerate(parts):  # back to shard-local docids for the next (first, maxitems)
                m.docids = (m.docids - s - 1) // n + 1
            assert host.docids.tolist() == ref.docids and host.weights.tobytes() == ow[i, :c].tobytes(), ctx
            if sp["sort_by"] != SORT_REL:
                assert ok[i, :c].tolist() == ref.keys, f"{ctx}: keys"
                assert host.sort_keys.tolist() == ref.keys, f"{ctx}: host merge keys"
                keyed += 1
            assert not od[i, c:].any() and not ow[i, c:].any(), f"{ctx}: written beyond the count"
            checked += 1
    return checked, keyed


@pytest.mark.parametrize("n", [2, 3, 8])
def test_real_shards_merge_under_each_querys_order(n):
    rng = random.Random(900 + n)
    tagged = query_mix(n, random.Random(500 + n), lacking_terms(shards(n)[1])) + sorted_mix(rng)
    checked, keyed = merge_real(n, tagged)
    assert checked == len(tagged) - 1 and keyed >= 36  # all but the declined query
