"""The OR kernels' MaxScore bounds against the oracle, on a corpus built so that each bound is met or nearly met by
documents the MSet needs (tests/bound_corpus.py; tests/test_bound_corpus.py pins the witnesses).

A bound that is too small silently drops documents and leaves a plausible MSet, so every query is compared with
the oracle bit for bit, on every OR route, under a matrix of BM25 parameters, factors, wqf and global statistics
in which the leaves' weight order is not their termfreq order:
  tile     relevance-ordered OR of <= 5 bitmap leaves: xgm_or_tile_kernel, then xgm_or3_kernel<1>
  or3      the same queries with XGM_OR_TILE=0: xgm_or3_kernel<0>
  general  the same queries with XGM_OR_KERNEL=1: xgm_or_kernel
  wide     6..16 leaves, leaves without a membership bitmap, FILTER / AND_NOT groups: xgm_or_kernel on its own
Each (route, weighting) cell must also have pruned: most queries carry MSET_BOUNDS_APPROX, and on the or3 and
general cells at least one a skipped work item (MSET_COUNT_LOWER_BOUND)."""
import shutil
import tempfile

import pytest

from oracle import oracle as O
from tests import bound_corpus as B
from tests.util import assert_matches_oracle, bits
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

MAX_TOPK = 128
# (maxitems, first, check_at_least): check_at_least 0 or k + 1, so that the threshold may rise and prune
ARGS = ((1, 0, 0), (10, 0, 11), (10, 3, 0), (100, 0, 0), (100, 3, 104), (1, 3, 5))

WEIGHTINGS = {"default": None}
WEIGHTINGS.update({f"k1={k1} b={b}": (k1, 1.0, b, 0.5) for k1 in (0.0, 0.5, 2.0, 20.0, 100.0) for b in (0.0, 0.3, 1.0)})
WEIGHTINGS.update({"mnl=0": (1.2, 1.0, 0.75, 0.0), "mnl=3": (1.2, 1.0, 0.75, 3.0),
                   "k3=0 wqf": (1.2, 0.0, 0.75, 0.5), "k3=7 wqf": (1.2, 7.0, 0.75, 0.5), "stats": (1.2, 1.0, 0.75, 0.5)})
WIDE_WEIGHTINGS = ("default", "k1=0.0 b=0.0", "k1=2.0 b=1.0", "k1=20.0 b=0.0", "k1=100.0 b=0.3", "mnl=0", "k3=7 wqf",
                   "stats")


@pytest.fixture(scope="module")
def bounds():
    tmp = tempfile.mkdtemp(prefix="xgm_bounds_")
    path, names = B.write_bound_corpus(tmp)
    yield path, {n: i for i, n in enumerate(names)}, xgm.Index.load_flat(path), O.Index.load_flat(path)
    shutil.rmtree(tmp, ignore_errors=True)


_refs = {}


def oracle(orc, o):
    """Oracle MSets are the same on every route: computed once per query."""
    key = repr(o)
    if key not in _refs:
        _refs[key] = orc.match(o)
    return _refs[key]


def specs(cell, ids, orc, wide):
    """(leaf names, factors, wqf, stats, filter names, not names) of one weighting cell."""
    tf = lambda names: [orc.termfreq(ids[n]) for n in names]  # noqa: E731
    if wide:
        sets = [(s, None) for s in B.WIDE_SETS] + [(B.G_NAMES, [3.25 if k % 3 == 0 else 1e-3 for k in range(16)])]
        out = [(s, f, None, None, (), ()) for s, f in sets]
        out += [(B.W1_SETS[0], None, None, None, ("z_bool",), ()), (B.W3_SET, B.W3_FACTORS[0], None, None, (), ("g14",)),
                (B.W2_SET, B.tie_factors(tf(B.W2_SET)), None, None, ("z_bool",), ("g13",))]
    else:
        out = [(s, None, None, None, (), ()) for s in B.W1_SETS]
        out.append((B.W2_SET, B.tie_factors(tf(B.W2_SET)), None, None, (), ()))
        out += [(B.W3_SET, f, None, None, (), ()) for f in B.W3_FACTORS]
        out += [(s, B.w4_factors(s), None, None, (), ()) for s in B.W4_SETS]
    if cell.endswith("wqf"):
        out = [(s, f, [(1, 3, 7)[j % 3] for j in range(len(s))], None, a, n) for s, f, _, _, a, n in out]
        out.append((B.W3_SET, None, B.W3_WQF, None, (), ()))
    if cell == "stats":
        out = [(s, f, None, B.reversed_stats(tf(s), orc.total_length), a, n) for s, f, _, _, a, n in out if not a and not n]
    return out


def cell_pairs(cell, ids, orc, wide=False):
    bm25 = WEIGHTINGS[cell]
    out = []
    for names, fac, wqf, stats, filt, nots in specs(cell, ids, orc, wide):
        for k, first, cal in ARGS:
            kw = dict(first=first, maxitems=k, check_at_least=cal, factors=fac, wqf=wqf, bm25=bm25, stats=stats)
            x = xgm.Query(xgm.OP_OR, list(names), filter_terms=list(filt), not_terms=list(nots), **kw)
            o = O.Query(op=O.OP_OR, terms=[ids[n] for n in names], filter_terms=[ids[n] for n in filt],
                        not_terms=[ids[n] for n in nots], **kw)
            out.append((x, o))
    return out


def run_cells(searcher, orc, cells, route):
    """One batch per route (a batch of many queries has more work items than the grid has warps, so the later
    leaves' items start after the thresholds rose); returns {cell: (queries, approx, skipped)}."""
    flat = [(cell, x, o) for cell, pairs in cells.items() for x, o in pairs]
    res = searcher.search([x for _, x, _ in flat])
    seen = {cell: [0, 0, 0] for cell in cells}
    for i, ((cell, x, o), m) in enumerate(zip(flat, res)):
        assert_matches_oracle(m, oracle(orc, o), ctx=f"{route}/{cell}[{i}] {list(x.terms)} F{list(x.filter_terms)} "
                                                     f"N{list(x.not_terms)} fac={x.factors} wqf={x.wqf} k={x.maxitems} "
                                                     f"first={x.first} cal={x.check_at_least}")
        c = seen[cell]
        c[0] += 1
        c[1] += bool(m.flags & xgm.MSET_BOUNDS_APPROX)
        c[2] += bool(m.flags & xgm.MSET_COUNT_LOWER_BOUND)
    for cell, (n, approx, skipped) in seen.items():
        print(f"{route}/{cell}: {n} queries, {approx} pruned, {skipped} with a skipped item")
    return seen


@pytest.mark.parametrize("route", ["tile", "or3", "general", "wide"])
def test_or_bounds_match_oracle(bounds, route, monkeypatch):
    _, ids, ix, orc = bounds
    if route == "or3":
        monkeypatch.setenv("XGM_OR_TILE", "0")
    if route == "general":
        monkeypatch.setenv("XGM_OR_KERNEL", "1")
    wide = route == "wide"
    cells = {c: cell_pairs(c, ids, orc, wide) for c in (WIDE_WEIGHTINGS if wide else WEIGHTINGS)}
    s = xgm.Searcher(ix, max_batch=sum(len(p) for p in cells.values()), max_topk=MAX_TOPK)
    seen = run_cells(s, orc, cells, route)
    for cell, (n, approx, skipped) in seen.items():
        assert 2 * approx > n, f"{route}/{cell}: only {approx} of {n} queries pruned"
        if route != "tile":
            assert skipped > 0, f"{route}/{cell}: no query skipped a work item"


def test_wide_ors_without_bitmaps(bounds, monkeypatch):
    """The 6..16-leaf queries on an index without membership bitmaps (every leaf probed by decoding its blocks)
    give the same MSets."""
    path, ids, _, orc = bounds
    monkeypatch.setenv("XGM_BITMAP_K", "0")
    ix = xgm.Index.load_flat(path)
    assert ix.info().nbitmaps == 0
    cells = {c: cell_pairs(c, ids, orc, wide=True) for c in WIDE_WEIGHTINGS}
    s = xgm.Searcher(ix, max_batch=sum(len(p) for p in cells.values()), max_topk=MAX_TOPK)
    run_cells(s, orc, cells, "wide/no-bitmap")


def fingerprint(m):
    return (m.status, m.flags, m.docids.tobytes(), m.weights.tobytes(), m.matches_lower_bound,
            m.matches_estimated_raw, m.matches_upper_bound, m.exact_matches, bits(m.max_possible),
            bits(m.max_attained), bits(m.percent_scale_factor))


# out-of-range BM25 parameters and the values BM25Weight's constructor clamps them to
CLAMPED = (((1.2, 1.0, 1.5, 0.5), (1.2, 1.0, 1.0, 0.5)), ((1.2, 1.0, -0.5, 0.5), (1.2, 1.0, 0.0, 0.5)),
           ((-1.0, 1.0, 0.75, 0.5), (0.0, 1.0, 0.75, 0.5)), ((1.2, -2.0, 0.75, 0.5), (1.2, 0.0, 0.75, 0.5)),
           ((-1.0, -2.0, 1.5, 0.0), (0.0, 0.0, 1.0, 0.0)))


def test_bm25_parameters_are_clamped(bounds):
    """k1, k3 < 0 weigh as 0 and b outside [0, 1] as its nearest end, as in the reference: the device equals the
    oracle at the clamped values and its own run at the clamped values, on AND and OR routes."""
    _, ids, ix, orc = bounds
    shapes = [(xgm.OP_OR, B.W3_SET, B.W3_WQF), (xgm.OP_OR, B.W1_SETS[1], None), (xgm.OP_OR, B.G_NAMES[4:12], None),
              (xgm.OP_AND, ("h_freq", "l_mid"), (2, 5)), (xgm.OP_AND, ("w_att",), None)]
    xs, os_ = [], []
    for raw, clamped in CLAMPED:
        for op, names, wqf in shapes:
            for k, first, cal in ((10, 0, 0), (100, 3, B.NDOCS)):
                for p in (raw, clamped):
                    kw = dict(first=first, maxitems=k, check_at_least=cal, wqf=wqf, bm25=p)
                    xs.append(xgm.Query(op, list(names), **kw))
                    os_.append(O.Query(op=op, terms=[ids[n] for n in names], **dict(kw, bm25=clamped)))
    res = xgm.Searcher(ix, max_batch=len(xs), max_topk=MAX_TOPK).search(xs)
    for i in range(0, len(xs), 2):
        ctx = f"clamp[{i}] {list(xs[i].terms)} {xs[i].bm25} -> {xs[i + 1].bm25}"
        assert_matches_oracle(res[i], oracle(orc, os_[i]), ctx)
        assert fingerprint(res[i]) == fingerprint(res[i + 1]), ctx
