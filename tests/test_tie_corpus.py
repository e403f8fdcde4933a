"""Pins the corpora of tests/test_gpu_topk_stress.py and tests/test_gpu_work_split.py with the oracle alone (no GPU):
an edit to tests/tie_corpus.py that took away the tie masses, the exact intersection sizes or the missing values
would leave those tests passing without exercising what they are for."""
import shutil
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import tie_corpus as T


@pytest.fixture(scope="module")
def tie_oracle():
    tmp = tempfile.mkdtemp(prefix="xgm_ties_")
    path, names = T.write_tie_corpus(tmp)
    yield {n: i for i, n in enumerate(names)}, O.Index.load_flat(path)
    shutil.rmtree(tmp, ignore_errors=True)


def full(orc, op, terms, factors=None):
    return orc.match(O.Query(op=O.OP_AND if op == "AND" else O.OP_OR, terms=terms, factors=factors,
                             maxitems=T.NDOCS, check_at_least=T.NDOCS))


def test_corpus_shape(tie_oracle):
    ids, orc = tie_oracle
    assert orc.doccount == T.NDOCS and orc.lastdocid == T.LASTDOCID  # docid gaps
    assert set(np.unique(orc.doclen()[orc.doclen() > 0]).tolist()) == set(T.LENGTHS)
    bitmap_min = max(64, T.LASTDOCID // 256)  # termfreq that earns a membership bitmap
    assert orc.termfreq(ids["r_rare"]) < bitmap_min
    for i in range(1, 9):
        assert orc.termfreq(ids[f"t{i:02d}"]) >= 3000
    assert orc.termfreq(ids["t01"]) > 35000
    _, w = orc.postings(ids["b_bool"])
    assert len(w) > 0 and not w.any()


@pytest.mark.parametrize("route", list(T.TIE_ROUTES))
def test_tie_routes_have_a_top_tie_mass(tie_oracle, route):
    """More than keep_cap matches share the best weight (so the radix select must run), and the ANDs have few
    distinct weights: three document lengths times wdf 1 or 2 per term."""
    ids, orc = tie_oracle
    for op, terms, factors in T.TIE_ROUTES[route]:
        r = full(orc, op, [ids[t] for t in terms], factors)
        top = int((r.weights == r.weights.max()).sum())
        assert top > T.KEEP_CAP, (terms, top)
        if op == "AND":
            assert len(np.unique(r.weights)) <= len(T.LENGTHS) * 2 ** len(terms), terms


def test_flat_term_overflows_the_largest_top_k(tie_oracle):
    """keep_cap is 8192 when max_topk is the C-ABI's 4096: f_flat's tie mass must still exceed it."""
    ids, orc = tie_oracle
    w = full(orc, "AND", [ids["f_flat"]]).weights
    assert int((w == w.max()).sum()) > 8192


@pytest.mark.parametrize("n", T.EDGE_SIZES)
def test_edge_intersections_are_exact(tie_oracle, n):
    ids, orc = tie_oracle
    a, b = T.edge_names(n)
    r = full(orc, "AND", [ids[a], ids[b]])
    assert r.exact == n and len(r.docids) == n
    assert len(np.unique(r.weights)) <= len(T.LENGTHS)


def test_value_slot_missing_share():
    orc = O.Index.synthetic(T.VALUE_NDOCS, T.VALUE_VOCAB, values=True)
    voff, keys = T.value_slot_arrays(orc)
    nv = orc.values()[0]
    missing = float((nv[1:] == 0).mean())
    assert abs(missing - T.VALUE_MISSING_SHARE) < 0.02
    assert len(voff) == orc.lastdocid + 2 and int(voff[-1]) == len(keys) and keys.min() >= 1
    for ts in T.VALUE_AND_SETS:
        for rev in (False, True):
            r = orc.match(O.Query(op=O.OP_AND, terms=ts, maxitems=T.VALUE_NDOCS, sort_by=O.SORT_VAL, sort_slot=0,
                                  sort_reverse=rev, sort_keymaker=True, sort_missing=T.missing_key(rev)))
            assert r.sortvals[0] == T.missing_key(rev)
            assert int((r.sortvals == T.missing_key(rev)).sum()) > T.KEEP_CAP
