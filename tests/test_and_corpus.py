"""The witnesses of tests/and_corpus.py, pinned with the oracle and numpy alone: each holds, so that
tests/test_gpu_and_weights.py fails when the AND kernels read a neighbour's wdf, weigh a leaf without a Weight, or
add the weighted range source at the wrong place.  The FILTER and factor-0 shapes are also pinned against the
compiled reference where it is built."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests import and_corpus as A
from tests.util import bits

K1_0 = (0.0, 1.0, 0.5, 0.5)


@pytest.fixture(scope="module")
def corpus():
    tmp = tempfile.mkdtemp(prefix="xgm_and_")
    path, built = A.write_and_corpus(tmp)
    doclen, terms, doccount, nvals, vals, groups = built
    orc = O.Index.load_flat(path)
    orc.set_slot0(nvals, vals)
    yield dict(orc=orc, ids={t[0]: i for i, t in enumerate(terms)}, terms={t[0]: t[1:] for t in terms},
               doclen=doclen, groups=groups, nvals=nvals)
    shutil.rmtree(tmp, ignore_errors=True)


def specs(witness):
    return [s for s in A.witness_specs() if s["witness"] == witness]


def test_w1_queries_hit_wdf0_postings_under_k1_0(corpus):
    c = corpus
    zero = set(c["groups"]["zero"].tolist())
    hit_zero_len = False
    for s in specs("W1"):
        m = c["orc"].match(A.oracle_query(c["ids"], s, "k1=0.0 b=0.0 mnl=0.5", maxitems=100, check_at_least=A.NDOCS))
        assert len(m.docids) and m.exact > 0, s
        # every match holds a wdf-0 posting of a boolean list, weighed under k1 = 0
        for n in s["names"] + s["filter_terms"]:
            d, w = c["terms"][n]
            if n.startswith("z_"):
                assert (w == 0).all() and np.isin(m.docids, d).all(), (s, n)
        hit_zero_len |= bool(zero & set(m.docids.tolist()))
    assert hit_zero_len, "no W1 query returns a document of length 0"


def depth(prog):
    sp = most = 0
    for op in prog:
        sp = sp + 1 if op >= 0 else sp - 1
        most = max(most, sp)
    return most


def test_w3_optional_trees_are_deeper_than_8(corpus):
    c = corpus
    for s in specs("W3"):
        tfs = [c["orc"].termfreq(c["ids"][n]) for n in s["maybe"]]
        assert 9 <= len(tfs) <= 15 and depth(O.or_program(tfs)) > 8, s
        m = c["orc"].match(A.oracle_query(c["ids"], s, "k1=1.2 b=0.5 mnl=0.5"))
        assert set(c["groups"]["all_maybe"].tolist()) & set(m.docids.tolist()), s


def test_w4_wdfs_differ_from_their_neighbours(corpus):
    c = corpus
    core = c["groups"]["core"]
    for n, (d, w) in c["terms"].items():
        if n.startswith("z_"):
            continue
        assert (w[1:] != w[:-1]).all(), n
        if len(d) >= 2 * A.BLOCK and n in A.EXTRA:
            pos = np.searchsorted(d, core)
            assert (d[pos] == core).all(), n
            assert (pos % A.BLOCK == 0).any() and (pos % A.BLOCK == A.BLOCK - 1).any(), n
    assert max(int(w.max()) for d, w in c["terms"].values()) > 255
    near = [256 * g + e for g in range(1, A.LASTDOCID // 256 + 1) for e in (-1, 0, 1)]
    assert len(np.intersect1d(core, near)) >= 30 and len(np.intersect1d(core, np.arange(0, A.LASTDOCID, 32))) >= 10
    assert A.LASTDOCID % 32 and A.LASTDOCID % 256 and A.LASTDOCID % 65536
    # drivers and probes with and without a membership bitmap, and a probe list that loses it at MID_BITMAP_K
    tf = {n: len(c["terms"][n][0]) for n in A.EXTRA}
    assert tf["b_drv"] < A.BITMAP_MIN and tf["p_nobm"] < A.BITMAP_MIN and tf["b_drvbm"] >= A.BITMAP_MIN
    assert tf["p_coarse"] < A.LASTDOCID // A.MID_BITMAP_K <= tf["p_fine"]
    assert len(c["terms"]["z_rare"][0]) < min(tf.values())


def resum(c, s, cell, docids, src_at):
    """The weights of docids re-summed in numpy, MultiAndPostList order, the source added before child src_at."""
    L = O.lib()
    k1, k3, b, mnl = A.WEIGHTINGS[cell]
    fac, wqf = A.cell_spec(s, cell)
    o = c["orc"]
    n = len(s["names"])
    out = np.zeros(len(docids))
    tws = []
    for j, name in enumerate(s["names"]):
        tw, lf = C.c_double(), C.c_double()
        L.orc_bm25_init(o.doccount, o.total_length, o.termfreq(c["ids"][name]), wqf[j] if wqf else 1,
                        fac[j] if fac else 1.0, k1, k3, b, C.byref(tw), C.byref(lf))
        tws.append((tw.value, lf.value))
    order = O.and_order([o.termfreq(c["ids"][x]) for x in s["names"]])
    for i, d in enumerate(docids):
        acc = 0.0
        for pos in range(n + 1):
            if pos == src_at:
                acc += s["src"]
            if pos == n:
                break
            j = order[pos]
            dd, ww = c["terms"][s["names"][j]]
            wdf = int(ww[np.searchsorted(dd, d)])
            acc += L.orc_bm25_sumpart(tws[j][0], tws[j][1], k1, b, mnl, wdf, int(c["doclen"][d]))
        out[i] = acc
    return out


def test_w2_source_place_changes_the_bits(corpus):
    """The source sorts in at every place 0 .. n of 1-, 2- and 3-term bases, and for every witness query a re-sum
    with the source one place off changes the bits of at least one top-k weight under one of the source factors.
    Places 0 and 1 give the same sum (0 + s + a = 0 + a + s exactly), so only a move that involves a place >= 2 can
    show."""
    c = corpus
    vf = int((c["nvals"] != 0).sum())
    places = set()
    for names in A.SRC_SETS:
        tfs = [c["orc"].termfreq(c["ids"][n]) for n in names]
        n = len(tfs)
        at = O.and_order(tfs + [vf]).index(n)
        places.add((n, at))
        for cell in ("k1=1.2 b=0.5 mnl=0.5", "k1=0.0 b=0.0 mnl=0.0", "k1=20.0 b=1.0 mnl=0.0", "k3=0 wqf"):
            moved = set()
            for f in A.SRC_FACTORS:
                s = A.spec(names, src=f)
                m = c["orc"].match(A.oracle_query(c["ids"], s, cell))
                assert len(m.docids) >= 50, (s, cell)
                assert resum(c, s, cell, m.docids, at).tobytes() == m.weights.tobytes(), (s, cell)
                moved |= {off for off in (at - 1, at + 1)
                          if 0 <= off <= n and resum(c, s, cell, m.docids, off).tobytes() != m.weights.tobytes()}
            want = {off for off in (at - 1, at + 1) if 0 <= off <= n and max(at, off) >= 2}
            assert want <= moved, (names, cell, at, want - moved)
    assert places == {(n, p) for n in (1, 2, 3) for p in range(n + 1)}, places


def test_oracle_weights_are_never_nan(corpus):
    c = corpus
    for s in A.witness_specs():
        for cell in A.WEIGHTINGS:
            m = c["orc"].match(A.oracle_query(c["ids"], s, cell, maxitems=100, check_at_least=A.NDOCS))
            assert not np.isnan(m.weights).any(), (s, cell)
            assert not np.isnan(m.max_attained) and not np.isnan(m.percent_scale_factor), (s, cell)


@pytest.mark.skipif(not O.have_reference(), reason="oracle/_ref not built")
def test_unweighted_leaves_match_the_reference():
    """Boolean terms written by Document::add_boolean_term (wdf 0, some documents of length 0) as OP_FILTER terms and
    as OP_SCALE_WEIGHT(…, 0) leaves, at k1 = 0 and at b = 1 with min_normlen = 0: the reference never weighs them,
    and the oracle equals it bit for bit."""
    tmp = tempfile.mkdtemp(prefix="xgm_refbool_")
    try:
        db = os.path.join(tmp, "db")
        O.ref_build(db, 3000, 400, seed=9, boolean_terms=3)
        flat = os.path.join(tmp, "x.flat")
        subprocess.check_call([O.REF_RUNNER, "export", "--db", db, "--out", flat], stdout=subprocess.DEVNULL)
        orc = O.Index.load_flat(flat)
        ids = {orc.name(t): t for t in range(orc.nterms)}
        assert (orc.doclen()[1:] == 0).any()
        words = sorted((orc.termfreq(t), n) for n, t in ids.items() if not n.startswith("XB"))
        a, b_ = words[-30][1], words[-60][1]  # frequent enough to meet the boolean terms often
        shapes = [([a, b_], dict(filter_terms=["XB0"])), ([a], dict(filter_terms=["XB1", "XB2"])),
                  (["XB0", a], dict(factors=[0.0, 1.0])), (["XB0", "XB1"], dict(factors=[0.0, 0.0])),
                  (["XB2"], dict(factors=[0.0])), ([a, "XB1"], dict(factors=[1.0, 0.0], filter_terms=["XB0"]))]
        lines, qs = [], []
        for bm25 in ((0.0, 1.0, 0.5, 0.5), (0.0, 1.0, 0.0, 0.0), (1.2, 1.0, 1.0, 0.0)):
            for names, kw in shapes:
                fac = kw.get("factors")
                leaves = [f"{n}^{fac[j]!r}" if fac and fac[j] != 1.0 else n for j, n in enumerate(names)]
                lines.append(O.query_line("AND", leaves, 0, 100, 3000, filter_terms=kw.get("filter_terms", ()),
                                          bm25=bm25))
                qs.append(O.Query(op=O.OP_AND, terms=[ids[n] for n in names], maxitems=100, check_at_least=3000,
                                  factors=fac, filter_terms=[ids[n] for n in kw.get("filter_terms", ())], bm25=bm25))
        _, ref = O.ref_query([db], lines, tmp)
        for line, q, r in zip(lines, qs, ref):
            m = orc.match(q)
            assert len(r.docids) > 0, line
            assert list(m.docids) == r.docids, line
            assert m.weights.tobytes() == np.asarray(r.weights, np.float64).tobytes(), line
            assert bits(m.max_attained) == bits(r.max_attained) and not np.isnan(m.weights).any(), line
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
