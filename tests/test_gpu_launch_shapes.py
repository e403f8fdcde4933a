"""Launch shapes of a searcher: its kernels' grids, their shared-memory opt-ins and the number of launches a batch takes.

A searcher's max_topk sets its keep_cap (2048 at max_topk 10, 8192 at 1000), and keep_cap sets the top-k kernel's
shared memory and resident grid.  Searchers of different keep_cap must give the oracle's answers whichever of them
is created or launches first, in a fresh process, and when host threads create and use them at once.  A batch's
kernel_launches depends on the batch alone, and is pinned for three batch shapes."""
import json
import os
import random
import subprocess
import sys
import threading

import pytest

from oracle import oracle as O
from tests.util import assert_matches_oracle
from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ND, V = 30000, 20000


def corpus():
    return xgm.Index.synthetic(ND, V), O.Index.synthetic(ND, V)


@pytest.fixture(scope="module")
def indexes():
    return corpus()


def pair(op, terms, **kw):
    return xgm.Query(op, list(terms), **kw), O.Query(op=op, terms=list(terms), **kw)


def ranked_batch():
    """100 queries, top 10 each.  Half are ORs of 2-3 of the 50 most frequent terms counted in full, thousands of
    stored matches that xgm_topk_kernel ranks; the others are ANDs of two rarer terms with a handful of matches,
    which xgm_topk_small_kernel finishes."""
    rng = random.Random(4242)
    out = []
    for i in range(100):
        if i % 2:
            out.append(pair(xgm.OP_OR, rng.sample(range(50), rng.choice([2, 3])), maxitems=10, check_at_least=ND))
        else:
            out.append(pair(xgm.OP_AND, rng.sample(range(3000), 2), maxitems=10))
    return out


def check(orc, res, pairs, ctx):
    for i, (m, (x, o)) in enumerate(zip(res, pairs)):
        assert_matches_oracle(m, orc.match(o), ctx=f"{ctx}[{i}] op={x.op} {x.terms} k={x.maxitems}")


def searchers_in_order(max_topks):
    """Creates one searcher per max_topk in the given order, then runs ranked_batch() on each in that order and
    checks it against the oracle.  Returns kernel_launches per max_topk."""
    ix, orc = corpus()
    pairs = ranked_batch()
    searchers = [xgm.Searcher(ix, max_batch=len(pairs), max_topk=k) for k in max_topks]
    launches = {}
    for k, s in zip(max_topks, searchers):
        check(orc, s.search([x for x, _ in pairs]), pairs, f"max_topk={k}")
        launches[k] = s.last_stats().kernel_launches
    return launches


def test_searcher_order(indexes):
    """keep_cap 2048 and 8192 created small-first and large-first, each order in a fresh process, so that the first
    searcher is also the first to launch every kernel on the device."""
    _, orc = indexes
    assert any(orc.match(o).exact > 256 for _, o in ranked_batch()[1::2]), "the ORs must reach xgm_topk_kernel"
    runs = {}
    for order in ((10, 1000), (1000, 10)):
        p = subprocess.run([sys.executable, "-m", "tests.test_gpu_launch_shapes"] + [str(k) for k in order], cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, f"order {order}:\n{p.stderr[-3000:]}"
        runs[order] = json.loads(p.stdout.strip().splitlines()[-1])
    print(f"kernel_launches: {runs}")
    assert runs[(10, 1000)] == runs[(1000, 10)]
    assert len(set(runs[(10, 1000)].values())) == 1, "the same batch takes the same launches at any keep_cap"


def test_concurrent_searchers(indexes):
    """Four host threads at once, each creating its own searcher of a different max_topk (keep_cap 2048, 2048, 4096
    and 8192) on the same index and running ranked_batch() once."""
    ix, orc = indexes
    pairs = ranked_batch()
    max_topks = (10, 100, 300, 1000)
    start = threading.Barrier(len(max_topks))
    results, errors = {}, []

    def worker(k):
        try:
            start.wait()
            s = xgm.Searcher(ix, max_batch=len(pairs), max_topk=k)
            results[k] = (s.search([x for x, _ in pairs]), s.last_stats().kernel_launches)
            s.close()
        except Exception as e:  # noqa: BLE001 -- reported below, on the test's thread
            errors.append(f"max_topk={k}: {e!r}")

    threads = [threading.Thread(target=worker, args=(k,)) for k in max_topks]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for k, (res, _) in sorted(results.items()):
        check(orc, res, pairs, f"thread max_topk={k}")
    assert len({n for _, n in results.values()}) == 1


def bitmap_ands(n):
    """ANDs of 2-3 terms among the 1000 most frequent, which all have membership bitmaps."""
    rng = random.Random(500)
    return [pair(xgm.OP_AND, rng.sample(range(1000), rng.choice([2, 3])), maxitems=10) for _ in range(n)]


def tile_ors(n):
    """Relevance-ordered ORs of 2-5 bitmap leaves: the bitmap-union tile kernel, then xgm_or3_kernel<1>."""
    rng = random.Random(600)
    return [pair(xgm.OP_OR, rng.sample(range(600), rng.choice([2, 3, 4, 5])), maxitems=10) for _ in range(n)]


# kernel_launches of each batch.  bench.py reports it as launches_per_step: a change here is a change in the work a
# batch enqueues, not in how it is counted.
LAUNCHES = {"single AND": 5, "300 bitmap ANDs, range-major": 8, "150 tile ORs": 12}


def test_kernel_launches_pinned(indexes):
    """A one-query batch (level-order work list), 300 bitmap ANDs (range-major: three expansion kernels) and 150
    ORs on the tile route, each checked against the oracle."""
    ix, orc = indexes
    s = xgm.Searcher(ix, max_batch=300, max_topk=100)
    got = {}
    for name, pairs in (("single AND", [pair(xgm.OP_AND, [3, 17], maxitems=10)]),
                        ("300 bitmap ANDs, range-major", bitmap_ands(300)),
                        ("150 tile ORs", tile_ors(150))):
        check(orc, s.search([x for x, _ in pairs]), pairs, name)
        got[name] = s.last_stats().kernel_launches
    print(f"kernel_launches: {got}")
    assert got == LAUNCHES


if __name__ == "__main__":
    print(json.dumps(searchers_in_order([int(a) for a in sys.argv[1:]])))
