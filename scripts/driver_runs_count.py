"""Work of the bitmap AND list for bench.py's C2 and C5 batches (step 0): driver blocks the AND kernel decodes when
every query decodes its own driver (one item list per query) and when the queries that share a driver share the
decode (runs of up to RUN queries), computed from the index's term frequencies; and the work items of the list as
the library in this tree plans them (one batch on the GPU).  Prints one JSON line per configuration."""
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from xapiand_b200 import xgm  # noqa: E402

RUN = 6  # XGM_BM_RUN
BLOCK = 128  # postings per block


def count(name):
    cfg = bench.config(name)
    ix = xgm.Index.synthetic(cfg["docs"], bench.VOCAB, seed=bench.SEED, values=cfg["values"], host_threads=16)
    qs = bench.gen_queries(cfg, 0, cfg["batch"])
    names = sorted({bench.term_name(t) for terms, _ in qs for t in terms})
    tf = dict(zip(names, (int(f) for f in ix.term_freqs(names))))
    per_driver = collections.Counter()
    for terms, _ in qs:
        per_driver[min((bench.term_name(t) for t in terms), key=lambda n: (tf[n], n))] += 1
    nblk = {d: (tf[d] + BLOCK - 1) // BLOCK for d in per_driver}
    s = xgm.Searcher(ix, max_batch=cfg["batch"], max_topk=cfg["topk"])
    s.search([bench.xgm_query(cfg, q) for q in qs])
    return dict(config=name, queries=len(qs), drivers=len(per_driver), max_queries_per_driver=max(per_driver.values()),
                runs=sum((n + RUN - 1) // RUN for n in per_driver.values()),
                driver_blocks_per_query=sum(n * nblk[d] for d, n in per_driver.items()),
                driver_blocks_per_run=sum((n + RUN - 1) // RUN * nblk[d] for d, n in per_driver.items()),
                work_items=s.last_stats().work_items)


if __name__ == "__main__":
    for name in sys.argv[1:] or ["C2", "C5"]:
        print(json.dumps(count(name)), flush=True)
