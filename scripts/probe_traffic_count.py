"""Probe traffic of the bitmap AND kernel for bench.py's C2 and C5 batches (step 0), as a MODEL computed from the
bench index's term frequencies; not hardware counters.  It assumes that the terms are independent, which the synthetic
corpus guarantees, so a query's driver postings (terms[0]) fall uniformly over the docids.

For every query the kernel probes the second list (terms[1]) once per driver posting:
  fine route    one 32-bit word of the membership bitmap; a 32-byte sector covers 256 docids.  Counted: the distinct
                sectors a query's postings touch, S (1 - (1 - 1/S)^D) for S sectors and D postings.
  coarse route  one word of the coarse bitmap (a bit per 8 docids, a sector covers 2048 docids), distinct sectors as
                above, plus one fine sector per posting whose coarse bit is set, D (1 - (1 - tf1 / lastdocid)^8),
                counted per load ("in step": the postings of one probe step are far apart, so they rarely share one).
A query takes the coarse route when that expected pass rate is at most COARSE_MAX (XGM_COARSE_PASS_MAX).  Prints one
JSON line per configuration: the bytes moved from L2 to the SMs by today's fine probes of every query, by the probes
with the route chosen per query, and the share of queries on each route."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from xapiand_b200 import xgm  # noqa: E402

COARSE_MAX = 0.1  # XGM_COARSE_PASS_MAX
SECTOR = 32  # bytes
FINE_DOCS, COARSE_DOCS = 256, 2048  # docids per sector of the fine and of the coarse bitmap


def distinct(sectors, postings):
    return sectors * (1.0 - (1.0 - 1.0 / sectors) ** postings)


def count(name):
    cfg = bench.config(name)
    ix = xgm.Index.synthetic(cfg["docs"], bench.VOCAB, seed=bench.SEED, values=cfg["values"], host_threads=16)
    n = ix.info().lastdocid
    qs = bench.gen_queries(cfg, 0, cfg["batch"])
    names = sorted({bench.term_name(t) for terms, _ in qs for t in terms})
    tf = dict(zip(names, (int(f) for f in ix.term_freqs(names))))
    fine_s, coarse_s = (n + FINE_DOCS - 1) // FINE_DOCS, (n + COARSE_DOCS - 1) // COARSE_DOCS
    today = routed = coarse_sectors = fine_loads = 0.0
    ncoarse = nprobe = 0
    for terms, _ in qs:
        lists = sorted((tf[bench.term_name(t)], bench.term_name(t)) for t in terms)
        if len(lists) < 2:
            continue
        d, t1 = lists[0][0], lists[1][0]
        nprobe += 1
        fine = distinct(fine_s, d)
        today += fine
        rate = 1.0 - (1.0 - t1 / n) ** 8
        if rate <= COARSE_MAX:
            ncoarse += 1
            c, f = distinct(coarse_s, d), d * rate
            coarse_sectors += c
            fine_loads += f
            routed += c + f
        else:
            routed += fine
    gb = SECTOR / 1e9
    return dict(config=name, model="independent terms; not hardware counters", coarse_max=COARSE_MAX,
                queries=len(qs), probing_queries=nprobe, coarse_route_queries=ncoarse,
                coarse_route_share=round(ncoarse / max(1, nprobe), 4),
                fine_probe_gb_today=round(today * gb, 3), probe_gb_routed=round(routed * gb, 3),
                coarse_sector_gb=round(coarse_sectors * gb, 3), in_step_fine_load_gb=round(fine_loads * gb, 3))


if __name__ == "__main__":
    for name in sys.argv[1:] or ["C2", "C5"]:
        print(json.dumps(count(name)), flush=True)
