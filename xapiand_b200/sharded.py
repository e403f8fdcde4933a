"""Host-side logic of the sharded (multi-GPU) path — Xapiand's two-phase scheme
(src/database/handler.cc:1485-1551) expressed over torch.distributed:

  phase 1  DocMatcher::prepare_mset per shard + merger.add_prepared_mset  → global statistics
           (Weight::Internal::operator+=, src/xapian/weight/weightinternal.cc:54-72): one all-reduce
  phase 2  per-shard get_mset(0, first+maxitems) with those statistics, mset.unshard_docids(shard, n),
           merger.merge_mset(...)                                          → one all-gather + merge

Works with any backend (NCCL on GPUs, gloo in the CPU tests); the device-resident variant used for the
throughput numbers lives in bench.py (statistics through xapiand_b200/shm_exchange.py on one node, one all-to-all of
per-query-slice top-k + xgm_merge_topk_device, which merges by relevance).  A device path for value-sorted batches
exchanges whole result slabs, sort keys included, and merges them with xgm.merge_device_slabs
(xgm_merge_mset_device_slab: every sort order, reverse and first, records only); merge_over_ranks below is the
full merge, statistics included.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch
import torch.distributed as dist

from . import xgm


def global_stats(local_termfreqs: Sequence[int], doccount: int, total_length: int, device="cpu"):
    """Sum (collection_size, total_length, per-term termfreq) over all ranks."""
    t = torch.tensor([doccount, total_length] + list(local_termfreqs), dtype=torch.int64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t)
    v = t.tolist()
    return v[0], v[1], v[2:]


def merge_over_ranks(local: xgm.MSet, first: int, maxitems: int, sort_by: int = xgm.SORT_REL,
                     sort_reverse: bool = False) -> xgm.MSet:
    """all-gather the per-shard MSets (docids still shard-local), unshard and merge like Matcher::merge_mset."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    payload = dict(docids=xgm.unshard(local.docids, rank, world), weights=np.asarray(local.weights),
                   sort_keys=None if local.sort_keys is None else np.asarray(local.sort_keys),
                   info=(local.first, local.matches_lower_bound, local.matches_estimated_raw, local.matches_upper_bound,
                         local.max_possible, local.max_attained, local.percent_scale_factor, local.exact_matches,
                         local.status, local.flags))
    parts: List[dict] = [None] * world
    if world > 1:
        dist.all_gather_object(parts, payload)
    else:
        parts = [payload]
    msets = [xgm.MSet(p["docids"], p["weights"], p["sort_keys"], *p["info"]) for p in parts]
    return xgm.merge_msets(msets, first, maxitems, sort_by, sort_reverse)
