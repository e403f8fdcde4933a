"""Index and searcher lifecycles keep no device memory: every array, pinned buffer, stream and event of an index and a
searcher is freed when they are closed, including the work-list buffers a batch grows on first use."""
import gc
import random

import pytest

from xapiand_b200 import xgm

pytestmark = pytest.mark.gpu

ND, V = 30000, 20000
ROUNDS = 10
# 5000 queries x 32768 candidates (max_topk 1024) x 20 bytes: a round holds over 3 GB of device memory, large against
# what other work on the device moves between two readings of its free memory
MAX_BATCH, MAX_TOPK = 5000, 1024


def free_bytes():
    import torch
    torch.cuda.synchronize(0)
    return torch.cuda.mem_get_info(0)[0]


def batches():
    """16 ANDs and ORs, then MAX_BATCH all-bitmap ANDs (terms among the 1000 most frequent).  The second batch is
    range-major: its bitmap list stages 2 x 5000 rows, more than the 8192 a searcher starts with, and it allocates
    the per-range run table."""
    rng = random.Random(5)
    small = [xgm.Query(rng.choice([xgm.OP_AND, xgm.OP_OR]), rng.sample(range(1000), rng.choice([2, 3])), maxitems=10)
             for _ in range(16)]
    large = [xgm.Query(xgm.OP_AND, rng.sample(range(1000), rng.choice([2, 3, 4])), maxitems=10)
             for _ in range(MAX_BATCH)]
    return xgm.QueryBatch(small), xgm.QueryBatch(large)


def one_round(small, large):
    """Build, search twice, close.  Returns the MSets' docids and the free device memory while everything is held."""
    ix = xgm.Index.synthetic(ND, V)
    s = xgm.Searcher(ix, max_batch=MAX_BATCH, max_topk=MAX_TOPK)
    out = []
    for batch in (small, large):
        res = s.search(batch)
        assert all(m.status == 0 for m in res)
        out.append([m.docids.tobytes() for m in res])
    held = free_bytes()
    s.close()
    ix.close()
    return out, held


def test_rounds_keep_no_device_memory():
    small, large = batches()
    gc.collect()
    before = free_bytes()
    first, held = one_round(small, large)
    footprint = before - held
    after_first = free_bytes()
    for _ in range(ROUNDS - 1):
        res, _ = one_round(small, large)
        assert res == first
    after_last = free_bytes()
    print(f"round footprint {footprint / 2**30:.2f} GiB, free after round 1 {after_first / 2**30:.2f} GiB, "
          f"after round {ROUNDS} {after_last / 2**30:.2f} GiB")
    assert footprint >= 2 << 30
    # a leak shows as less free memory after the last round than after the first
    assert after_first - after_last < footprint / 4
