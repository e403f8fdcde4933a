"""Kernel time of the multi-shard device merge at the bench's sizes: N in {2, 4, 8} gathered result slabs of full
parts (every part holds k records), C2/C5 = 4096/N queries with k = 100, C3 = 512/N queries with k = 1000.

Columns, timed alternately in one process with CUDA events (median over rounds of LAUNCHES launches, after
warm-up; min-max of the rounds in brackets):
  topk_slab   xgm_merge_topk_device_slab (relevance, no keys)
  mset_rel    xgm_merge_mset_device_slab with every order XGM_SORT_REL (keys not read)
  mset_valrel xgm_merge_mset_device_slab with every order XGM_SORT_VAL_REL (keys read and written)
A library without xgm_merge_mset_device_slab (before the keyed merge) gets only the first column, so the relevance
entry point can be compared across versions.  Prints the card's name and power limit with the table.

    python scripts/merge_perf.py [--rounds R]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import os

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402
from xapiand_b200 import xgm  # noqa: E402

LAUNCHES = 20
SORT_REL, SORT_VAL_REL = 0, 1


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def gathered_slabs(nparts, nq, k, seed):
    """nparts slabs weights | docids | records | keys (256-byte aligned regions), every (part, query) holding k
    records sorted by weight descending and, at the same time, by key ascending."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    up = lambda v: (v + 255) // 256 * 256  # noqa: E731
    ns = nq * k
    off_d = up(ns * 8)
    off_c = off_d + up(ns * 4)
    off_k = off_c + up(nq * 32)
    nbytes = off_k + up(ns * 8)
    G = torch.zeros(nparts * nbytes, dtype=torch.uint8, device="cuda")
    for p in range(nparts):
        s = G[p * nbytes:(p + 1) * nbytes]
        w = torch.rand((nq, k), generator=g, device="cuda", dtype=torch.float64).sort(-1, descending=True).values * 30
        d = torch.rand((nq, 4 * k), generator=g, device="cuda").argsort(-1)[:, :k].to(torch.int32) + 1
        key = torch.randint(0, 1 << 62, (nq, k), generator=g, device="cuda").sort(-1).values
        s[:ns * 8].view(torch.float64).copy_(w.reshape(-1))
        s[off_d:off_d + ns * 4].view(torch.int32).copy_(d.reshape(-1))
        rec = torch.zeros((nq, 8), dtype=torch.int32, device="cuda")
        rec[:, 0] = k
        s[off_c:off_c + nq * 32].view(torch.int32).copy_(rec.reshape(-1))
        s[off_k:off_k + ns * 8].view(torch.int64).copy_(key.reshape(-1))
    return G, nbytes, off_d, off_c, off_k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    args = ap.parse_args()
    L = xgm.lib()
    L.xgm_merge_topk_device_slab.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
                                             C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    keyed = hasattr(L, "xgm_merge_mset_device_slab")
    if keyed:
        L.xgm_merge_mset_device_slab.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p,
                                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}; keyed entry point: {'yes' if keyed else 'no'}")
    stream = torch.cuda.current_stream().cuda_stream
    rows = []
    for cfg, nq_all, k in (("C2/C5", 4096, 100), ("C3", 512, 1000)):
        for n in (2, 4, 8):
            nq = nq_all // n
            G, nbytes, off_d, off_c, off_k = gathered_slabs(n, nq, k, seed=n * 1000 + k)
            ow = torch.empty(nq * k, dtype=torch.float64, device="cuda")
            od = torch.empty(nq * k, dtype=torch.int32, device="cuda")
            ok = torch.empty(nq * k, dtype=torch.int64, device="cuda")
            on = torch.empty(nq, dtype=torch.int32, device="cuda")
            rel = torch.full((nq,), SORT_REL, dtype=torch.uint8, device="cuda")
            valrel = torch.full((nq,), SORT_VAL_REL, dtype=torch.uint8, device="cuda")

            def topk_slab():
                return L.xgm_merge_topk_device_slab(G.data_ptr(), nbytes, off_d, off_c, n, nq, k, k, ow.data_ptr(),
                                                    od.data_ptr(), on.data_ptr(), stream)

            def mset(orders):
                return lambda: L.xgm_merge_mset_device_slab(G.data_ptr(), nbytes, off_d, off_c, off_k, orders.data_ptr(),
                                                            n, nq, k, 0, k, ow.data_ptr(), od.data_ptr(), ok.data_ptr(),
                                                            on.data_ptr(), stream)

            cols = {"topk_slab": topk_slab}
            if keyed:
                cols.update(mset_rel=mset(rel), mset_valrel=mset(valrel))
            for f in cols.values():  # warm-up (module load, shared-memory opt-in)
                for _ in range(5):
                    if f() != 0:
                        raise RuntimeError(L.xgm_last_error().decode())
            torch.cuda.synchronize()
            times = {c: [] for c in cols}
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            for _ in range(args.rounds):
                for c, f in cols.items():
                    ev[0].record()
                    for _ in range(LAUNCHES):
                        f()
                    ev[1].record()
                    ev[1].synchronize()
                    times[c].append(ev[0].elapsed_time(ev[1]) * 1e3 / LAUNCHES)
            row = {"config": cfg, "N": n, "nq": nq, "k": k}
            for c, ts in times.items():
                ts.sort()
                row[c] = {"median_us": round(ts[len(ts) // 2], 2), "min_us": round(ts[0], 2), "max_us": round(ts[-1], 2)}
            rows.append(row)
            cells = "  ".join(f"{c} {v['median_us']:8.2f} [{v['min_us']:.2f}-{v['max_us']:.2f}] us"
                              for c, v in row.items() if isinstance(v, dict))
            print(f"{cfg:6s} N={n} nq={nq:5d} k={k:5d}  {cells}", flush=True)
            del G
    print(json.dumps({"card": name, "power_limit": power, "keyed": keyed, "rows": rows}))


if __name__ == "__main__":
    main()
