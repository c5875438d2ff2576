"""Cost of a backfill (mm_backfill: open lobby slots filled from their queues, nearest rating first) against the host
alternative, mm_pool_read + numpy selection + mm_take.

config3 (32 groups, 5v5, rating order), 10 M resident players, no tick.  Cases: 1 request; 1 000 requests of 1-5
players over all queues; 10 000 requests of 1-5 players on one queue (the plan serves one queue's requests in order, in
one warp: its sequential worst case).  Every measured call starts from the same state (mm_restore of one mm_snapshot,
not timed).  Host clock over the blocking calls (median of --calls); the device time of the kernels one call launches
from torch.profiler in a separate run, split into the plan (k_bf_plan, k_bf_keys), the count pass (k_band_prep,
k_band_count, k_band_scan), the place pass (k_band_limit, k_band_place) and the output gather (k_bf_out).  Prints one
JSON line with the card's name and power limit, read in the same run.

    python tools/exp_backfill.py [--calls 7]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, kernel_us, stats  # noqa: E402

PARTS = {"plan": ("k_bf_plan", "k_bf_keys"), "count": ("k_band_prep", "k_band_count", "k_band_scan"),
         "place": ("k_band_limit", "k_band_place"), "out": ("k_bf_out",)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    rng = np.random.default_rng(1)
    G = cfg.n_groups

    def reqs(k, one_queue):
        g = np.full(k, 17) if one_queue else rng.integers(0, G, k)
        lo = np.array([cfg.group_lo[x] for x in g])
        hi = np.array([cfg.group_hi[x] for x in g])
        return (np.zeros(k, np.int64), g, rng.integers(lo, hi + 1), rng.integers(1, 6, k), np.full(k, -1))

    cases = {"1": reqs(1, False), "1000_all_queues": reqs(1000, False), "10000_one_queue": reqs(10_000, True)}
    out = {"workload": name, "players": n}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.snapshot()
        for label, r in cases.items():
            us = []
            for _ in range(args.calls + 1):  # the first call warms up
                e.restore()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                n_taken, got = e.backfill(*r)
                us.append((time.perf_counter() - t0) * 1e6)
            e.restore()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.backfill(*r)
                torch.cuda.synchronize()
            out[label] = {"players_taken": int(n_taken.sum()), "backfill_us": stats(us[1:]),
                          "kernels_us": {k: kernel_us(prof, v) for k, v in PARTS.items()}}
        # the host alternative, once per request set of 1 000: read the pool, select on the host, take
        from tests.test_backfill import restate
        e.restore()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p = e.pool_read()
        t1 = time.perf_counter()
        _, want = restate(cfg, p["id"], p["rating"], p["mode"], cases["1000_all_queues"])
        t2 = time.perf_counter()
        e.take(np.concatenate(want))
        t3 = time.perf_counter()
        out["host_alternative_1000_us"] = {"pool_read": (t1 - t0) * 1e6, "select": (t2 - t1) * 1e6,
                                           "take": (t3 - t2) * 1e6, "total": (t3 - t0) * 1e6}
    out["timing"] = ("host clock around the blocking calls (request upload, kernels, the counter read, the member copy); "
                     "kernels: torch.profiler device time of one call")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
