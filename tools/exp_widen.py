"""Cost of a widening search (mm_widen: lobbies around the players who waited longest, each in a window that grows
with its wait) after an S1 tick.

config3 (32 groups, 5v5, rating order): 10 M players, one tick at max_spread 2 under a lobby budget of 1 000 lobbies
per queue (without one the tick matches nearly everyone), then mm_widen with every queue on, min_wait chosen so that
0.1 %, 1 % and 10 % of the players left are anchors.  Every measured call starts from the same state (mm_restore of
one mm_snapshot, not timed).  Host clock over the blocking call (median of --calls, after one warm-up call) and the
call's own device time (mm_widen_stats.device_us); the kernels of one call from torch.profiler in a separate run,
split into the anchor passes and ranks, the plan, the gather / take and the output.
The plan serves each queue's anchors one after another in one warp, so a queue with many anchors bounds the call.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_widen.py [--calls 5]
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

PARTS = {"anchors": ("k_wd_anchors", "k_wd_part_scan", "k_loc_rmap", "k_wd_rank"), "plan": ("k_wd_plan", "k_bf_keys"),
         "take": ("k_band_prep", "k_band_count", "k_band_scan", "k_band_limit", "k_band_place"),
         "out": ("k_wd_bases", "k_wd_hdr", "k_bf_out")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
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
    out = {"workload": name, "players": n, "card": card()}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("max_spread", 2)
        now = int(ts.max()) + 1
        e.set_lobby_budget(per_queue=[1000] * cfg.n_groups)  # the S1 tick leaves most of the pool queued
        e.tick(now)
        left = e.pool_read()
        wait = now - left["enq_ts"].astype(np.int64)
        out["resident"] = int(len(wait))
        e.snapshot()
        for share in (0.001, 0.01, 0.1):
            min_wait = int(np.quantile(wait, 1.0 - share))
            rules = e.widen_rules({(mode_idx, g): (min_wait, 3, 50, 5, 400) for g in range(cfg.n_groups)})
            host_us, dev_us = [], []
            for _ in range(args.calls + 1):  # the first call warms up
                e.restore()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                lob, mem, st = e.widen(now, rules, lobby_cap=1 << 20, member_cap=1 << 23)
                host_us.append((time.perf_counter() - t0) * 1e6)
                dev_us.append(st.device_us)
            e.restore()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.widen(now, rules, lobby_cap=1 << 20, member_cap=1 << 23)
                torch.cuda.synchronize()
            out[f"anchors_{share:g}"] = {
                "anchors": st.n_anchors, "absorbed": st.n_absorbed, "lobbies": st.n_lobbies, "matched": st.n_matched,
                "call_us": stats(host_us[1:]), "device_us": stats(dev_us[1:]),
                "kernels_us": {k: kernel_us(prof, v) for k, v in PARTS.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
